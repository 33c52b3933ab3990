"""lf_jpeg_encode (csrc/jpeg_enc.cu) through jpeg.JpegEncoder against Pillow's encoder byte for byte, lf_draw_lane_points
through inference.draw_lane_points against the circle restatement, and inference.render_testset / test_model(...,
render_dir=...) against the golden overlays and the host loop (Pillow decode, cv2.circle, Pillow save)."""
import io
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import jpeg_enc_oracle as jo
from test_jpeg_enc_cpu import KINDS, MODES, QUALITIES, SIZES, content, frame, pil_encode, subsampling_of

pytestmark = pytest.mark.gpu


def _encode_all(frames, quality, sub):
    from lanedetection_end2end_b200.jpeg import JpegEncoder
    return JpegEncoder("cuda", quality=quality, subsampling=sub)(torch.from_numpy(np.stack(frames)).cuda())


@pytest.mark.parametrize("size", SIZES + [(720, 1280)], ids=["%dx%d" % s for s in SIZES + [(720, 1280)]])
def test_encoder_equals_pillow(size):
    """Every quality and mode, the five contents of a size in one batch."""
    h, w = size
    for mode in MODES:
        frames = [frame(kind, h, w, mode, seed=h * 1000 + w + k) for k, kind in enumerate(KINDS)]
        for q in QUALITIES:
            sub = subsampling_of(mode)
            got = _encode_all(frames, q, sub)
            for kind, a, d in zip(KINDS, frames, got):
                assert d == pil_encode(a, q, sub), (kind, mode, q)


def test_grayscale_4_4_4():
    a = frame("gradient", 33, 65, "gray")
    assert _encode_all([a], 75, "4:4:4")[0] == pil_encode(a, 75, "4:4:4")


@pytest.mark.parametrize("quality", [75, 95])
def test_batches_of_720p_frames(quality):
    """Batches of 1, 32 and 128 frames of 1280x720 (mixed contents) at 4:2:0."""
    rng = np.random.default_rng(quality)
    frames = [content(KINDS[k % 5] if k % 3 else "gradient", 720, 1280, seed=k) for k in range(128)]
    for k in range(0, 128, 4):   # local noise patches on the smooth frames
        y, x = rng.integers(0, 600), rng.integers(0, 1100)
        frames[k][y:y + 100, x:x + 150] = rng.integers(0, 256, (100, 150, 3), dtype=np.uint8)
    want = [pil_encode(a, quality, "4:2:0") for a in frames]
    for n in (1, 32, 128):
        assert _encode_all(frames[:n], quality, "4:2:0") == want[:n], n


def test_noise_at_q100_within_bound():
    from lanedetection_end2end_b200 import _capi
    from lanedetection_end2end_b200.jpeg import JpegEncoder
    for h, w, mode in [(720, 1280, "4:2:0"), (720, 1280, "4:4:4"), (17, 15, "4:4:4"), (256, 512, "gray")]:
        frames = torch.from_numpy(np.stack([frame("noise", h, w, mode, seed=s) for s in range(3)])).cuda()
        buf, offsets, lengths = JpegEncoder("cuda", quality=100, subsampling=subsampling_of(mode)).encode_async(frames)
        bound = _capi.lib().lf_jpeg_encode_bound(w, h, 1 if mode == "gray" else 3, 0 if mode == "4:4:4" else 2)
        assert buf.numel() == 3 * bound and offsets.tolist() == [0, bound, 2 * bound]
        assert 0 < int(lengths.max()) <= bound
        for n in range(3):
            d = bytes(buf[n * bound:n * bound + int(lengths[n])].cpu().numpy())
            assert d == pil_encode(frames[n].cpu().numpy(), 100, subsampling_of(mode))


def test_output_decodes_to_pillow():
    """The files decode through JpegDecoder to what Image.open(...).convert('RGB') gives."""
    from PIL import Image
    from lanedetection_end2end_b200.jpeg import JpegDecoder, JpegEncoder
    frames = torch.from_numpy(np.stack([content(k, 120, 200, seed=i) for i, k in enumerate(KINDS)])).cuda()
    for q, sub in [(75, "4:2:0"), (95, "4:4:4"), (20, "4:2:0")]:
        files = JpegEncoder("cuda", quality=q, subsampling=sub)(frames)
        got = JpegDecoder("cuda")(files).cpu().numpy()
        for n, d in enumerate(files):
            np.testing.assert_array_equal(got[n], np.asarray(Image.open(io.BytesIO(d)).convert("RGB")))


def test_encode_async_on_a_side_stream_and_graph():
    """encode_async orders on the current stream and captures into a CUDA graph (no synchronisation inside)."""
    from lanedetection_end2end_b200.jpeg import JpegEncoder
    a = np.stack([content("gradient", 64, 80, seed=1), content("noise", 64, 80, seed=2)])
    want = [pil_encode(x, 80, "4:2:0") for x in a]
    enc = JpegEncoder("cuda", quality=80)
    frames = torch.from_numpy(a).cuda()
    enc.encode_async(frames)                      # workspace allocated before capture
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            buf, offsets, lengths = enc.encode_async(frames)
        g.replay()
    torch.cuda.current_stream().wait_stream(side)
    for n in range(2):
        o, l = int(offsets[n]), int(lengths[n])
        assert bytes(buf[o:o + l].cpu().numpy()) == want[n]


def test_draw_lane_points_equals_restatement():
    from lanedetection_end2end_b200.inference import COLORMAP, draw_lane_points
    rng = np.random.default_rng(11)
    N, H, W, S = 6, 90, 160, 20
    for r in (0, 1, 3, 8, 16):
        for L in (1, 4, 5, 8):
            colors = [tuple(int(v) for v in rng.integers(0, 256, 3)) for _ in range(L)]
            base = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
            lanes = rng.integers(-20, W + 20, (N, L, S)).astype(np.int32)
            lanes[rng.random((N, L, S)) < 0.2] = -2
            lanes[:, :, 0] = lanes[:, :1, 0]          # one point shared by every lane
            lanes[0, 0, 1] = 2 ** 31 - 1
            lanes[0, 0, 2] = -2 ** 31
            h = rng.integers(-20, H + 20, (N, S)).astype(np.int32)
            got = draw_lane_points(torch.from_numpy(base).cuda(), torch.from_numpy(lanes).cuda(), torch.from_numpy(h).cuda(),
                                   colors, r).cpu().numpy()
            for n in range(N):
                want = jo.draw_lane_points(base[n].copy(), lanes[n], h[n], colors, r)
                np.testing.assert_array_equal(got[n], want, err_msg="r %d L %d n %d" % (r, L, n))
    assert COLORMAP[:4] == [(255, 0, 0), (0, 255, 0), (255, 255, 0), (0, 0, 255)]


def _golden_testset(tmp_path):
    g = np.load(os.path.join(GOLDEN, "render_testset.npz"))
    rows = [json.loads(line) for line in bytes(g["rows_json"]).decode().splitlines()]
    for k, row in enumerate(rows):
        p = tmp_path / "test" / row["raw_file"]
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(bytes(g["frame%d" % k]))
    return g, rows


@pytest.mark.parametrize("batch_size", [1, 2, 32])
def test_render_testset_equals_golden(tmp_path, batch_size):
    """The reference's overlays (cv2 + Pillow, tests/golden/render_testset.npz), including stamps clipped at every border."""
    from lanedetection_end2end_b200.inference import render_testset
    g, rows = _golden_testset(tmp_path)
    out = tmp_path / "out"
    paths = render_testset(torch.from_numpy(g["lanes"]).cuda(), rows, str(tmp_path / "test"), str(out), batch_size=batch_size)
    assert paths == [str(out / ("%d.jpg" % k)) for k in range(len(rows))]
    for k in range(len(rows)):
        assert (out / ("%d.jpg" % k)).read_bytes() == bytes(g["overlay%d" % k]), k


def test_render_testset_refuses_frames_by_name(tmp_path):
    from lanedetection_end2end_b200.inference import render_testset
    g, rows = _golden_testset(tmp_path)
    lanes = torch.from_numpy(g["lanes"]).cuda()
    bad = tmp_path / "test" / rows[1]["raw_file"]
    data = bytes(g["frame1"])
    bad.write_bytes(data[:2] + b"\xff\xc2" + data[4:])              # a progressive frame header
    with pytest.raises(ValueError, match=str(bad)):
        render_testset(lanes, rows, str(tmp_path / "test"), str(tmp_path / "out"))
    sos = data.index(b"\xff\xda")
    bad.write_bytes(data[:sos + 40] + b"\xff\xd9")                  # entropy-coded data cut short
    with pytest.raises(ValueError, match=str(bad)):
        render_testset(lanes, rows, str(tmp_path / "test"), str(tmp_path / "out"), batch_size=3)


def _host_overlay(path, lanes, h_samples):
    """The reference's drawing loop on the host: Pillow decode, cv2.circle per point, Pillow save."""
    import cv2
    from PIL import Image
    from lanedetection_end2end_b200.inference import COLORMAP
    with open(path, "rb") as f:
        img = np.array(Image.open(f).convert("RGB"))
    for l, lane in enumerate(lanes):
        for x, y in zip(lane, h_samples):
            if x != -2:
                img = cv2.circle(img, (int(x), int(y)), thickness=-1, color=COLORMAP[l], radius=3)
    bio = io.BytesIO()
    Image.fromarray(np.uint8(img)).save(bio, "JPEG")
    return bio.getvalue()


def test_test_model_render_dir(tmp_path, capsys):
    """test_model(..., render_dir=...) on a 40-image synthetic test set (batches 32, 8) with a random-weight --clas model:
    the overlays are drawn from the pass's own gated lanes and equal the host loop's files; render_dir=None writes none."""
    pytest.importorskip("cv2")
    from PIL import Image
    from oracle import inputs
    from oracle.make_render_golden import make_frame
    from lanedetection_end2end_b200 import inference
    from test_tusimple_gpu import _clas_model, _eager_host_path, _ground_truth
    N, B = 40, 32
    model, args = _clas_model(B)
    with torch.no_grad():        # every lane on and the horizon at the top, so the random-weight model's lanes are drawn
        model.line_classification.fully_connected_line1.bias.fill_(20.0)
        model.horizon_estimation.fully_connected_horizon.bias.fill_(-20.0)
    images = torch.from_numpy(inputs.make_images(N, 256, 512, seed=41))
    batches = [images[i:i + B] for i in range(0, N, B)]
    lanes = _eager_host_path(model, args, batches)
    assert sum(x != -2 for img in lanes for lane in img for x in lane) > 100
    rows = _ground_truth(lanes, 9)
    with open(tmp_path / "test_label.json", "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    pictures = [make_frame(k) for k in range(3)]
    for i, r in enumerate(rows):
        p = tmp_path / r["raw_file"]
        p.parent.mkdir(parents=True, exist_ok=True)
        a = pictures[i % 3]
        Image.fromarray(np.ascontiguousarray(a[:, ::-1]) if i % 2 else a).save(str(p), "JPEG", quality=85)
    args.test_dir = args.save_path = str(tmp_path)
    inference.test_model(batches, model, None, None, None, None, args)
    assert not (tmp_path / "render").exists()
    inference.test_model(batches, model, None, None, None, None, args, render_dir=str(tmp_path / "render"))
    capsys.readouterr()
    for i, r in enumerate(rows):
        got = (tmp_path / "render" / ("%d.jpg" % i)).read_bytes()
        assert got == _host_overlay(str(tmp_path / r["raw_file"]), lanes[i], r["h_samples"]), i
