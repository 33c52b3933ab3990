"""lf_jpeg_decode (csrc/jpeg.cu) through jpeg.JpegDecoder against Pillow's decode: the golden fixtures, a mixed restart /
no-restart batch, a live-Pillow sweep, the full loader path into FramePreprocessor, corrupt data and a side stream.
Every comparison is exact."""
import io
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.make_jpeg_golden import CASES, make_frame

pytestmark = pytest.mark.gpu


def _golden():
    return np.load(os.path.join(GOLDEN, "jpeg_pil.npz"))


def _check(name, got, g):
    import hashlib
    if name + "/rgb" in g:
        np.testing.assert_array_equal(got, g[name + "/rgb"])
    else:
        np.testing.assert_array_equal(got.reshape(-1)[g[name + "/idx"]], g[name + "/val"])
    assert hashlib.sha256(got.tobytes()).hexdigest() == str(g[name + "/sha256"])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fixture_decodes_bit_exact(case):
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    g = _golden()
    dec = JpegDecoder("cuda")
    out = dec([bytes(g[case[0] + "/jpeg"])] * 2)
    assert out.dtype == torch.uint8 and tuple(out.shape) == (2,) + tuple(g[case[0] + "/shape"])
    for n in range(2):
        _check(case[0], out[n].cpu().numpy(), g)
    dec.check()


def _encode(a, mode="RGB", **kw):
    from PIL import Image
    bio = io.BytesIO()
    Image.fromarray(a, mode).save(bio, "JPEG", **kw)
    return bio.getvalue()


def _pil(d):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(d)).convert("RGB"))


def test_mixed_restart_batch():
    pytest.importorskip("PIL.Image")
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    datas = [_encode(make_frame(120, 200, s), quality=q, subsampling=sub, **kw) for s, (q, sub, kw) in enumerate(
        [(75, 2, {}), (90, 2, {"restart_marker_blocks": 7}), (60, 0, {"restart_marker_rows": 1}), (95, 1, {}),
         (80, 2, {"restart_marker_rows": 3})])]
    datas.append(_encode(make_frame(120, 200, 9, "L"), "L", quality=70, restart_marker_blocks=4))
    dec = JpegDecoder("cuda")
    out = dec(datas).cpu().numpy()
    for n, d in enumerate(datas):
        np.testing.assert_array_equal(out[n], _pil(d))
    dec.check()


def test_live_pillow_sweep():
    pytest.importorskip("PIL.Image")
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    dec = JpegDecoder("cuda")
    rng = np.random.default_rng(7)
    for h, w in ((5, 1), (9, 2), (3, 3), (17, 4), (8, 8), (9, 33), (45, 77), (130, 71), (256, 384), (720, 1280)):
        datas = []
        for s in range(4):
            q = int(rng.choice([5, 30, 50, 75, 90, 97, 100]))
            sub = int(rng.integers(0, 3))
            kw = {"restart_marker_blocks": int(rng.integers(1, 9))} if s == 3 else {}
            datas.append(_encode(make_frame(h, w, int(rng.integers(1 << 20))), quality=q, subsampling=sub, **kw))
        out = dec(datas).cpu().numpy()
        for n, d in enumerate(datas):
            np.testing.assert_array_equal(out[n], _pil(d), err_msg="%dx%d #%d" % (h, w, n))
    dec.check()


@pytest.mark.parametrize("layout", ["nchw", "nhwc4"])
def test_jpeg_to_preprocessor_equals_reference_loader(layout):
    Image = pytest.importorskip("PIL.Image")
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    datas = [_encode(make_frame(720, 1280, 30 + s), quality=80, subsampling=2) for s in range(3)]
    flip = [False, True, False]
    x = FramePreprocessor(256)(JpegDecoder("cuda")(datas), flip=flip, layout=layout)
    if layout == "nhwc4":
        x = x[..., :3].permute(0, 3, 1, 2)
    for n, d in enumerate(datas):
        im = Image.open(io.BytesIO(d)).convert("RGB").crop((0, 80, 1280, 720)).resize((512, 256), Image.BILINEAR)
        if flip[n]:
            im = im.transpose(Image.FLIP_LEFT_RIGHT)
        want = np.transpose(np.asarray(im).astype(np.float32) / np.float32(255), (2, 0, 1))
        np.testing.assert_array_equal(x[n].cpu().numpy(), want)


def test_truncated_scan_sets_status_and_check_raises():
    from lanedetection_end2end_b200.jpeg import JpegDecoder, parse
    g = _golden()
    good = bytes(g["q90_420/jpeg"])
    h = parse(good)
    cut = good[:h.ecs_off + h.ecs_len // 2]
    dec = JpegDecoder("cuda")
    dec([good, cut])
    with pytest.raises(ValueError, match="corrupt"):
        dec.check()
    dec([good])           # check() cleared the word
    dec.check()


def test_side_stream_decode_then_compute_stream():
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    g = _golden()
    datas = [bytes(g["frame_q75_420/jpeg"]), bytes(g["frame_q90_420_rst/jpeg"])]
    dec, pre = JpegDecoder("cuda"), FramePreprocessor(256)
    ref = pre(dec(datas))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(20000000)           # keep the side stream busy so a missing wait would show
        frames = dec(datas)
    torch.cuda.current_stream().wait_stream(side)
    frames.record_stream(torch.cuda.current_stream())
    got = pre(frames)
    del frames
    assert torch.equal(got, ref)
    _check("frame_q75_420", dec(datas)[0].cpu().numpy(), g)
    dec.check()


@pytest.mark.parametrize("sub", [0, 1, 2])
def test_narrow_widths_bit_exact(sub):
    """widths 1..5 in every sampling: chroma 1..2 samples wide is replicated, not fancy-filtered (as libjpeg does)"""
    pytest.importorskip("PIL.Image")
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    dec = JpegDecoder("cuda")
    rng = np.random.default_rng(50 + sub)
    for w in (1, 2, 3, 4, 5):
        for h in (1, 2, 3, 7, 17):
            datas = [_encode(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), quality=q, subsampling=sub) for q in (60, 95)]
            out = dec(datas).cpu().numpy()
            for n, d in enumerate(datas):
                np.testing.assert_array_equal(out[n], _pil(d), err_msg="%dx%d q#%d" % (w, h, n))
    dec.check()


def test_check_waits_for_a_side_stream_decode():
    """check() on the compute stream sees the status of a decode still running on a side stream, and the next decode
    (on that side stream) starts after check() cleared the word"""
    from lanedetection_end2end_b200.jpeg import JpegDecoder, parse
    g = _golden()
    good = bytes(g["q90_420/jpeg"])
    h = parse(good)
    cut = good[:h.ecs_off + h.ecs_len // 2]
    dec = JpegDecoder("cuda")
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50000000)
        dec([good, cut])
    with pytest.raises(ValueError, match="corrupt"):
        dec.check()                       # the compute stream never waited for `side` itself
    with torch.cuda.stream(side):
        dec([good])
    dec.check()
    with torch.cuda.stream(side):
        dec([cut])
    with pytest.raises(ValueError, match="corrupt"):
        dec.check()
