"""lf_png_decode (csrc/png.cu) through png.PngDecoder against Pillow's decode, and lf_label_preprocess through
input_pipeline.LabelPreprocessor against the reference loader's gt: the golden fixtures, a batch mixing encoders, a
live-Pillow width sweep, the full loader path, side-stream decoding and corrupt streams.  Every comparison is exact."""
import io
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle.make_png_golden import LOADER_CASES, LOADER_MAPS, lane_map, noise_map, write_png

pytestmark = pytest.mark.gpu

_G = np.load(os.path.join(GOLDEN, "png_labels.npz"))
NAMES = [str(n) for n in _G["names"]]


def _bytes(name):
    return bytes(_G[name + "/png"])


@pytest.mark.parametrize("name", NAMES)
def test_fixture_decodes_bit_exact(name):
    from lanedetection_end2end_b200.png import PngDecoder
    dec = PngDecoder("cuda")
    out = dec([_bytes(name)] * 2)
    want = _G[name + "/map"]
    assert out.dtype == torch.uint8 and tuple(out.shape) == (2,) + want.shape
    for n in range(2):
        np.testing.assert_array_equal(out[n].cpu().numpy(), want)
    dec.check()


def test_batch_mixing_encoders():
    """Pillow L at every level, OpenCV at two levels, fixed Huffman, forced filters, many IDATs: one batch"""
    from lanedetection_end2end_b200.png import PngDecoder
    names = ["pil_L1_frame", "pil_L6_frame", "pil_L9_frame", "cv2_frame", "cv2_c9_frame"]
    dec = PngDecoder("cuda")
    out = dec([_bytes(n) for n in names]).cpu().numpy()
    for k, n in enumerate(names):
        np.testing.assert_array_equal(out[k], _G[n + "/map"], err_msg=n)
    small = ["hand_fixed", "hand_filter0", "hand_filter3", "hand_filter4", "hand_many_idat", "hand_trns_text",
             "hand_trns_p8", "hand_filter_random_p4"]
    out = dec([_bytes(n) for n in small]).cpu().numpy()
    for k, n in enumerate(small):
        np.testing.assert_array_equal(out[k], _G[n + "/map"], err_msg=n)
    dec.check()


def test_live_pillow_width_sweep():
    """L and 4-bit P written by Pillow at every width 1..1280 (a few rows each, compress levels 1 and 9 in one batch)"""
    Image = pytest.importorskip("PIL.Image")
    from lanedetection_end2end_b200.png import PngDecoder
    dec = PngDecoder("cuda")
    rng = np.random.default_rng(3)
    for mode in ("L", "P"):
        for w in range(1, 1281):
            h = 2 + w % 5
            m = lane_map(h, w, w) * (1 if mode == "L" else 3) % 16
            m[:, ::3] = rng.integers(0, 16, m[:, ::3].shape)
            datas = []
            for lvl in (1, 9):
                im = Image.fromarray(m, mode)
                if mode == "P":
                    im.putpalette(list(range(48)))
                bio = io.BytesIO()
                im.save(bio, "PNG", compress_level=lvl)
                datas.append(bio.getvalue())
            out = dec(datas).cpu().numpy()
            for k, d in enumerate(datas):
                np.testing.assert_array_equal(out[k], np.array(Image.open(io.BytesIO(d)).convert("P")),
                                              err_msg="%s w=%d" % (mode, w))
    dec.check()


@pytest.mark.parametrize("name", LOADER_MAPS)
def test_png_to_label_preprocessor_equals_reference_loader(name):
    from lanedetection_end2end_b200.input_pipeline import LabelPreprocessor
    from lanedetection_end2end_b200.png import PngDecoder
    dec = PngDecoder("cuda")
    maps = dec([_bytes(name)] * 2)
    for r, nc, fl in LOADER_CASES:
        gt = LabelPreprocessor(r, nc)(maps, flip=[fl, 1 - fl])
        assert gt.dtype == torch.int64 and tuple(gt.shape) == (2, 1, r, 2 * r)
        want = _G["loader/%s/r%d_c%d_f%d" % (name, r, nc, fl)].astype(np.int64)
        other = _G["loader/%s/r%d_c%d_f%d" % (name, r, nc, 1 - fl)].astype(np.int64)
        np.testing.assert_array_equal(gt[0].cpu().numpy(), want, err_msg="r%d nc%d flip%d" % (r, nc, fl))
        np.testing.assert_array_equal(gt[1].cpu().numpy(), other, err_msg="r%d nc%d flip%d" % (r, nc, 1 - fl))
    dec.check()


@pytest.mark.parametrize("resize", [1, 77, 128, 333, 640])
def test_label_preprocessor_matches_oracle_at_other_sizes(resize):
    from lanedetection_end2end_b200.input_pipeline import LabelPreprocessor
    from oracle.png_oracle import label_transform
    m = lane_map(720, 1280, 9, nlanes=4)
    m[::11, ::13] = 200
    maps = torch.from_numpy(np.stack([m, m[:, ::-1].copy()])).cuda()
    for nc in (2, 4):
        gt = LabelPreprocessor(resize, nc)(maps, flip=torch.tensor([True, False])).cpu().numpy()
        np.testing.assert_array_equal(gt[0], label_transform(m, resize, nc, True))
        np.testing.assert_array_equal(gt[1], label_transform(m[:, ::-1], resize, nc, False))


def test_side_stream_decode_then_compute_stream():
    """JPEG frames and PNG maps decoded (and preprocessed) on a side stream, consumed on the compute stream"""
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor, LabelPreprocessor
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    from lanedetection_end2end_b200.png import PngDecoder
    gj = np.load(os.path.join(GOLDEN, "jpeg_pil.npz"))
    jpegs = [bytes(gj["frame_q75_420/jpeg"]), bytes(gj["frame_q90_420_rst/jpeg"])]
    pngs = [_bytes("pil_L6_frame"), _bytes("cv2_frame")]
    jd, pd, fp, lp = JpegDecoder("cuda"), PngDecoder("cuda"), FramePreprocessor(256), LabelPreprocessor(256, 4)
    flip = torch.tensor([False, True], device="cuda")
    x_ref, gt_ref = fp(jd(jpegs), flip=flip), lp(pd(pngs), flip=flip)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(20000000)           # keep the side stream busy so a missing wait would show
        x, gt = fp(jd(jpegs), flip=flip), lp(pd(pngs), flip=flip)
    torch.cuda.current_stream().wait_stream(side)
    x.record_stream(torch.cuda.current_stream())
    gt.record_stream(torch.cuda.current_stream())
    got_x, got_gt = x * 2, gt + 1                # consumed on the compute stream
    assert torch.equal(got_x, x_ref * 2) and torch.equal(got_gt, gt_ref + 1)
    np.testing.assert_array_equal(gt_ref[1].cpu().numpy(), _G["loader/cv2_frame/r256_c4_f1"].astype(np.int64))
    pd.check()
    jd.check()


def _replace_z(data, z):
    """the same PNG with its IDAT payloads replaced by one IDAT holding z"""
    out, i = data[:8], 8
    done = False
    while i < len(data):
        n, t = struct.unpack(">I4s", data[i:i + 8])
        if t == b"IDAT":
            if not done:
                out += struct.pack(">I", len(z)) + b"IDAT" + z + struct.pack(">I", zlib.crc32(b"IDAT" + z) & 0xFFFFFFFF)
                done = True
        else:
            out += data[i:i + 12 + n]
        i += 12 + n
    return out


def _corrupt_cases():
    from lanedetection_end2end_b200.png import parse
    good = _bytes("hand_filter_random")
    z = parse(good).zdata
    cases = {"truncated_idat": z[:len(z) // 2], "wrong_adler": z[:-1] + bytes([z[-1] ^ 0x55])}
    # damaged dynamic header: every code-length code length set to 7 (an incomplete code-length code)
    noisy = parse(_bytes("noise_geometric")).zdata
    bits = int.from_bytes(noisy[2:], "little")
    assert (bits >> 1) & 3 == 2                               # first block is dynamic
    for k in range(19):
        bits |= 7 << (17 + 3 * k)
    cases["damaged_dynamic_header"] = noisy[:2] + bits.to_bytes(len(noisy) - 2, "little")
    # distance too far back: a fixed block whose first symbol is a match (length 3, distance 1) with no output yet
    raw = b"".join(bytes([0]) + bytes(101) for _ in range(64))
    co = zlib.compressobj(6, zlib.DEFLATED, 15, 9, zlib.Z_FIXED)
    zf = co.compress(raw) + co.flush()
    assert (zf[2] >> 1) & 3 == 1
    # fixed block: header bits 1,01 then literal/length 257 (7-bit code 0000001) then distance code 0 (00000)
    stream = 1 | (1 << 1)
    pos = 3
    for b in (0, 0, 0, 0, 0, 0, 1):                             # Huffman codes are sent most significant bit first
        stream |= b << pos
        pos += 1
    pos += 5
    cases["distance_too_far"] = zf[:2] + stream.to_bytes(4, "little") + zf[-4:]
    return good, cases


@pytest.mark.parametrize("case", ["truncated_idat", "wrong_adler", "damaged_dynamic_header", "distance_too_far"])
def test_corrupt_stream_sets_status_and_check_raises(case):
    from lanedetection_end2end_b200.png import PngDecoder
    from oracle import png_oracle as po
    good, cases = _corrupt_cases()
    bad = _replace_z(good, cases[case])
    with pytest.raises(po.Corrupt):
        po.decode(bad)
    dec = PngDecoder("cuda")
    out = dec([good, bad, good])
    np.testing.assert_array_equal(out[0].cpu().numpy(), _G["hand_filter_random/map"])
    np.testing.assert_array_equal(out[2].cpu().numpy(), _G["hand_filter_random/map"])
    with pytest.raises(ValueError, match="corrupt"):
        dec.check()
    assert int(dec.status.item()) == 0                        # check() cleared the word
    dec([good])
    dec.check()


def test_filter_type_above_4_sets_status():
    from lanedetection_end2end_b200.png import PngDecoder
    m = noise_map(8, 9, 4)
    good = write_png(m, types=[1] * 8)
    raw = bytearray(b"".join(bytes([1]) + bytes(9) for _ in range(8)))
    raw[10 * 5] = 5                                            # row 5's filter type
    bad = _replace_z(good, zlib.compress(bytes(raw)))
    dec = PngDecoder("cuda")
    dec([bad])
    with pytest.raises(ValueError, match="corrupt"):
        dec.check()
    dec([good])
    dec.check()
