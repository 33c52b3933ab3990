"""The JPEG encoder's numpy restatement (oracle/jpeg_enc_oracle.py) against Pillow's encoder byte for byte, the circle
restatement against cv2.circle, the render fixture against the restatement, and the C ABI's argument checks (host-side,
no device needed)."""
import ctypes
import io
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import jpeg_enc_oracle as jo

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 65), (256, 512)]
QUALITIES = [1, 10, 50, 75, 90, 95, 100]
MODES = ["4:2:0", "4:4:4", "gray"]


def content(kind, h, w, seed=0):
    """uint8 [h, w, 3] test frames: noise, smooth gradients, flat (EOB-only blocks), sparse detail on flat (ZRL runs),
    saturated black / white checks (largest DC differences and AC categories)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        return np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), (x + 2 * y) * 3 % 256], -1).astype(np.uint8)
    if kind == "flat":
        return np.broadcast_to(np.array([37, 200, 90], np.uint8), (h, w, 3)).copy()
    if kind == "sparse":
        a = np.full((h, w, 3), 128, np.uint8)
        a[(x % 8 == 7) & (y % 8 == 7)] = 255
        return a
    if kind == "saturated":
        return np.where((((x // 8) + (y // 8)) % 2 == 0)[..., None] ^ (rng.random((h, w, 1)) < 0.05), 255, 0).astype(np.uint8) \
            * np.ones(3, np.uint8)
    raise ValueError(kind)


KINDS = ["noise", "gradient", "flat", "sparse", "saturated"]


def pil_encode(a, quality, subsampling):
    from PIL import Image
    bio = io.BytesIO()
    Image.fromarray(a).save(bio, "JPEG", quality=quality, subsampling=subsampling)
    return bio.getvalue()


def frame(kind, h, w, mode, seed=0):
    a = content(kind, h, w, seed)
    return np.ascontiguousarray(a[..., 1]) if mode == "gray" else a


def subsampling_of(mode):
    return "4:2:0" if mode == "gray" else mode


@pytest.mark.parametrize("size", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_oracle_equals_pillow(size):
    pytest.importorskip("PIL.Image")
    h, w = size
    for kind in KINDS:
        for mode in MODES:
            a = frame(kind, h, w, mode, seed=h * 1000 + w)
            for q in QUALITIES:
                sub = subsampling_of(mode)
                assert jo.encode(a, q, sub) == pil_encode(a, q, sub), (kind, mode, q)


def test_oracle_equals_pillow_720p():
    pytest.importorskip("PIL.Image")
    for q, kind, mode in [(100, "noise", "4:2:0"), (1, "noise", "4:4:4"), (75, "gradient", "4:2:0"), (95, "saturated", "4:2:0"),
                          (50, "sparse", "gray"), (90, "flat", "4:4:4"), (10, "gradient", "gray")]:
        a = frame(kind, 720, 1280, mode, seed=q)
        assert jo.encode(a, q, subsampling_of(mode)) == pil_encode(a, q, subsampling_of(mode)), (q, kind, mode)


def test_grayscale_4_4_4_header():
    """A grayscale frame under 4:4:4 records 1x1 sampling, as Pillow's does; the scan is the same as under 4:2:0."""
    pytest.importorskip("PIL.Image")
    a = frame("gradient", 33, 65, "gray")
    assert jo.encode(a, 75, "4:4:4") == pil_encode(a, 75, "4:4:4")


def _segments(data):
    out, i = [], 2
    while True:
        m, ln = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        out.append((m, ln))
        if m == 0xDA:
            return out
        i += 2 + ln


def test_header_segments():
    assert _segments(jo.encode(content("noise", 9, 7), 75)) == [(0xE0, 16), (0xDB, 67), (0xDB, 67), (0xC0, 17), (0xC4, 31),
                                                                 (0xC4, 181), (0xC4, 31), (0xC4, 181), (0xDA, 12)]
    assert _segments(jo.encode(content("noise", 9, 7)[..., 0].copy(), 75)) == [(0xE0, 16), (0xDB, 67), (0xC0, 11), (0xC4, 31),
                                                                               (0xC4, 181), (0xDA, 8)]


def _lib():
    from lanedetection_end2end_b200 import _capi
    try:
        return _capi.lib()
    except _capi.LanefitError as e:
        pytest.skip(str(e))


def test_quality_tables_equal_oracle():
    lib = _lib()
    for ncomp in (1, 3):
        for q in range(1, 101):
            got = np.zeros((2, 64), np.uint16)
            assert lib.lf_jpeg_quality_tables(q, ncomp, got.ctypes.data) == 0
            want = jo.quality_tables(q, ncomp)
            np.testing.assert_array_equal(got[:len(want)], want, err_msg="q%d ncomp %d" % (q, ncomp))


def test_bound_covers_worst_case_and_refuses_bad_shapes():
    """The bound is the headers, every block at its longest code (22 + 63 * 26 bits, rounded up to 208 bytes) with every
    byte stuffed, and EOI; a noise frame at quality 100 stays well inside it."""
    lib = _lib()
    a = content("noise", 64, 48)
    n = len(jo.encode(a, 100, "4:4:4"))
    blocks = 8 * 6 * 3
    assert lib.lf_jpeg_encode_bound(48, 64, 3, 0) == 623 + 2 * (blocks * 208 + 1) + 2 > n
    for args in [(0, 8, 3, 2), (8, 0, 3, 2), (65536, 8, 3, 2), (8, 8, 2, 2), (8, 8, 3, 1), (8, 8, 3, 3)]:
        assert lib.lf_jpeg_encode_bound(*args) == 0, args
        assert lib.lf_jpeg_encode_workspace_bytes(1, *args) == 0, args
    assert lib.lf_jpeg_encode_workspace_bytes(0, 8, 8, 3, 2) == 0


def test_c_abi_refuses_bad_arguments():
    """Refusals happen on the host before any launch: quality, shapes, tables, capacity, null pointers, draw limits."""
    lib = _lib()
    qt = np.zeros((2, 64), np.uint16)
    for q in (0, -5, 101):
        assert lib.lf_jpeg_quality_tables(q, 3, qt.ctypes.data) == -1
    assert lib.lf_jpeg_quality_tables(75, 2, qt.ctypes.data) == -1
    assert lib.lf_jpeg_quality_tables(75, 3, None) == -1
    lib.lf_jpeg_quality_tables(75, 3, qt.ctypes.data)
    fake = ctypes.c_void_p(16)       # never dereferenced: every call below is refused first
    cap = lib.lf_jpeg_encode_bound(16, 16, 3, 2)
    ok = lambda **kw: dict(dict(frames=fake, N=1, W=16, H=16, ncomp=3, sampling=2, qt=qt.ctypes.data, out=fake, cap=cap,
                                out_len=fake, ws=fake), **kw)
    enc = lambda d: lib.lf_jpeg_encode(d["frames"], d["N"], d["W"], d["H"], d["ncomp"], d["sampling"], d["qt"], d["out"],
                                       d["cap"], d["out_len"], d["ws"], None)
    for bad in [dict(N=0), dict(W=0), dict(H=70000), dict(ncomp=4), dict(sampling=1), dict(cap=cap - 1), dict(frames=None),
                dict(out=None), dict(out_len=None), dict(ws=None), dict(qt=None)]:
        assert enc(ok(**bad)) == -1, bad
    zero = qt.copy()
    zero[1, 5] = 0
    assert enc(ok(qt=zero.ctypes.data)) == -1
    big = qt.copy()
    big[0, 0] = 256
    assert enc(ok(qt=big.ctypes.data)) == -1
    rgb = np.zeros((4, 3), np.uint8)
    draw = lambda N=1, L=4, S=56, radius=3, colors=rgb.ctypes.data: lib.lf_draw_lane_points(fake, N, 720, 1280, fake, L, S, fake,
                                                                                           colors, radius, None)
    for bad in [dict(N=0), dict(L=0), dict(L=9), dict(S=65), dict(radius=-1), dict(radius=17), dict(colors=None)]:
        assert draw(**bad) == -1, bad


def test_encoder_refuses_bad_settings():
    from lanedetection_end2end_b200.jpeg import JpegEncoder
    _lib()
    for kw in [dict(quality=0), dict(quality=101), dict(quality=7.5), dict(quality=True), dict(subsampling="4:2:2"),
               dict(subsampling=2)]:
        with pytest.raises(ValueError):
            JpegEncoder("cpu", **kw)
    with pytest.raises(ValueError):
        jo.quality_tables(0)


def _cv2_draw(img, lanes, h_samples, colors, radius):
    import cv2
    for l, lane in enumerate(lanes):
        for x, y in zip(lane, h_samples):
            if x != -2:
                img = cv2.circle(img, (int(x), int(y)), radius=radius, color=colors[l], thickness=-1)
    return img


def test_circle_stamp_equals_cv2():
    """circle_halfwidths / draw_lane_points against cv2.circle(..., thickness=-1) for radius 0-8 at interior, edge and
    corner centres (and centres just outside the frame), one point at a time."""
    pytest.importorskip("cv2")
    H, W = 23, 31
    centres = [(15, 11), (0, 11), (30, 11), (15, 0), (15, 22), (0, 0), (30, 0), (0, 22), (30, 22), (1, 1), (-2, 5), (33, 20),
               (10, -3), (12, 24)]
    assert sum(2 * h + 1 for h in jo.circle_halfwidths(3)[1:]) * 2 + 2 * 3 + 1 == 29   # the reference's radius-3 stamp
    for r in range(9):
        for cx, cy in centres:
            want = _cv2_draw(np.zeros((H, W, 3), np.uint8), [[cx]], [cy], [(255, 0, 0)], r)
            got = jo.draw_lane_points(np.zeros((H, W, 3), np.uint8), [[cx]], [cy], [(255, 0, 0)], r)
            np.testing.assert_array_equal(got, want, err_msg="r %d centre %s" % (r, (cx, cy)))


def test_overlapping_lanes_equal_cv2():
    """Several lanes whose stamps overlap, with gaps (-2) and points on and past the borders: the last stamp wins."""
    pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    H, W, S = 40, 50, 12
    colors = [(255, 0, 0), (0, 255, 0), (255, 255, 0), (0, 0, 255), (0, 128, 128)]
    for trial in range(40):
        L = int(rng.integers(1, 6))
        h = rng.integers(-4, H + 4, S)
        lanes = rng.integers(-5, W + 5, (L, S))
        lanes[rng.random((L, S)) < 0.2] = -2
        lanes[:, 0] = lanes[0, 0]             # the same point in every lane
        r = int(rng.integers(0, 9))
        base = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        want = _cv2_draw(base.copy(), lanes.tolist(), h.tolist(), colors, r)
        got = jo.draw_lane_points(base.copy(), lanes, h, colors, r)
        np.testing.assert_array_equal(got, want, err_msg="trial %d" % trial)


def test_render_fixture_equals_restatement():
    """The golden overlays (the reference's own drawing lines: Pillow decode, cv2.circle, Pillow save) equal Pillow decode +
    the circle restatement + the encoder restatement."""
    pytest.importorskip("PIL.Image")
    from PIL import Image
    from lanedetection_end2end_b200.inference import COLORMAP
    g = np.load(os.path.join(GOLDEN, "render_testset.npz"))
    rows = [json.loads(line) for line in bytes(g["rows_json"]).decode().splitlines()]
    assert len(rows) == g["lanes"].shape[0] >= 3
    for k, row in enumerate(rows):
        img = np.array(Image.open(io.BytesIO(bytes(g["frame%d" % k]))).convert("RGB"))
        np.testing.assert_array_equal(g["h_samples"][k], row["h_samples"])
        jo.draw_lane_points(img, g["lanes"][k], g["h_samples"][k], COLORMAP[:4], 3)
        assert jo.encode(img, 75, "4:2:0") == bytes(g["overlay%d" % k]), k
