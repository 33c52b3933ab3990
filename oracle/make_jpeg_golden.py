"""Golden fixture of the JPEG decoder, generated with Pillow itself (the reference's loader decodes with it):
`python -m oracle.make_jpeg_golden` -> tests/golden/jpeg_pil.npz.  TEST INFRASTRUCTURE.
For every case it stores the JPEG bytes Pillow encoded and Pillow's decode of them (Image.open(...).convert('RGB')): the
full array for small images, sha256 plus 8192 sampled bytes for full frames; and the Pillow / libjpeg-turbo versions."""
import hashlib
import io
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "jpeg_pil.npz")
FULL_ARRAY_MAX = 64 * 1024       # pixels * 3 up to this many bytes are stored whole

# name, H, W, mode, quality, subsampling (0 4:4:4, 1 4:2:2, 2 4:2:0), extra save options, seed
CASES = [
    ("q5_420", 96, 160, "RGB", 5, 2, {}, 1),
    ("q50_420", 96, 160, "RGB", 50, 2, {}, 2),
    ("q75_420", 96, 160, "RGB", 75, 2, {}, 3),
    ("q90_420", 96, 160, "RGB", 90, 2, {}, 4),
    ("q100_420", 96, 160, "RGB", 100, 2, {}, 5),
    ("q75_444", 96, 160, "RGB", 75, 0, {}, 6),
    ("q75_422", 96, 160, "RGB", 75, 1, {}, 7),
    ("q90_444", 64, 120, "RGB", 90, 0, {}, 8),
    ("q90_422", 64, 120, "RGB", 90, 1, {}, 9),
    ("gray_q75", 96, 160, "L", 75, None, {}, 10),
    ("gray_odd_61x97", 97, 61, "L", 85, None, {}, 11),
    ("rst_blocks_420", 96, 160, "RGB", 75, 2, {"restart_marker_blocks": 5}, 12),
    ("rst_rows_444", 96, 160, "RGB", 80, 0, {"restart_marker_rows": 1}, 13),
    ("rst_blocks_gray", 64, 72, "L", 60, None, {"restart_marker_blocks": 3}, 14),
    ("odd_61x97_420", 97, 61, "RGB", 85, 2, {}, 15),
    ("odd_61x97_422", 97, 61, "RGB", 85, 1, {}, 16),
    ("odd_17x1000_420", 1000, 17, "RGB", 70, 2, {}, 17),
    ("odd_1000x17_420", 17, 1000, "RGB", 70, 2, {}, 18),
    ("qt16bit_444", 48, 64, "RGB", None, 0, {"qtables": "16bit"}, 19),
    # chroma at most 2 samples wide: libjpeg replicates instead of the fancy filter
    ("narrow_3x20_422", 20, 3, "RGB", 80, 1, {}, 22),
    ("narrow_4x9_420", 9, 4, "RGB", 80, 2, {}, 23),
    ("narrow_2x13_420", 13, 2, "RGB", 90, 2, {}, 24),
    ("narrow_1x5_422", 5, 1, "RGB", 90, 1, {}, 25),
    ("narrow_5x7_420", 7, 5, "RGB", 85, 2, {}, 26),
    ("frame_q75_420", 720, 1280, "RGB", 75, 2, {}, 20),
    ("frame_q90_420_rst", 720, 1280, "RGB", 90, 2, {"restart_marker_rows": 2}, 21),
]


def make_frame(h, w, seed, mode="RGB"):
    """Smooth lane-like synthetic frame (dark road, bright slanted lane lines, sky gradient) with mild noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    t = yy / max(h - 1, 1)
    base = np.stack([60 + 120 * (1 - t) ** 2, 70 + 110 * (1 - t) ** 2, 80 + 150 * (1 - t) ** 2], -1)
    for k, x0 in enumerate((0.3, 0.5, 0.7)):
        cx = w * (x0 + (k - 1) * 0.35 * t)
        base += (150 * np.exp(-((xx - cx) / (2 + 6 * t)) ** 2) * (t > 0.4))[..., None]
    base += 20 * np.sin(xx / 23.0 + seed)[..., None] * np.cos(yy / 17.0)[..., None]
    img = np.clip(base + rng.normal(0, 4, base.shape), 0, 255).astype(np.uint8)
    return img.mean(-1).astype(np.uint8) if mode == "L" else img


def encode(case):
    from PIL import Image
    name, h, w, mode, q, sub, extra, seed = case
    im = Image.fromarray(make_frame(h, w, seed, mode), mode)
    kw = dict(extra)
    if kw.get("qtables") == "16bit":   # > 255 entries: 16-bit DQT, written as SOF1 (extended sequential)
        rng = np.random.default_rng(seed)
        kw["qtables"] = [list(rng.integers(1, 40, 64) * (k + 1)) for k in range(2)]
        kw["qtables"][0][1] = 300
    else:
        kw["quality"] = q
    if sub is not None:
        kw["subsampling"] = sub
    bio = io.BytesIO()
    im.save(bio, "JPEG", **kw)
    return bio.getvalue()


def pil_decode(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def main():
    import PIL
    from PIL import features
    out = {"pillow_version": PIL.__version__, "libjpeg_turbo_version": str(features.version("libjpeg_turbo"))}
    for case in CASES:
        name = case[0]
        data = encode(case)
        ref = pil_decode(data)
        out[name + "/jpeg"] = np.frombuffer(data, np.uint8)
        out[name + "/shape"] = np.array(ref.shape)
        out[name + "/sha256"] = hashlib.sha256(ref.tobytes()).hexdigest()
        if ref.size <= FULL_ARRAY_MAX:
            out[name + "/rgb"] = ref
        else:
            idx = np.random.default_rng(case[-1] + 100).integers(0, ref.size, 8192)
            out[name + "/idx"] = idx
            out[name + "/val"] = ref.reshape(-1)[idx]
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
