"""Golden fixture of the PNG label-map path: `python -m oracle.make_png_golden` -> tests/golden/png_labels.npz.
TEST INFRASTRUCTURE.

For every case it stores the PNG bytes and Pillow's decode of them (np.array(Image.open(f).convert('P'))): maps written
by Pillow (L at compress levels 0 / 1 / 6 / 9, P at 1 / 2 / 4 / 8 bits), by OpenCV (their bytes are kept, so cv2 is not
needed to read the fixture), and streams built here with zlib and struct (fixed-Huffman blocks, every filter type forced
on all rows, random filters per row, many IDAT chunks down to 1 byte, tRNS and text chunks, widths 1-37 at 1/2/4 bits,
1x1, noise maps whose dynamic codes reach long lengths).

It also stores the reference loader's `gt` for two full 1280x720 maps, flip on and off x nclasses 2 and 4 x resize 256 and
320.  Those come from running the reference's unmodified LaneDataset.__getitem__ on synthetic files in a temporary
directory (the object is made with object.__new__ and given the attributes the method reads; matplotlib is stubbed as
oracle/reference_import.py does).  The reference checkout is needed to regenerate the file, not to read it."""
import io
import os
import struct
import zlib

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "png_labels.npz")
LOADER_MAPS = ("pil_L6_frame", "cv2_frame")
LOADER_CASES = [(r, nc, fl) for r in (256, 320) for nc in (2, 4) for fl in (0, 1)]


def lane_map(h, w, seed, nlanes=4, width=15):
    """Synthetic label map: background 0, `nlanes` slanted lanes of `width` px labelled 1..nlanes in the lower part."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    m = np.zeros((h, w), np.uint8)
    t = yy / max(h - 1, 1)
    for k in range(nlanes):
        x0 = w * (0.2 + 0.6 * k / max(nlanes - 1, 1)) + rng.uniform(-0.05, 0.05) * w
        cx = w / 2 + (x0 - w / 2) * (0.1 + 0.9 * t)
        wid = np.maximum(1.0, width * (0.2 + 0.8 * t))
        m[(np.abs(xx - cx) < wid / 2) & (t > 0.3 + 0.05 * k)] = k + 1
    return m


def noise_map(h, w, seed, geometric=True):
    rng = np.random.default_rng(seed)
    if geometric:     # skewed symbol frequencies: long Huffman codes
        return np.minimum(rng.geometric(0.35, (h, w)) - 1, 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w), dtype=np.uint8)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(rows, types):
    """PNG-filter packed rows uint8 [H, rowbytes] with a 1-byte unit; types[y] in 0..4"""
    out, prev = [], np.zeros(rows.shape[1], np.int64)
    for y, ft in enumerate(types):
        x = rows[y].astype(np.int64)
        a = np.concatenate([[0], x[:-1]])
        c = np.concatenate([[0], prev[:-1]])
        pred = [0 * x, a, prev, (a + prev) >> 1, _paeth(a, prev, c)][ft]
        out.append(bytes([ft]) + ((x - pred) & 255).astype(np.uint8).tobytes())
        prev = x
    return b"".join(out)


def pack(m, depth):
    if depth == 8:
        return m
    ppb = 8 // depth
    h, w = m.shape
    padded = np.zeros((h, -(-w // ppb) * ppb), np.uint8)
    padded[:, :w] = m
    bits = (padded[..., None] >> np.arange(depth - 1, -1, -1, dtype=np.uint8)) & 1
    return np.packbits(bits.reshape(h, -1), axis=1)


def _chunk(ctype, data):
    return struct.pack(">I", len(data)) + ctype + data + struct.pack(">I", zlib.crc32(ctype + data) & 0xFFFFFFFF)


def write_png(m, depth=8, colour=0, types=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, idat_sizes=None, extra=()):
    """PNG of label map m built here: filters `types` (default None on every row), zlib at `level` / `strategy`, the
    stream cut into IDAT chunks of the cycling `idat_sizes`, `extra` chunks before the first IDAT."""
    h, w = m.shape
    rows = pack(m, depth)
    raw = filter_rows(rows, types if types is not None else [0] * h)
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    z = co.compress(raw) + co.flush()
    out = b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, colour, 0, 0, 0))
    if colour == 3:
        out += _chunk(b"PLTE", (np.arange(3 << depth) * 3 % 256).astype(np.uint8).tobytes())
    for ctype, data in extra:
        out += _chunk(ctype, data)
    sizes = idat_sizes or [len(z)]
    i = k = 0
    while i < len(z):
        n = sizes[k % len(sizes)]
        out += _chunk(b"IDAT", z[i:i + n])
        i, k = i + n, k + 1
    return out + _chunk(b"IEND", b"")


def pil_png(m, mode="L", ncolours=None, **kw):
    from PIL import Image
    im = Image.fromarray(m, "L")
    if mode == "P":
        im = Image.fromarray(m, "P")
        im.putpalette(list(np.arange(3 * ncolours) % 256))
    bio = io.BytesIO()
    im.save(bio, "PNG", **kw)
    return bio.getvalue()


def cv2_png(m, level=None):
    import cv2
    ok, buf = cv2.imencode(".png", m, [] if level is None else [cv2.IMWRITE_PNG_COMPRESSION, level])
    assert ok
    return buf.tobytes()


def cases():
    """name -> PNG bytes, built fresh (Pillow, OpenCV and zlib needed)"""
    rng = np.random.default_rng(123)
    c = {}
    c["pil_L0_stored"] = pil_png(lane_map(200, 360, 1), compress_level=0)     # > 65535 bytes: several stored blocks
    for lvl in (1, 6, 9):
        c["pil_L%d_frame" % lvl] = pil_png(lane_map(720, 1280, 10 + lvl), compress_level=lvl)
    for depth, ncol in ((1, 2), (2, 4), (4, 16), (8, 200)):
        m = lane_map(120, 203, 20 + depth, nlanes=min(ncol - 1, 6))
        m[::7, ::5] = (np.arange(m[::7, ::5].size).reshape(m[::7, ::5].shape) % ncol).astype(np.uint8)
        c["pil_P%d" % depth] = pil_png(m, "P", ncol)
    c["cv2_frame"] = cv2_png(lane_map(720, 1280, 30))
    c["cv2_c9_frame"] = cv2_png(lane_map(720, 1280, 31), 9)
    c["cv2_small"] = cv2_png(lane_map(90, 157, 32))
    small = lane_map(64, 101, 40)
    small[::3, ::2] = noise_map(22, 51, 41)
    c["hand_fixed"] = write_png(small, strategy=zlib.Z_FIXED)
    for ft in range(5):
        c["hand_filter%d" % ft] = write_png(small, types=[ft] * 64)
    c["hand_filter_random"] = write_png(small, types=list(rng.integers(0, 5, 64)))
    p4 = (lane_map(64, 101, 42, nlanes=6) * 2 + noise_map(64, 101, 43) % 2).astype(np.uint8) % 16
    c["hand_filter_random_p4"] = write_png(p4, depth=4, colour=3, types=list(rng.integers(0, 5, 64)))
    c["hand_many_idat"] = write_png(small, types=list(rng.integers(0, 5, 64)), idat_sizes=[1, 1, 7, 1, 100, 3])
    c["hand_trns_text"] = write_png(small, extra=[(b"tRNS", b"\x00\x03"), (b"tEXt", b"Comment\x00label map"),
                                                  (b"zTXt", b"Title\x00\x00" + zlib.compress(b"lanes"))])
    c["hand_trns_p8"] = write_png(small, depth=8, colour=3, extra=[(b"tRNS", bytes(range(0, 256, 3)))])
    for depth in (1, 2, 4):
        for w in range(1, 38):
            m = noise_map(3 + w % 4, w, 100 * depth + w, geometric=False) % (1 << depth)
            c["w%d_p%d" % (w, depth)] = write_png(m, depth=depth, colour=3, types=list(rng.integers(0, 5, m.shape[0])))
    c["one_L"] = write_png(np.array([[7]], np.uint8))
    c["one_P1"] = write_png(np.array([[1]], np.uint8), depth=1, colour=3)
    c["noise_geometric"] = pil_png(noise_map(97, 131, 50), compress_level=9)
    c["noise_uniform"] = write_png(noise_map(64, 64, 51, geometric=False), types=list(rng.integers(0, 5, 64)), level=9)
    return c


def pil_decode(data):
    from PIL import Image
    return np.array(Image.open(io.BytesIO(data)).convert("P"))


def _seed_for(flip):
    """a seed whose first np.random.uniform decides the reference's flip as wanted"""
    s = 0
    while True:
        np.random.seed(s)
        if (np.random.uniform(0.0, 1.0) > 0.5) == bool(flip):
            return s
        s += 1


def reference_gt(png_bytes, cases_):
    """the reference loader's gt for one 720x1280 map: {(resize, nclasses, flip): uint8 [1, resize, 2 resize]}"""
    import importlib.util
    import sys
    import tempfile
    from PIL import Image
    from oracle import reference_import
    reference_import._stub_matplotlib()
    if not hasattr(np, "RankWarning"):
        np.RankWarning = np.exceptions.RankWarning
    path = os.path.join(reference_import.SOURCE_ROOT, "Backprojection_Loss", "Dataloader", "Load_Data_new.py")
    spec = importlib.util.spec_from_file_location("_ref_load_data_new", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    from torchvision import transforms
    out = {}
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "img"))
        os.makedirs(os.path.join(d, "gt"))
        Image.fromarray(np.full((720, 1280, 3), 90, np.uint8)).save(os.path.join(d, "img", "1.jpg"))
        with open(os.path.join(d, "gt", "1.png"), "wb") as f:
            f.write(png_bytes)
        hs = list(range(160, 720, 10))
        lanes = [[-2] * 20 + [300 + 200 * k + 2 * j for j in range(36)] for k in range(4)]
        for resize, nclasses, flip in cases_:
            ds = object.__new__(mod.LaneDataset)
            ds.image_dir, ds.gt_dir = os.path.join(d, "img"), os.path.join(d, "gt")
            ds.rgb_lst, ds.gt_lst = ["1.jpg"], ["1.png"]
            ds.ordered_lanes = [{"lanes": lanes, "h_samples": hs}]
            ds.line_file = [{"lines": [0, 1, 1, 0, 1, 0, 1, 1]}]
            ds.valid_idx, ds.flip_on, ds.resize, ds.nclasses = [], bool(flip), resize, nclasses
            ds.totensor = transforms.ToTensor()
            np.random.seed(_seed_for(flip) if flip else 0)
            gt = ds[0][1]
            assert gt.dtype.is_floating_point is False and gt.shape == (1, resize, 2 * resize)
            assert int(gt.max()) < 256 and int(gt.min()) >= 0
            out[(resize, nclasses, flip)] = gt.numpy().astype(np.uint8)
    return out


def main():
    import PIL
    c = cases()
    out = {"pillow_version": PIL.__version__, "names": np.array(sorted(c))}
    for name in sorted(c):
        out[name + "/png"] = np.frombuffer(c[name], np.uint8)
        out[name + "/map"] = pil_decode(c[name])
    for name in LOADER_MAPS:
        for (r, nc, fl), gt in reference_gt(c[name], LOADER_CASES).items():
            out["loader/%s/r%d_c%d_f%d" % (name, r, nc, fl)] = gt
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
