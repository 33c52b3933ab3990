"""PNG label maps without a GPU: the chunk parser against Pillow's header, every rejection, the numpy / Python
restatement (oracle/png_oracle.py) against zlib, Pillow and the golden arrays (tests/golden/png_labels.npz), its label
transform against the reference loader's golden gt tensors, the NEAREST index tables against Pillow, and the C ABI
(LfPngImage layout, prototypes, exports)."""
import ctypes
import io
import os
import re
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import png_oracle as po
from oracle.make_png_golden import LOADER_CASES, LOADER_MAPS, lane_map, write_png
from lanedetection_end2end_b200 import png
from lanedetection_end2end_b200.input_pipeline import nearest_table

_G = np.load(os.path.join(GOLDEN, "png_labels.npz"))
NAMES = [str(n) for n in _G["names"]]
FAST = [n for n in NAMES if not n.endswith("_frame")]


def _bytes(name):
    return bytes(_G[name + "/png"])


@pytest.mark.parametrize("name", NAMES)
def test_parser_agrees_with_pillow(name):
    Image = pytest.importorskip("PIL.Image")
    data = _bytes(name)
    h = png.parse(data)
    im = Image.open(io.BytesIO(data))
    assert (h.width, h.height) == im.size
    assert im.mode == ("L" if h.colour == 0 else "P")
    assert zlib.decompress(h.zdata)          # the joined IDAT payloads are one complete zlib stream


@pytest.mark.parametrize("name", FAST)
def test_oracle_reproduces_golden(name):
    data = _bytes(name)
    h = png.parse(data)
    rowbytes = (h.width * h.depth + 7) // 8
    raw, _ = po.inflate(h.zdata, h.height * (rowbytes + 1))
    assert raw == zlib.decompress(h.zdata)
    got, _ = po.decode(data)
    np.testing.assert_array_equal(got, _G[name + "/map"])


@pytest.mark.parametrize("name", ["pil_L1_frame", "cv2_c9_frame"])
def test_oracle_reproduces_golden_full_frame(name):
    got, _ = po.decode(_bytes(name))
    np.testing.assert_array_equal(got, _G[name + "/map"])


def test_fixtures_cover_the_block_types_and_filters():
    seen = {"stored": 0, "fixed": 0, "dynamic": 0}
    filters = set()
    for name in ("pil_L0_stored", "hand_fixed", "noise_geometric", "hand_filter_random", "pil_L6_frame"):
        _, st = po.decode(_bytes(name))
        for k in seen:
            seen[k] += st[k]
        filters |= set(st["filters"])
    assert po.inflate(png.parse(_bytes("pil_L0_stored")).zdata, 200 * 361)[1]["stored"] >= 2
    assert all(seen.values()) and filters == {0, 1, 2, 3, 4}
    h = png.parse(_bytes("noise_geometric"))
    assert max(_code_lengths(h.zdata)) >= 10            # codes longer than the device's 9-bit lookahead


def _code_lengths(z):
    """literal/length code lengths of the first (dynamic) block"""
    br = po._Bits(z, 2)
    assert br.get(1) in (0, 1) and br.get(2) == 2
    hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
    cl = [0] * 19
    for k in range(hclen):
        cl[po.CLEN_ORDER[k]] = br.get(3)
    code, lens = po._code(cl, False), []
    while len(lens) < hlit:
        s = po._decode(br, code)
        if s < 16:
            lens.append(s)
        else:
            rep = 3 + br.get(2) if s == 16 else (3 + br.get(3) if s == 17 else 11 + br.get(7))
            lens += [lens[-1] if s == 16 else 0] * rep
    return lens[:hlit]


@pytest.mark.parametrize("name", LOADER_MAPS)
def test_oracle_label_transform_matches_reference_loader(name):
    m = _G[name + "/map"]
    for r, nc, fl in LOADER_CASES:
        want = _G["loader/%s/r%d_c%d_f%d" % (name, r, nc, fl)]
        np.testing.assert_array_equal(po.label_transform(m, r, nc, fl), want, err_msg="r%d nc%d flip%d" % (r, nc, fl))


def test_flip_quirk_restores_classes_3_and_4():
    """the reference's masks of 3 and 4 are taken before the flip: a flipped nclasses=2 sample carries 3 and 4 again"""
    g = _G["loader/cv2_frame/r256_c2_f1"]
    assert {3, 4} <= set(np.unique(g).tolist())
    assert not {3, 4} & set(np.unique(_G["loader/cv2_frame/r256_c2_f0"]).tolist())


def test_nearest_tables_match_pillow():
    """every output size 1..1280 of the 1280-wide and 640-tall crops (and upsampling), against Pillow's NEAREST resize
    of an index image"""
    Image = pytest.importorskip("PIL.Image")
    for n_in in (1280, 640):
        col = Image.fromarray(np.arange(n_in, dtype=np.int32)[None], "I")
        for n_out in list(range(1, n_in + 1)) + [n_in + 7, 2 * n_in + 1]:
            got = np.array(col.resize((n_out, 1), Image.NEAREST))[0]
            np.testing.assert_array_equal(nearest_table(n_in, n_out), got, err_msg="%d -> %d" % (n_in, n_out))


@pytest.mark.parametrize("resize", [64, 100, 256, 320, 333])
def test_oracle_label_transform_matches_pillow_resize(resize):
    Image = pytest.importorskip("PIL.Image")
    m = lane_map(720, 1280, 5)
    want = np.array(Image.fromarray(m, "P").crop((0, 80, 1280, 720)).resize((2 * resize, resize), Image.NEAREST))
    np.testing.assert_array_equal(po.label_transform(m, resize, 4, False)[0], want)


# ---- rejections ------------------------------------------------------------------------------------------------------
def _ihdr(data, **kw):
    """rewrite IHDR fields (width, height, depth, colour, comp, filt, interlace) of a PNG, fixing the CRC"""
    fields = dict(zip(("width", "height", "depth", "colour", "comp", "filt", "interlace"), struct.unpack(">IIBBBBB", data[16:29])))
    fields.update(kw)
    body = struct.pack(">IIBBBBB", *fields.values())
    return data[:16] + body + struct.pack(">I", zlib.crc32(b"IHDR" + body) & 0xFFFFFFFF) + data[33:]


def _pil(mode, **kw):
    Image = pytest.importorskip("PIL.Image")
    a = lane_map(16, 24, 3)
    im = Image.fromarray(np.stack([a] * 4, -1)[..., :{"RGB": 3, "RGBA": 4, "LA": 2}.get(mode, 1)].squeeze(), mode)
    bio = io.BytesIO()
    im.save(bio, "PNG", **kw)
    return bio.getvalue()


@pytest.mark.parametrize("mode,msg", [("RGB", "colour type 2"), ("LA", "colour type 4"), ("RGBA", "colour type 6")])
def test_rejects_colour_types(mode, msg):
    with pytest.raises(ValueError, match=msg):
        png.parse(_pil(mode))


def test_rejects_interlace_16bit_low_gray_and_methods():
    base = _bytes("hand_filter2")
    with pytest.raises(ValueError, match="Adam7"):
        png.parse(_ihdr(base, interlace=1))
    with pytest.raises(ValueError, match="16-bit"):
        png.parse(_ihdr(base, depth=16))
    with pytest.raises(ValueError, match="4-bit grayscale"):
        png.parse(_ihdr(base, depth=4))
    with pytest.raises(ValueError, match="compression method 1"):
        png.parse(_ihdr(base, comp=1))
    with pytest.raises(ValueError, match="filter method 1"):
        png.parse(_ihdr(base, filt=1))
    with pytest.raises(ValueError, match="bad IHDR"):
        png.parse(_ihdr(base, colour=3, depth=16))
    with pytest.raises(ValueError, match="bad IHDR"):
        png.parse(_ihdr(base, width=0))


def test_rejects_a_pillow_16bit_file():
    Image = pytest.importorskip("PIL.Image")
    bio = io.BytesIO()
    Image.fromarray(lane_map(16, 24, 3).astype(np.uint16) * 1000).save(bio, "PNG")
    with pytest.raises(ValueError, match="16-bit"):
        png.parse(bio.getvalue())


def test_rejects_zlib_header_problems():
    m = lane_map(8, 9, 1)
    good = write_png(m)
    z = png.parse(good).zdata

    def with_z(z2):
        i = good.index(b"IDAT") - 4
        n = struct.unpack(">I", good[i:i + 4])[0]
        return good[:i] + struct.pack(">I", len(z2)) + b"IDAT" + z2 + struct.pack(">I", zlib.crc32(b"IDAT" + z2)) + good[i + 12 + n:]
    png.parse(with_z(z))
    d = zlib.compressobj(6, zlib.DEFLATED, 15, 9, zlib.Z_DEFAULT_STRATEGY, zdict=b"\x00" * 64)
    with pytest.raises(ValueError, match="preset dictionary"):
        png.parse(with_z(d.compress(b"\x00" * 90) + d.flush()))
    with pytest.raises(ValueError, match="zlib compression method"):
        png.parse(with_z(bytes([z[0] & 0xF0 | 7]) + z[1:]))
    with pytest.raises(ValueError, match="bad zlib header"):
        png.parse(with_z(bytes([z[0], z[1] ^ 1]) + z[2:]))


def test_rejects_signature_missing_idat_and_truncation():
    good = _bytes("hand_filter1")
    with pytest.raises(ValueError, match="signature"):
        png.parse(b"\x89PNX" + good[4:])
    with pytest.raises(ValueError, match="bad IHDR"):
        png.parse(good[:8] + good[33:])                    # first chunk is not IHDR
    i = good.index(b"IDAT") - 4
    n = struct.unpack(">I", good[i:i + 4])[0]
    with pytest.raises(ValueError, match="no IDAT"):
        png.parse(good[:i] + good[i + 12 + n:])
    with pytest.raises(ValueError, match="truncated"):
        png.parse(good[:i + 20])


def test_rejects_mixed_sizes_in_one_batch():
    dec = png.PngDecoder.__new__(png.PngDecoder)
    with pytest.raises(ValueError, match="different sizes"):
        dec.prepare([_bytes("hand_filter0"), _bytes("cv2_small")])


def test_oracle_flags_corrupt_streams():
    good = _bytes("hand_filter_random")
    h = png.parse(good)
    total = h.height * (1 + (h.width * h.depth + 7) // 8)
    z = h.zdata
    with pytest.raises(po.Corrupt):
        po.inflate(z[:len(z) // 2], total)                # truncated
    with pytest.raises(po.Corrupt, match="Adler"):
        po.inflate(z[:-1] + bytes([z[-1] ^ 1]), total)
    with pytest.raises(po.Corrupt):
        po.inflate(z, total + 1)                           # output shorter than the image


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def test_png_struct_matches_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header structs")
    cls = _capi.LfPngImage
    body = '    printf("%zu\\n", sizeof(LfPngImage));\n'
    body += "".join('    printf("%%zu\\n", offsetof(LfPngImage, %s));\n' % f[0] for f in cls._fields_)
    body += '    printf("%d\\n", LF_STATUS_PNG_CORRUPT);\n'
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n' + body +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    want = [str(ctypes.sizeof(cls))] + [str(getattr(cls, f[0]).offset) for f in cls._fields_]
    assert lines[:len(want)] == want
    assert lines[len(want)] == str(_capi.STATUS_PNG_CORRUPT)


@pytest.mark.parametrize("name", ["lf_png_workspace_bytes", "lf_png_decode", "lf_label_preprocess"])
def test_png_prototypes_match_declaration_and_export(name):
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\b(int|size_t)\s+%s\s*\((.*?)\);" % name, hdr, re.S)
    assert decl
    res, args = _capi.PROTOTYPES[name]
    assert res is {"int": ctypes.c_int, "size_t": ctypes.c_size_t}[decl.group(1)]
    assert len(args) == len(decl.group(2).split(","))
    assert hasattr(_capi.lib(), name)


def test_workspace_query_lays_out_a_batch():
    dec = png.PngDecoder.__new__(png.PngDecoder)
    names = ["hand_filter0", "hand_filter_random", "hand_many_idat"]
    blob, N, W, H, wsb = dec.prepare([_bytes(n) for n in names])
    desc = np.frombuffer(blob[:N * png._IMG_DTYPE.itemsize].tobytes(), dtype=png._IMG_DTYPE)
    assert (N, W, H) == (3, 101, 64)
    assert all(int(d["rowbytes"]) == 101 for d in desc)
    for d, n in zip(desc, names):
        z = png.parse(_bytes(n)).zdata
        assert blob[int(d["zoff"]):int(d["zoff"]) + int(d["zlen"])].tobytes() == z
    assert int(desc[-1]["raw_off"]) + 64 * 102 <= wsb and int(desc[0]["raw_off"]) >= 16 * N
