"""JPEG decode without a GPU: the marker parser against Pillow's view of every fixture, the numpy / Python restatement
(oracle/jpeg_oracle.py) against the golden bytes Pillow produced (tests/golden/jpeg_pil.npz) and against live Pillow,
every rejection of an unsupported file, and the C ABI (LfJpegImage layout, prototypes, exports)."""
import ctypes
import hashlib
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import jpeg_oracle as jo
from oracle.make_jpeg_golden import CASES, encode, make_frame
from lanedetection_end2end_b200 import jpeg

SMALL = [c for c in CASES if c[1] * c[2] <= 200000]


def _golden():
    return np.load(os.path.join(GOLDEN, "jpeg_pil.npz"))


def _bytes(name):
    return bytes(_golden()[name + "/jpeg"])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_parser_agrees_with_pillow(case):
    Image = pytest.importorskip("PIL.Image")
    from PIL import JpegImagePlugin
    data = _bytes(case[0])
    h = jpeg.parse(data)
    im = Image.open(io.BytesIO(data))
    assert (h.width, h.height) == im.size
    assert h.sampling == JpegImagePlugin.get_sampling(im)
    assert set(h.qtables) == set(im.quantization)
    for t, q in im.quantization.items():        # both in natural (row-major) order
        np.testing.assert_array_equal(h.qtables[t], np.asarray(q))
    assert h.ecs_off + h.ecs_len <= len(data)


@pytest.mark.parametrize("case", SMALL, ids=[c[0] for c in SMALL])
def test_oracle_reproduces_golden(case):
    g = _golden()
    name = case[0]
    got, stats = jo.decode(_bytes(name))
    assert hashlib.sha256(got.tobytes()).hexdigest() == str(g[name + "/sha256"])
    np.testing.assert_array_equal(got, g[name + "/rgb"])
    assert stats["symbols"] > 0


def test_oracle_reproduces_golden_full_frame():
    g = _golden()
    got, stats = jo.decode(_bytes("frame_q75_420"))
    np.testing.assert_array_equal(got.reshape(-1)[g["frame_q75_420/idx"]], g["frame_q75_420/val"])
    assert hashlib.sha256(got.tobytes()).hexdigest() == str(g["frame_q75_420/sha256"])


@pytest.mark.parametrize("case", SMALL[:6] + SMALL[9:12], ids=[c[0] for c in SMALL[:6] + SMALL[9:12]])
def test_oracle_matches_live_pillow(case):
    pytest.importorskip("PIL.Image")
    from oracle.make_jpeg_golden import pil_decode
    data = encode(case)
    np.testing.assert_array_equal(jo.decode(data)[0], pil_decode(data))


# ---- rejections ------------------------------------------------------------------------------------------------------
def _pillow(mode, **kw):
    Image = pytest.importorskip("PIL.Image")
    a = make_frame(32, 48, 3, "RGB")
    im = Image.fromarray(a).convert(mode)
    bio = io.BytesIO()
    im.save(bio, "JPEG", **kw)
    return bio.getvalue()


def _marker_pos(data, m):
    i = data.find(bytes([0xFF, m]))
    assert i > 0
    return i


def _with_sof(data, m, precision=None):
    d = bytearray(data)
    i = _marker_pos(data, 0xC0)
    d[i + 1] = m
    if precision is not None:
        d[i + 4] = precision
    return bytes(d)


def test_rejects_progressive_and_cmyk():
    with pytest.raises(ValueError, match="progressive"):
        jpeg.parse(_pillow("RGB", progressive=True))
    with pytest.raises(ValueError, match="4 components"):
        jpeg.parse(_pillow("CMYK"))


@pytest.mark.parametrize("m,msg", [(0xC2, "progressive"), (0xC3, "lossless"), (0xC9, "arithmetic")])
def test_rejects_other_frame_types(m, msg):
    with pytest.raises(ValueError, match=msg):
        jpeg.parse(_with_sof(_bytes("q75_420"), m))


def test_rejects_12bit_second_scan_dnl_rgb_and_sampling():
    base = _bytes("q75_420")
    with pytest.raises(ValueError, match="12-bit"):
        jpeg.parse(_with_sof(base, 0xC1, precision=12))
    h = jpeg.parse(base)
    end = h.ecs_off + h.ecs_len
    sos = _marker_pos(base, 0xDA)
    two = base[:end] + base[sos:end] + base[end:]          # a second SOS + scan before EOI
    with pytest.raises(ValueError, match="more than one scan"):
        jpeg.parse(two)
    dnl = base[:end] + bytes([0xFF, 0xDC, 0, 4, 0, 96]) + base[end:]
    with pytest.raises(ValueError, match="DNL"):
        jpeg.parse(dnl)
    d = bytearray(base)
    i = _marker_pos(base, 0xC0)
    d[i + 5:i + 7] = b"\x00\x00"                            # height 0: defined by a DNL marker
    with pytest.raises(ValueError, match="DNL"):
        jpeg.parse(bytes(d))
    with pytest.raises(ValueError, match="stored RGB"):
        jpeg.parse(_pillow("RGB", keep_rgb=True))
    d = bytearray(base)
    d[i + 11] = 0x12                                       # Cb sampled 1x2
    with pytest.raises(ValueError, match="sampling"):
        jpeg.parse(bytes(d))
    with pytest.raises(ValueError, match="more than one scan"):
        jpeg.parse(_with_sos_components(base, 1))


def _with_sos_components(data, ns):
    """rewrite the SOS header to code only the first `ns` components (a non-interleaved first scan)"""
    i = _marker_pos(data, 0xDA)
    n0 = data[i + 4]
    seg = bytes([ns]) + data[i + 5:i + 5 + 2 * ns] + data[i + 5 + 2 * n0:i + 8 + 2 * n0]
    return data[:i + 2] + (len(seg) + 2).to_bytes(2, "big") + seg + data[i + 8 + 2 * n0:]


def test_rejects_mixed_sizes_in_one_batch():
    dec = jpeg.JpegDecoder.__new__(jpeg.JpegDecoder)
    with pytest.raises(ValueError, match="different sizes"):
        dec.prepare([_bytes("q75_420"), _bytes("q90_444")])


def test_huffman_tables_decode_every_code():
    """lookahead / maxcode tables give back every (code, symbol) of the canonical code"""
    h = jpeg.parse(_bytes("q100_420"))
    for tabs, dc in ((h.dc_tables, True), (h.ac_tables, False)):
        for bits, vals in tabs.values():
            t = jpeg.huffman_table(bits, vals, dc)
            for (l, code), sym in jo._codes(list(bits), list(vals)).items():
                win = code << (32 - l)
                look = int(t["look"][win >> 23])
                if l <= 9:
                    assert look == (l << 8) | sym
                else:
                    assert look == 0
                    got = next(ll for ll in range(10, 17) if (win >> (32 - ll)) <= t["maxcode"][ll])
                    assert got == l and t["val"][(win >> (32 - l)) + t["valoff"][l]] == sym


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def test_jpeg_structs_match_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header structs")
    structs = {"LfJpegHuff": _capi.LfJpegHuff, "LfJpegImage": _capi.LfJpegImage}
    body = ""
    for name, cls in structs.items():
        body += '    printf("%%zu\\n", sizeof(%s));\n' % name
        body += "".join('    printf("%%zu\\n", offsetof(%s, %s));\n' % (name, f[0]) for f in cls._fields_)
    body += '    printf("%d %d %d\\n", LF_STATUS_JPEG_CORRUPT, LF_JPEG_PIECE_BYTES, LF_JPEG_MAX_BPM);\n'
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n' + body +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    want = []
    for cls in structs.values():
        want.append(str(ctypes.sizeof(cls)))
        want += [str(getattr(cls, f[0]).offset) for f in cls._fields_]
    assert lines[:len(want)] == want
    assert lines[len(want)] == "%d %d %d" % (_capi.STATUS_JPEG_CORRUPT, _capi.JPEG_PIECE_BYTES, _capi.JPEG_MAX_BPM)


@pytest.mark.parametrize("name", ["lf_jpeg_workspace_bytes", "lf_jpeg_decode"])
def test_jpeg_prototypes_match_declaration_and_export(name):
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\b(int|size_t)\s+%s\s*\((.*?)\);" % name, hdr, re.S)
    assert decl
    res, args = _capi.PROTOTYPES[name]
    assert res is {"int": ctypes.c_int, "size_t": ctypes.c_size_t}[decl.group(1)]
    assert len(args) == len(decl.group(2).split(","))
    assert hasattr(_capi.lib(), name)


def test_workspace_query_lays_out_a_batch():
    dec = jpeg.JpegDecoder.__new__(jpeg.JpegDecoder)
    blob, N, W, H, wsb, cb = dec.prepare([_bytes("rst_blocks_420"), _bytes("q75_420"), _bytes("q75_444")])
    desc = np.frombuffer(blob[:N * jpeg._IMG_DTYPE.itemsize].tobytes(), dtype=jpeg._IMG_DTYPE)
    assert (N, W, H) == (3, 160, 96)
    assert cb == 128 * sum(int(d["mcux"] * d["mcuy"] * d["bpm"]) for d in desc)
    assert int(desc[0]["nint"]) == 12 and int(desc[1]["nint"]) == 1 and int(desc[2]["bpm"]) == 3
    ends = [int(d["plane_off"][2]) + int(d["plane_stride"][2]) * int(d["mcuy"]) * 8 * int(d["vs"][2]) for d in desc]
    assert max(ends) <= wsb


@pytest.mark.parametrize("sub", [0, 1, 2])
def test_oracle_matches_live_pillow_narrow_widths(sub):
    """widths 1..4 (chroma 1..2 samples wide in 4:2:2 / 4:2:0: libjpeg replicates instead of the fancy filter)"""
    pytest.importorskip("PIL.Image")
    from oracle.make_jpeg_golden import pil_decode
    from PIL import Image
    rng = np.random.default_rng(40 + sub)
    for w in (1, 2, 3, 4, 5):
        for h in (1, 2, 3, 7, 17):
            bio = io.BytesIO()
            Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(bio, "JPEG", quality=85, subsampling=sub)
            data = bio.getvalue()
            np.testing.assert_array_equal(jo.decode(data)[0], pil_decode(data), err_msg="%dx%d" % (w, h))


def test_rejects_huffman_table_with_an_all_ones_code():
    bits = bytes([0, 3] + [0] * 14)               # 4 codes of length 2 would use 11: libjpeg's JERR_BAD_HUFF_TABLE
    jpeg.huffman_table(bits, bytes([0, 1, 2]), True)
    with pytest.raises(ValueError, match="bad Huffman table"):
        jpeg.huffman_table(bytes([0, 4] + [0] * 14), bytes([0, 1, 2, 3]), True)


def test_huffman_table_cache_is_bounded():
    for k in range(200):                           # distinct (optimised-looking) tables
        jpeg.huffman_table(bytes([0, 2, 1] + [0] * 13), bytes([k % 12, (k // 12) % 12 + 1, 0]), True)
    assert jpeg._huffman_table.cache_info().currsize <= jpeg._huffman_table.cache_info().maxsize
