"""C ABI of the bf16 storage entry points, checked without a GPU: the ctypes mirrors of LfConvTcArgs (with its appended
in_dtype / out_dtype / mask_dtype fields) and LfWgradTcgArgs (with its appended a_dtype field) against the C compiler's
layout of the header structs, and the prototypes against their declarations and the library's exports."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

HEADER_DIR = os.path.join(ROOT, "include")
NEW_ENTRIES = ("lf_bn_apply_bf16", "lf_wgrad_tcg_ctas")
# the weight-gradient entry points that lf_wgrad_tcg (LfWgradTcgArgs.a_dtype) and lf_wgrad_tcg_ctas (min_patches) replace
REMOVED_ENTRIES = ("lf_wgrad3_tc", "lf_wgrad3_tc_x3", "lf_wgrad3_tc_bf16", "lf_wgrad3_tc_bf16a", "lf_wgrad3_tc_ctas",
                   "lf_wgrad3_tc_x3_ctas", "lf_wgrad3_tc_bf16_ctas", "lf_wgrad_tcg_ctas_x3", "lf_wgrad_tcg_ctas_bf16")


def _header():
    return open(os.path.join(HEADER_DIR, "lanefit_b200.h")).read()


def _c_layout(tmp_path, cname, cnames):
    """[sizeof(cname), offsetof(cname, f) for f in cnames] as the C compiler lays the header struct out."""
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header struct")
    src = tmp_path / ("%s.c" % cname)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n'
                   '    printf("%%zu", sizeof(%s));\n' % cname +
                   "".join('    printf(" %%zu", offsetof(%s, %s));\n' % (cname, n) for n in cnames) +
                   "    return 0;\n}\n")
    exe = tmp_path / cname
    subprocess.run([cc, "-I", HEADER_DIR, str(src), "-o", str(exe)], check=True)
    return [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def test_conv_tc_args_size_and_offsets_match_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    fields = [f[0] for f in _capi.LfConvTcArgs._fields_]
    assert fields[-3:] == ["in_dtype", "out_dtype", "mask_dtype"]
    got = _c_layout(tmp_path, "LfConvTcArgs", ["in" if f == "inp" else f for f in fields])
    assert got[0] == ctypes.sizeof(_capi.LfConvTcArgs)
    assert got[1:] == [getattr(_capi.LfConvTcArgs, f).offset for f in fields]
    a = _capi.LfConvTcArgs()
    assert (a.in_dtype, a.out_dtype, a.mask_dtype) == (_capi.LF_F32,) * 3   # zero-initialised = the fp32 behaviour


def test_wgrad_tcg_args_size_and_offsets_match_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    fields = [f[0] for f in _capi.LfWgradTcgArgs._fields_]
    assert fields[-2:] == ["precision", "a_dtype"]
    got = _c_layout(tmp_path, "LfWgradTcgArgs", fields)
    assert got[0] == ctypes.sizeof(_capi.LfWgradTcgArgs)
    assert got[1:] == [getattr(_capi.LfWgradTcgArgs, f).offset for f in fields]
    assert _capi.LfWgradTcgArgs().a_dtype == _capi.LF_F32                    # zero-initialised = fp32 A views


def test_bf16_and_wgrad_tcg_prototypes_match_declarations_and_exports():
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    h = _capi.lib()
    for name in NEW_ENTRIES:
        decl = re.search(r"\bint\s+%s\s*\((.*?)\);" % name, hdr, re.S)
        assert decl, name
        nargs = len(decl.group(1).split(","))
        res, args = _capi.PROTOTYPES[name]
        assert res is ctypes.c_int and len(args) == nargs, name
        assert hasattr(h, name), name
    for name in REMOVED_ENTRIES:
        assert not re.search(r"\b%s\b" % name, _header()), name
        assert name not in _capi.PROTOTYPES and not hasattr(h, name), name
    # same argument list as its fp32-output sibling
    assert _capi.PROTOTYPES["lf_bn_apply_bf16"] == _capi.PROTOTYPES["lf_bn_apply"]
