"""C ABI of the bf16 storage entry points, checked without a GPU: the ctypes mirror of LfConvTcArgs (with its appended
in_dtype / out_dtype / mask_dtype fields) against the C compiler's layout of the header struct, and the new prototypes
against their declarations and the library's exports."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

HEADER_DIR = os.path.join(ROOT, "include")
NEW_ENTRIES = ("lf_wgrad3_tc_bf16a", "lf_bn_apply_bf16")


def _header():
    return open(os.path.join(HEADER_DIR, "lanefit_b200.h")).read()


def test_conv_tc_args_size_and_offsets_match_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header struct")
    fields = [f[0] for f in _capi.LfConvTcArgs._fields_]
    assert fields[-3:] == ["in_dtype", "out_dtype", "mask_dtype"]
    cnames = ["in" if f == "inp" else f for f in fields]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n'
                   '    printf("%zu", sizeof(LfConvTcArgs));\n' +
                   "".join('    printf(" %%zu", offsetof(LfConvTcArgs, %s));\n' % n for n in cnames) +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", HEADER_DIR, str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[0] == ctypes.sizeof(_capi.LfConvTcArgs)
    assert got[1:] == [getattr(_capi.LfConvTcArgs, f).offset for f in fields]
    a = _capi.LfConvTcArgs()
    assert (a.in_dtype, a.out_dtype, a.mask_dtype) == (_capi.LF_F32,) * 3   # zero-initialised = the fp32 behaviour


def test_new_prototypes_match_declarations_and_exports():
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
    # same argument lists as their fp32-operand siblings
    assert _capi.PROTOTYPES["lf_wgrad3_tc_bf16a"] == _capi.PROTOTYPES["lf_wgrad3_tc_bf16"]
    assert _capi.PROTOTYPES["lf_bn_apply_bf16"] == _capi.PROTOTYPES["lf_bn_apply"]
