"""The per-parameter step count of the fused optimizer without a GPU: the C ABI of lf_optim_step_pp (the ctypes mirror of
LfOptimSegPP against the C compiler's layout of the header, the prototype against its declaration and the library's
export), every argument refusal of the entry point, no spills in either of its kernels, the Python argument checks, the
torch-format checkpoints of FusedOptimizer(per_param_step=True) with differing steps and parameters without state, and
the default mode's refusals of both."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import optim_cases as oc
from conftest import ROOT

HEADER_DIR = os.path.join(ROOT, "include")
INVALID = -1


def _capi():
    from lanedetection_end2end_b200 import _capi
    return _capi


def test_segpp_struct_matches_the_header(tmp_path):
    capi = _capi()
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header structs")
    cls = capi.LfOptimSegPP
    body = '    printf("%zu\\n", sizeof(LfOptimSegPP));\n'
    body += "".join('    printf("%%zu\\n", offsetof(LfOptimSegPP, %s));\n' % f[0] for f in cls._fields_)
    body += '    printf("%d\\n", LF_OPTIM_PP_SCALAR_BYTES);\n'
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n' + body +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", HEADER_DIR, str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    want = [str(ctypes.sizeof(cls))] + [str(getattr(cls, f[0]).offset) for f in cls._fields_]
    assert lines[:len(want)] == want
    assert lines[len(want)] == str(capi.OPTIM_PP_SCALAR_BYTES)
    # the Python table rows: seven int64 per row, the slot in the low half of the last
    assert ctypes.sizeof(cls) == 7 * 8 and cls.slot.offset == 6 * 8


def test_pp_prototype_matches_declaration_and_export():
    capi = _capi()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(HEADER_DIR, "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+lf_optim_step_pp\s*\((.*?)\);", hdr, re.S)
    assert decl
    res, args = capi.PROTOTYPES["lf_optim_step_pp"]
    assert res is ctypes.c_int and len(args) == len(decl.group(1).split(","))
    assert hasattr(capi.lib(), "lf_optim_step_pp")


# ---------------------------------------------------------------------------------------------------------------------
# argument refusals (no launch happens: no device needed)
# ---------------------------------------------------------------------------------------------------------------------
class _Bufs:
    """Host buffers standing in for device pointers: every call below is refused before anything reads them."""

    def __init__(self):
        self.mem = np.zeros(1 << 12, np.float64)
        base = self.mem.ctypes.data
        self.p = lambda k: base + 64 * k + (64 - base % 64) % 64


def _call(b, slots=(0, 2, 1), **kw):
    a = dict(algo=0, segs=b.p(0), nsegs=3 if slots is None else len(slots), nchunks=5, hyper=b.p(8), steps=b.p(9),
             nparams=3, scalars=b.p(10), skipped=b.p(11), status=None)
    a.update(kw)
    host = None if slots is None else (ctypes.c_int * max(1, len(slots)))(*slots)
    return _capi().lib().lf_optim_step_pp(a["algo"], a["segs"], host, a["nsegs"], a["nchunks"], a["hyper"], a["steps"],
                                           a["nparams"], a["scalars"], a["skipped"], a["status"], None)


no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="host addresses as device pointers: CPU-only machines")


@no_device
@pytest.mark.parametrize("bad", [
    dict(segs=None), dict(hyper=None), dict(steps=None), dict(scalars=None), dict(skipped=None), dict(nsegs=0),
    dict(nsegs=-1), dict(nchunks=0), dict(nparams=0), dict(algo=3), dict(algo=-1), dict(slots=None),
    dict(slots=(0, 3, 1)), dict(slots=(0, -1, 1)), dict(slots=(0, 2, 0)), dict(slots=(1, 1, 1)),
    dict(slots=(0, 1, 2, 3), nparams=3), dict(scalars="odd")])
def test_pp_refuses_bad_arguments(bad):
    b = _Bufs()
    if bad.get("scalars") == "odd":
        bad = dict(scalars=b.p(10) + 8)               # not 16-byte aligned
    assert _call(b, **bad) == INVALID


def test_pp_kernels_do_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "optim.cu"), "-o",
                                              str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            found[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    pp = [k for k in found if "optim_pp_kernel" in k]
    sc = [k for k in found if "optim_pp_scalars_kernel" in k]
    assert len(pp) == 3 and len(sc) == 1, sorted(found)
    for k in pp + sc:
        assert found[k] == (0, 0), (k, found[k])


# ---------------------------------------------------------------------------------------------------------------------
# Python argument checks and checkpoints (a CPU FusedOptimizer can load and save; only its update needs the GPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_python_argument_checks():
    from lanedetection_end2end_b200.Networks.utils import define_optim
    from lanedetection_end2end_b200.optim import FusedOptimizer
    p = [torch.zeros(4, requires_grad=True), torch.zeros(3, requires_grad=True)]
    for bad in (1, 0, "yes", None):
        with pytest.raises(TypeError, match="per_param_step"):
            FusedOptimizer(p, "adam", 1e-3, 0, per_param_step=bad)
    assert FusedOptimizer(p, "adam", 1e-3, 0).per_param_step is False
    o = define_optim("rmsprop", p, 1e-3, 0, fused=True, per_param_step=True)
    assert isinstance(o, FusedOptimizer) and o.per_param_step and o.kind == "rmsprop"
    assert o.step_counts == [0, 0] and o.step_count == 0
    assert not define_optim("sgd", p, 1e-3, 0, fused=True).per_param_step
    assert type(define_optim("adam", p, 1e-3, 0, fused=False, per_param_step=True)) is torch.optim.Adam


def _subset_grads(steps=6):
    """grads[step][tensor] over oc.SHAPES: a changing subset of the parameters (starts with some, adds, drops, brings
    back), so the per-parameter steps of torch.optim differ."""
    full = oc.make_grads(steps=steps)
    n = len(oc.SHAPES)
    have = [set(range(0, n, 2)), set(range(n)), set(range(n)) - {1, 3, 4}, set(range(n)) - {1, 3, 4}, set(range(n)),
            set(range(3, n))]
    return [[g if i in have[t % len(have)] else None for i, g in enumerate(full[t])] for t in range(steps)]


@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_checkpoints_with_differing_steps_round_trip(kind):
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), _subset_grads(4)
    pt, ot = oc.torch_run(kind, 1e-4, params, grads, torch.float32, "cpu", 4)
    sd_t = ot.state_dict()
    if kind != "sgd":
        assert len({float(st["step"]) for st in sd_t["state"].values()}) > 1
    assert oc.NONE_GRAD not in sd_t["state"]
    ours = FusedOptimizer([p.clone() for p in pt], kind, oc.LR[kind], 1e-4, per_param_step=True)
    ours.load_state_dict(sd_t)
    want = [0] * len(pt)
    for i, st in sd_t["state"].items():
        want[i] = 1 if kind == "sgd" else int(st["step"])     # torch's SGD keeps no step: 1 = has a momentum buffer
    assert ours.step_counts == want and ours.step_count == max(want)
    sd_o = ours.state_dict()
    assert sd_o["param_groups"] == sd_t["param_groups"] and set(sd_o["state"]) == set(sd_t["state"])
    for i, st in sd_t["state"].items():
        assert list(sd_o["state"][i]) == list(st)
        for k, v in st.items():
            assert sd_o["state"][i][k].dtype == v.dtype and sd_o["state"][i][k].device == v.device
            assert torch.equal(sd_o["state"][i][k], v), (i, k)
    back = oc.KINDS[kind][0]([p.clone() for p in pt], lr=oc.LR[kind], weight_decay=1e-4, **oc.KINDS[kind][1])
    back.load_state_dict(sd_o)
    # a dict with fewer parameters than the optimizer has state for: the others return to step 0 and zero state
    drop = next(iter(sd_t["state"]))
    fewer = {"state": {i: st for i, st in sd_t["state"].items() if i != drop}, "param_groups": sd_t["param_groups"]}
    ours.load_state_dict(fewer)
    assert ours.step_counts[drop] == 0 and drop not in ours.state_dict()["state"]
    p_drop = ours.param_groups[0]["params"][drop]
    assert all(not bool(ours.state[p_drop][k].any()) for k in oc.STATE_NAMES[kind])


def test_default_mode_refusals_still_raise():
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), _subset_grads(2)
    pt, ot = oc.torch_run("adam", 0.0, params, grads, torch.float32, "cpu", 2)
    sd = ot.state_dict()
    ours = FusedOptimizer([p.clone() for p in pt], "adam", 1e-3, 0.0)
    with pytest.raises(ValueError, match="FusedOptimizer keeps one step count for all parameters"):
        ours.load_state_dict(sd)
    pp = FusedOptimizer([p.clone() for p in pt], "adam", 1e-3, 0.0, per_param_step=True)
    pp.load_state_dict(sd)
    # a checkpoint of equal steps loads in the default mode; one that leaves out a parameter with state does not
    _, o2 = oc.torch_run("adam", 0.0, params, oc.make_grads(steps=2), torch.float32, "cpu", 2)
    ours.load_state_dict(o2.state_dict())
    assert ours.step_count == 2
    less = o2.state_dict()
    del less["state"][0]
    with pytest.raises(ValueError, match="parameter 0 has optimizer state but none in the state dict"):
        ours.load_state_dict(less)
    pp.load_state_dict(less)
    assert pp.step_counts[0] == 0 and pp.step_counts[1] == 2
