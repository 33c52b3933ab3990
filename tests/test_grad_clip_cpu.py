"""Gradient clipping in the fused optimizer without a GPU: the C ABI of lf_grad_norm / lf_grad_norm_pp /
lf_optim_step_clip / lf_optim_step_pp_clip (the ctypes mirror of LfGradClip against the C compiler's layout of the header,
the prototypes against their declarations and the library's exports, every argument refusal), no spills in the new
kernels, FusedOptimizer's max_grad_norm checks, torch-format checkpoints with clipping on, define_optim's pass-through,
and an fp32 restatement of the kernel's clip coefficient bit for bit against torch.nn.utils.clip_grads_with_norm_."""
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
NEW_ENTRIES = ("lf_grad_norm_workspace_bytes", "lf_grad_norm", "lf_grad_norm_pp", "lf_optim_step_clip",
               "lf_optim_step_pp_clip")


def _capi():
    from lanedetection_end2end_b200 import _capi
    return _capi


def test_gradclip_struct_matches_the_header(tmp_path):
    capi = _capi()
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header structs")
    cls = capi.LfGradClip
    body = '    printf("%zu\\n", sizeof(LfGradClip));\n'
    body += "".join('    printf("%%zu\\n", offsetof(LfGradClip, %s));\n' % f[0] for f in cls._fields_)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n' + body +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", HEADER_DIR, str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    want = [str(ctypes.sizeof(cls))] + [str(getattr(cls, f[0]).offset) for f in cls._fields_]
    assert lines[:len(want)] == want
    # optim.FusedOptimizer's block: four int64, max_norm / total_norm / clip_coef as fp32 words 0-2, the count in int64 2
    assert ctypes.sizeof(cls) == 4 * 8 and cls.total_norm.offset == 4 and cls.nonfinite_skipped.offset == 2 * 8


def test_prototypes_match_declarations_and_exports():
    capi = _capi()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(HEADER_DIR, "lanefit_b200.h")).read(), flags=re.S)
    for name in NEW_ENTRIES:
        decl = re.search(r"\b(int|size_t)\s+%s\s*\((.*?)\);" % name, hdr, re.S)
        assert decl, name
        res, args = capi.PROTOTYPES[name]
        assert res is (ctypes.c_int if decl.group(1) == "int" else ctypes.c_size_t), name
        assert len(args) == len(decl.group(2).split(",")), name
        assert hasattr(capi.lib(), name), name


def test_workspace_query():
    lib = _capi().lib()
    assert lib.lf_grad_norm_workspace_bytes(1) == 8
    assert lib.lf_grad_norm_workspace_bytes(3580) == 3580 * 8
    assert lib.lf_grad_norm_workspace_bytes(0) == 0 and lib.lf_grad_norm_workspace_bytes(-2) == 0


# ---------------------------------------------------------------------------------------------------------------------
# argument refusals (no launch happens: no device needed)
# ---------------------------------------------------------------------------------------------------------------------
class _Bufs:
    """Host buffers standing in for device pointers: every call below is refused before anything reads them."""

    def __init__(self):
        self.mem = np.zeros(1 << 12, np.float64)
        base = self.mem.ctypes.data
        self.p = lambda k: base + 64 * k + (64 - base % 64) % 64


no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="host addresses as device pointers: CPU-only machines")


def _norm(b, pp, **kw):
    a = dict(segs=b.p(0), nsegs=3, nchunks=5, clip=b.p(8), ws=b.p(9), ws_bytes=5 * 8)
    a.update(kw)
    fn = _capi().lib().lf_grad_norm_pp if pp else _capi().lib().lf_grad_norm
    return fn(a["segs"], a["nsegs"], a["nchunks"], a["clip"], a["ws"], a["ws_bytes"], None)


@no_device
@pytest.mark.parametrize("pp", [False, True])
@pytest.mark.parametrize("bad", [
    dict(segs=None), dict(clip=None), dict(ws=None), dict(nsegs=0), dict(nsegs=-1), dict(nchunks=0), dict(nchunks=-3),
    dict(ws_bytes=4 * 8), dict(ws_bytes=0), dict(ws="odd")])
def test_norm_refuses_bad_arguments(pp, bad):
    b = _Bufs()
    if bad.get("ws") == "odd":
        bad = dict(ws=b.p(9) + 4)                      # not 8-byte aligned
    assert _norm(b, pp, **bad) == INVALID


def _step_clip(b, **kw):
    a = dict(algo=0, segs=b.p(0), nsegs=3, nchunks=5, hyper=b.p(8), state=b.p(9), status=None, clip=b.p(10))
    a.update(kw)
    return _capi().lib().lf_optim_step_clip(a["algo"], a["segs"], a["nsegs"], a["nchunks"], a["hyper"], a["state"],
                                            a["status"], a["clip"], None)


@no_device
@pytest.mark.parametrize("bad", [dict(clip=None), dict(segs=None), dict(hyper=None), dict(state=None), dict(nsegs=0),
                                 dict(nchunks=0), dict(algo=3), dict(algo=-1)])
def test_step_clip_refuses_bad_arguments(bad):
    assert _step_clip(_Bufs(), **bad) == INVALID


def _step_pp_clip(b, slots=(0, 2, 1), **kw):
    a = dict(algo=0, segs=b.p(0), nsegs=3 if slots is None else len(slots), nchunks=5, hyper=b.p(8), steps=b.p(9),
             nparams=3, scalars=b.p(10), skipped=b.p(11), status=None, clip=b.p(12))
    a.update(kw)
    host = None if slots is None else (ctypes.c_int * max(1, len(slots)))(*slots)
    return _capi().lib().lf_optim_step_pp_clip(a["algo"], a["segs"], host, a["nsegs"], a["nchunks"], a["hyper"],
                                               a["steps"], a["nparams"], a["scalars"], a["skipped"], a["status"],
                                               a["clip"], None)


@no_device
@pytest.mark.parametrize("bad", [
    dict(clip=None), dict(segs=None), dict(skipped=None), dict(scalars=None), dict(nsegs=0), dict(nchunks=0),
    dict(algo=3), dict(slots=None), dict(slots=(0, 2, 0)), dict(slots=(0, 3, 1)), dict(scalars="odd")])
def test_step_pp_clip_refuses_bad_arguments(bad):
    b = _Bufs()
    if bad.get("scalars") == "odd":
        bad = dict(scalars=b.p(10) + 8)
    assert _step_pp_clip(b, **bad) == INVALID


def test_clip_kernels_do_not_spill(tmp_path):
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
    norm = [k for k in found if "grad_norm_kernel" in k]
    step = [k for k in found if "optim_kernel" in k and "Lb1E" in k]
    pp = [k for k in found if "optim_pp_clip_kernel" in k]
    assert len(norm) == 2 and len(step) == 3 and len(pp) == 3, sorted(found)
    for k in norm + step + pp:
        assert found[k] == (0, 0), (k, found[k])


# ---------------------------------------------------------------------------------------------------------------------
# FusedOptimizer(max_grad_norm=...)
# ---------------------------------------------------------------------------------------------------------------------
BAD_NORMS = (0, 0.0, -1.0, float("inf"), float("-inf"), float("nan"), "1.0", True, 1e39, 1e-50, [1.0])


def test_max_grad_norm_is_checked():
    from lanedetection_end2end_b200.optim import FusedOptimizer
    p = [torch.zeros(4, requires_grad=True)]
    for bad in BAD_NORMS:
        with pytest.raises(ValueError, match="max_grad_norm"):
            FusedOptimizer(p, "adam", 1e-3, 0, max_grad_norm=bad)
    assert FusedOptimizer(p, "adam", 1e-3, 0).max_grad_norm is None
    o = FusedOptimizer(p, "sgd", 1e-3, 0, per_param_step=True, max_grad_norm=2)
    assert o.max_grad_norm == 2.0 and isinstance(o.max_grad_norm, float)
    for bad in BAD_NORMS:
        with pytest.raises(ValueError, match="max_grad_norm"):
            o.max_grad_norm = bad
    assert o.max_grad_norm == 2.0
    o.max_grad_norm = 0.25
    o.sync_hyperparameters()                     # the threshold reaches the fp32 word the kernel reads
    assert o._clip.view(torch.float32)[0].item() == 0.25
    o.max_grad_norm = None
    assert o.max_grad_norm is None
    # the read-outs before any clipped update
    assert o.nonfinite_skipped == 0
    g = o.grad_norm
    assert g.dtype == torch.float32 and g.dim() == 0 and float(g) == 0.0


@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_state_dict_is_torch_format_with_clipping(kind):
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), oc.make_grads(steps=3)
    pt, ot = oc.torch_run(kind, 1e-4, params, grads, torch.float32, "cpu", 3)
    sd_t = ot.state_dict()
    cls, extra = oc.KINDS[kind]
    for pp in (False, True):
        ours = FusedOptimizer([p.clone() for p in pt], kind, oc.LR[kind], 1e-4, per_param_step=pp, max_grad_norm=0.5)
        fresh_t = cls([p.clone() for p in pt], lr=oc.LR[kind], weight_decay=1e-4, **extra).state_dict()
        assert ours.state_dict() == fresh_t
        ours.load_state_dict(sd_t)
        sd_o = ours.state_dict()
        assert sd_o["param_groups"] == sd_t["param_groups"] and set(sd_o["state"]) == set(sd_t["state"])
        assert "max_grad_norm" not in sd_o["param_groups"][0]
        for i, st in sd_t["state"].items():
            assert list(sd_o["state"][i]) == list(st)
            for k, v in st.items():
                assert torch.equal(sd_o["state"][i][k], v), (i, k)
        back = cls([p.clone() for p in pt], lr=oc.LR[kind], weight_decay=1e-4, **extra)
        back.load_state_dict(sd_o)
        assert back.state_dict()["param_groups"] == sd_t["param_groups"]
        assert ours.max_grad_norm == 0.5


def test_define_optim_passes_max_grad_norm():
    from lanedetection_end2end_b200.Networks.utils import define_optim
    from lanedetection_end2end_b200.optim import FusedOptimizer
    p = [torch.zeros(4, requires_grad=True)]
    o = define_optim("rmsprop", p, 1e-3, 0, fused=True, per_param_step=True, max_grad_norm=3.0)
    assert isinstance(o, FusedOptimizer) and o.max_grad_norm == 3.0 and o.per_param_step
    assert define_optim("adam", p, 1e-3, 0, fused=True).max_grad_norm is None
    t = define_optim("sgd", p, 1e-3, 0, fused=False, max_grad_norm=3.0)
    assert type(t) is torch.optim.SGD and "max_grad_norm" not in t.param_groups[0]
    with pytest.raises(ValueError, match="max_grad_norm"):
        define_optim("adam", p, 1e-3, 0, fused=True, max_grad_norm=-1.0)


# ---------------------------------------------------------------------------------------------------------------------
# the clip coefficient: the kernel's fp32 op order against torch's own call
# ---------------------------------------------------------------------------------------------------------------------
def restated_coef(norm, max_norm):
    """optim.cu's coefficient in numpy fp32: min(fl(fl(1 / fl(n + fl(1e-6))) * fl(max_norm)), 1), a NaN kept."""
    n = np.asarray(norm, np.float32)
    r = np.float32(1) / (n + np.float32(1e-6))
    c = r * np.float32(max_norm)
    return np.where(np.isnan(c) | (c <= 1), c, np.float32(1)).astype(np.float32)


def torch_coef(norm, max_norm):
    """The factor torch.nn.utils.clip_grads_with_norm_ applies, given the fp32 total norm: the clipped value of a
    gradient of ones."""
    p = torch.zeros(1, requires_grad=True)
    p.grad = torch.ones(1)
    torch.nn.utils.clip_grads_with_norm_([p], max_norm, torch.tensor(norm, dtype=torch.float32))
    return p.grad.numpy()[0]


def _sweep(max_norm, rng):
    m = np.float32(max_norm)
    near = [m, np.nextafter(m, np.float32(0)), np.nextafter(m, np.float32(np.inf)), m - np.float32(1e-6),
            np.nextafter(m - np.float32(1e-6), np.float32(0)), np.nextafter(m - np.float32(1e-6), np.float32(np.inf))]
    walk = [m * np.float32(1 + k * 2.0 ** -20) for k in range(-64, 65)]
    tiny = [0.0, np.float32(1e-45), np.float32(1e-40), np.float32(1.17e-38), np.float32(1e-7), np.float32(1e-6),
            np.float32(9.9e-7)]
    large = [np.float32(1e30), np.finfo(np.float32).max, np.float32(np.inf)]
    rnd = (10.0 ** rng.uniform(-12, 12, 1500)).astype(np.float32)
    return np.concatenate([np.array(near + walk + tiny + large, np.float32), rnd])


@pytest.mark.parametrize("max_norm", [1.0, 0.1, 5.0, 3.3, 1e-3, 250.0])
def test_restated_coefficient_equals_torch_clip(max_norm):
    rng = np.random.default_rng(int(max_norm * 1000))
    norms = _sweep(max_norm, rng)
    ours = restated_coef(norms, max_norm)
    want = np.array([torch_coef(float(n), max_norm) for n in norms], np.float32)
    assert np.array_equal(ours.view(np.int32), want.view(np.int32)), norms[ours.view(np.int32) != want.view(np.int32)]
    # the sweep reaches both sides of the clamp
    assert (ours == 1).any() and (ours < 1).any()
