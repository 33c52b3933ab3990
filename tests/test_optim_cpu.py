"""The fused optimizer update without a GPU: the C ABI (ctypes mirrors of LfOptimSeg / LfOptimHyper / LfOptimState against
the C compiler's layout of the header, the prototype against its declaration and the library's exports), a torch-CPU
restatement of the kernel's op order (csrc/optim.cu) against torch.optim at the GPU test's gates, and the torch-format
state_dict conversion of optim.FusedOptimizer."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

import optim_cases as oc
from conftest import ROOT

HEADER_DIR = os.path.join(ROOT, "include")


def test_optim_structs_match_the_header(tmp_path):
    from lanedetection_end2end_b200 import _capi
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("clang")
    if cc is None:
        pytest.skip("no C compiler to lay out the header structs")
    structs = {"LfOptimSeg": _capi.LfOptimSeg, "LfOptimHyper": _capi.LfOptimHyper, "LfOptimState": _capi.LfOptimState}
    body = ""
    for name, cls in structs.items():
        body += '    printf("%%zu\\n", sizeof(%s));\n' % name
        body += "".join('    printf("%%zu\\n", offsetof(%s, %s));\n' % (name, f[0]) for f in cls._fields_)
    body += '    printf("%d %d %d %d\\n", LF_OPTIM_ADAM, LF_OPTIM_SGD, LF_OPTIM_RMSPROP, LF_OPTIM_CHUNK);\n'
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lanefit_b200.h"\nint main(void) {\n' + body +
                   "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", HEADER_DIR, str(src), "-o", str(exe)], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    want = []
    for cls in structs.values():
        want.append(str(ctypes.sizeof(cls)))
        want += [str(getattr(cls, f[0]).offset) for f in cls._fields_]
    assert lines[:len(want)] == want
    assert lines[len(want)] == "%d %d %d %d" % (_capi.OPTIM_ADAM, _capi.OPTIM_SGD, _capi.OPTIM_RMSPROP, _capi.OPTIM_CHUNK)


def test_optim_prototype_matches_declaration_and_export():
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(HEADER_DIR, "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+lf_optim_step\s*\((.*?)\);", hdr, re.S)
    assert decl
    res, args = _capi.PROTOTYPES["lf_optim_step"]
    assert res is ctypes.c_int and len(args) == len(decl.group(1).split(","))
    assert hasattr(_capi.lib(), "lf_optim_step")


# ---------------------------------------------------------------------------------------------------------------------
# restatement of optim_kernel: scalars in fp64 rounded to fp32, one fp32 rounding per elementwise operation
# ---------------------------------------------------------------------------------------------------------------------
def _f(x):
    return torch.tensor(x, dtype=torch.float32)


def _fma(a, b, c):
    """fp32 fused multiply-add: the fp32 product is exact in fp64, so one fp64 add and the fp32 rounding give the single
    rounding of __fmaf_rn (up to a double-rounding tie, which the gates do not see)."""
    return (a.double() * b.double() + c.double()).float()


def restated_step(kind, hyper, t_before, p, g, s0, s1):
    """One update of one tensor (in place), in optim.cu's operation order; hyper = LfOptimHyper values."""
    lr, b1, b2, eps, wd, mu = hyper
    if wd != 0:
        g = _fma(_f(wd), p, g)
    if kind == "adam":
        t = float(t_before + 1)
        w = 1.0 - b1
        assert abs(w) < 0.5
        s0.copy_(_fma(_f(w), g - s0, s0))
        s1.copy_(_fma(_f(1.0 - b2), g * g, s1 * _f(b2)))
        denom = torch.sqrt(s1) / _f(math.sqrt(1.0 - b2 ** t)) + _f(eps)
        p.copy_(_fma(-_f(lr / (1.0 - b1 ** t)), s0 / denom, p))
    elif kind == "sgd":
        s0.copy_(g if t_before == 0 else s0 * _f(mu) + g)
        p.copy_(_fma(-_f(lr), s0, p))
    else:
        s0.copy_(_fma(_f(1.0 - b2), g * g, s0 * _f(b2)))
        avg = torch.sqrt(s0) + _f(eps)
        s1.copy_(s1 * _f(mu) + g / avg)
        p.copy_(_fma(-_f(lr), s1, p))


def restated_run(kind, wd, params, grads, steps):
    hyper = {"adam": (oc.LR["adam"], 0.9, 0.999, 1e-8, wd, 0.0), "sgd": (oc.LR["sgd"], 0.0, 0.0, 0.0, wd, 0.9),
             "rmsprop": (oc.LR["rmsprop"], 0.0, 0.99, 1e-8, wd, 0.9)}[kind]
    ps = [p.clone() for p in params]
    st = [(torch.zeros_like(p), torch.zeros_like(p)) for p in ps]
    for t in range(steps):
        for i, (p, g) in enumerate(zip(ps, grads[t])):
            if g is not None:
                restated_step(kind, hyper, t, p, g, *st[i])
    out = {}
    for i, p in enumerate(ps):
        out["p%d" % i] = p
        if i != oc.NONE_GRAD:
            for k, s in zip(oc.STATE_NAMES[kind], st[i]):
                out["p%d.%s" % (i, k)] = s
    return out


@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_restated_kernel_meets_the_gates_against_torch_optim(kind, wd):
    params, grads = oc.make_params(), oc.make_grads()
    ours = restated_run(kind, wd, params, grads, oc.STEPS)
    p32, o32 = oc.torch_run(kind, wd, params, grads, torch.float32, "cpu", oc.STEPS)
    p64, o64 = oc.torch_run(kind, wd, params, grads, torch.float64, "cpu", oc.STEPS)
    t32, t64 = oc.tensors_of(p32, o32, kind), oc.tensors_of(p64, o64, kind)
    assert set(ours) == set(t64)
    for name, x64 in t64.items():
        e_ours, e_t32 = oc.rel_err(ours[name], x64), oc.rel_err(t32[name], x64)
        assert e_ours <= 2 * e_t32 + 1e-7, (name, e_ours, e_t32)
    # one step.  The GPU test holds every element to 2 ulp of torch's CUDA result, whose kernels group the operations as
    # optim.cu does; torch's CPU kernels group some differently (addcdiv as (s*a)/b, no fused multiply-add), which moves
    # a parameter that nearly cancels by many of its own ulp.  Here: state tensors within 2 ulp, and each parameter
    # within 2 ulp of itself plus 4 ulp of torch's update p_new - p_old.
    one = restated_run(kind, wd, params, grads, 1)
    q32, r32 = oc.torch_run(kind, wd, params, grads, torch.float32, "cpu", 1)
    for name, x in oc.tensors_of(q32, r32, kind).items():
        if "." in name:
            assert oc.ulp_distance(one[name], x) <= 2, name
        else:
            ulp = (torch.nextafter(x.abs(), torch.tensor(float("inf"))) - x.abs()).double()
            d_torch = x.double() - params[int(name[1:])].double()
            assert bool(((one[name].double() - x.double()).abs() <= 2 * ulp + 4 * 2.0 ** -24 * d_torch.abs()).all()), name


# ---------------------------------------------------------------------------------------------------------------------
# state_dict conversion (a CPU FusedOptimizer can load and save; only its update needs the GPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_state_dict_round_trips_torch_format(kind):
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), oc.make_grads(steps=3)
    pt, ot = oc.torch_run(kind, 1e-4, params, grads, torch.float32, "cpu", 3)
    sd_t = ot.state_dict()
    ours = FusedOptimizer([p.clone() for p in pt], kind, oc.LR[kind], 1e-4)
    # before any update: torch's empty state, same param_groups
    fresh_t = oc.KINDS[kind][0]([p.clone() for p in pt], lr=oc.LR[kind], weight_decay=1e-4, **oc.KINDS[kind][1]).state_dict()
    assert ours.state_dict() == fresh_t
    ours.load_state_dict(sd_t)
    if kind != "sgd":
        assert ours.step_count == 3
    sd_o = ours.state_dict()
    assert list(sd_o["param_groups"][0]) == list(sd_t["param_groups"][0])
    assert sd_o["param_groups"] == sd_t["param_groups"]
    assert set(sd_o["state"]) == set(sd_t["state"]) and oc.NONE_GRAD not in sd_o["state"]
    for i, st in sd_t["state"].items():
        assert list(sd_o["state"][i]) == list(st)
        for k, v in st.items():
            assert sd_o["state"][i][k].dtype == v.dtype and sd_o["state"][i][k].device == v.device
            assert torch.equal(sd_o["state"][i][k], v), (i, k)
    # and back into torch.optim
    back = oc.KINDS[kind][0]([p.clone() for p in pt], lr=oc.LR[kind], weight_decay=1e-4, **oc.KINDS[kind][1])
    back.load_state_dict(sd_o)
    assert back.state_dict()["param_groups"] == sd_t["param_groups"]


def test_load_rejects_per_parameter_steps_and_unsupported_flags():
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), oc.make_grads(steps=2)
    pt, ot = oc.torch_run("adam", 0.0, params, grads, torch.float32, "cpu", 2)
    sd = ot.state_dict()
    sd["state"][3]["step"] = torch.tensor(7.0)
    ours = FusedOptimizer([p.clone() for p in pt], "adam", 1e-3, 0.0)
    with pytest.raises(ValueError, match="parameter 3 has step 7"):
        ours.load_state_dict(sd)
    _, oa = oc.torch_run("adam", 0.0, params, grads, torch.float32, "cpu", 1, amsgrad=True)
    with pytest.raises(ValueError, match="amsgrad"):
        ours.load_state_dict(oa.state_dict())
    with pytest.raises(ValueError, match="one parameter group"):
        FusedOptimizer([{"params": [pt[0]]}, {"params": [pt[1]]}], "adam", 1e-3, 0.0)
    with pytest.raises(ValueError):
        FusedOptimizer([pt[0]], "adamw", 1e-3, 0.0)


def test_define_optim_default_is_unchanged(monkeypatch):
    from lanedetection_end2end_b200.Networks.utils import define_optim
    from lanedetection_end2end_b200.optim import FusedOptimizer
    p = [torch.zeros(4, requires_grad=True)]
    monkeypatch.delenv("LANEFIT_FUSED_OPTIM", raising=False)
    assert type(define_optim("adam", p, 1e-3, 0)) is torch.optim.Adam
    assert type(define_optim("rmsprop", p, 1e-3, 0, fused=False)) is torch.optim.RMSprop
    monkeypatch.setenv("LANEFIT_FUSED_OPTIM", "1")
    o = define_optim("sgd", p, 1e-3, 0)
    assert isinstance(o, FusedOptimizer) and o.kind == "sgd" and o.param_groups[0]["momentum"] == 0.9
    with pytest.raises(KeyError):
        define_optim("lbfgs", p, 1e-3, 0)


def test_load_copies_into_existing_state_tensors():
    """A graph captured before a load reads the state tensors by address: loading must write into them, not replace them."""
    from lanedetection_end2end_b200.optim import FusedOptimizer
    params, grads = oc.make_params(), oc.make_grads(steps=4)
    _, o2 = oc.torch_run("rmsprop", 0.0, params, grads, torch.float32, "cpu", 2)
    _, o4 = oc.torch_run("rmsprop", 0.0, params, grads, torch.float32, "cpu", 4)
    ours = FusedOptimizer([p.clone() for p in params], "rmsprop", oc.LR["rmsprop"], 0.0)
    sd2 = o2.state_dict()
    ours.load_state_dict(sd2)
    st = {i: [ours.state[p][k] for k in oc.STATE_NAMES["rmsprop"]] for i, p in enumerate(ours.param_groups[0]["params"])
          if ours.state[p]}
    for i, ts in st.items():       # independent of the caller's tensors
        assert all(t.data_ptr() != sd2["state"][i][k].data_ptr() for t, k in zip(ts, oc.STATE_NAMES["rmsprop"]))
    ours.load_state_dict(o4.state_dict())
    assert ours.step_count == 4
    for i, p in enumerate(ours.param_groups[0]["params"]):
        if i in st:
            for t, k in zip(st[i], oc.STATE_NAMES["rmsprop"]):
                assert ours.state[p][k] is t and torch.equal(t, o4.state_dict()["state"][i][k])
    # a state dict without state (before any update) zeroes the same tensors
    ours.load_state_dict(oc.KINDS["rmsprop"][0]([p.clone() for p in params], lr=oc.LR["rmsprop"], momentum=0.9).state_dict())
    assert ours.step_count == 0 and ours.state_dict()["state"] == {}
    p0 = ours.param_groups[0]["params"][0]
    assert ours.state[p0]["square_avg"] is st[0][0] and not bool(st[0][0].any())


def _gloo_worker(rank, port, words, q):
    import torch.distributed as dist
    from lanedetection_end2end_b200.ddp import any_rank_nonzero
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    out = torch.zeros(1, dtype=torch.int32)
    res = [int(any_rank_nonzero(torch.tensor([w[rank]], dtype=torch.int32), out)[0]) for w in words]
    q.put((rank, res))
    dist.destroy_process_group()


def test_status_word_is_reduced_over_the_ranks():
    """The guarded update under data parallelism reads max over the ranks of the status word (ddp.any_rank_nonzero)."""
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    words = [(0, 0), (0, 1), (4, 0), (2, 5)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, port, words, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0] == res[1] == [0, 1, 4, 5]
