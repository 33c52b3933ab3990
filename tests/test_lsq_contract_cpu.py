"""The fp64 / exact contract of the least-squares layer (tests/lsq_contract.py) checked without a GPU:
  * the restatement agrees with oracle/lsq_oracle.py: wls_forward (float64, both solvers), wls_backward_closed_form and
    float64 autograd through activate_and_mask + wls_forward, for all six activations;
  * the activation error table holds for any expf / log1pf within the math library's documented accuracy: results moved
    to the edge of 2 ulp / 1 ulp in either direction stay within e_a and e_phi;
  * a kernel-faithful fp32 emulation (row-separable forward sums in the kernel's order, the backward's per-pixel
    arithmetic) passes the gate on every coverage case with headroom, also with expf / log1pf at the edge of their
    bounds, and every fp64 mutation breaks it;
  * every coverage case is in the linear regime, and the coverage table reaches all 40 kernel instances, partial lane
    groups in both directions, nchunks = 1 and nchunks at its cap ceil(H / 8) -- through lf_lsq_plan;
  * lf_lsq_plan agrees with the Python restatement of the selection over a wide sweep of shapes;
  * every argument refusal of lf_lsq_fwd, lf_lsq_bwd and lf_lsq_plan returns before any launch, so no device is needed.
    The entry-point refusals pass host addresses as device pointers, so they run only where no device is present: there a
    refusal that regressed would fail with LF_ERR_CUDA instead of launching on host memory.
"""
import ctypes

import numpy as np
import pytest
import torch

import lsq_contract as lc
from oracle import lsq_oracle as lo


def _lib():
    from lanedetection_end2end_b200 import _capi
    return _capi.lib()


def _plan(c, bwd):
    rc, pl = lc.query_plan(bwd, c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"],
                           c["act"])
    assert rc == 0, rc
    return pl


def _small_case(act, order, solver, reg, seed):
    c = dict(name="oracle%d" % seed, dtype=lc.LF_F32, act=act, L=2, H=12, W=16, B=2, order=order, solver=solver,
             reg_ls=reg, mask_rows=3, grid="bev", yrow=True)
    return c, lc.case_operands(c, seed)


@pytest.mark.parametrize("solver", [0, 1])
@pytest.mark.parametrize("order", [0, 1, 2, 3, 4])
def test_forward_restatement_matches_the_oracle(order, solver):
    c, (o, xtab, ytab, yrow) = _small_case(1, order, solver, 1e-3, order)
    H, W = c["H"], c["W"]
    ref = lc.forward_reference(o.astype(np.float64), xtab, yrow, H, W, order, 3, 1, 1e-3, True, 1, lc.LF_F32)
    grid = torch.from_numpy(np.stack([xtab, 1.0 - ytab.astype(np.float64)], 1))
    m = lo.activate_and_mask(torch.from_numpy(o).double(), "square", 3)
    b, zi = lo.wls_forward(m, grid, order, 1.0, reg_ls=1e-3, skip_rows=3, use_cholesky=bool(solver))
    scale = np.abs(ref["beta"]).max(-1, keepdims=True)
    assert np.abs(b.numpy() - ref["beta"]).max() <= 1e-8 * scale.max()
    assert np.allclose(zi.numpy(), ref["zinv"], rtol=1e-6, atol=1e-9 * np.abs(ref["zinv"]).max())


@pytest.mark.parametrize("act", range(6), ids=lc.ACTS)
def test_backward_restatement_matches_closed_form_and_autograd(act):
    c, (o, xtab, ytab, yrow) = _small_case(act, 2, 0, 0.0, 10 + act)
    H, W, mr = c["H"], c["W"], 3
    o = (o * 4.0).astype(np.float32)
    o[..., 5, :3] = np.array([19.9, 20.0, 20.1], np.float32)          # both sides of the softplus threshold
    o64 = o.astype(np.float64)
    ref = lc.forward_reference(o64, xtab, yrow, H, W, 2, mr, act, 0.0, True, 1, lc.LF_F32)
    g = np.random.default_rng(act).standard_normal((2, 2, 3))
    mine, _ = lc.backward_reference(o64, xtab, yrow, H, W, 2, mr, act, ref["beta"], ref["zinv"], g, True, lc.LF_F32)
    grid = np.stack([xtab, 1.0 - ytab.astype(np.float64)], 1)
    closed = lo.wls_backward_closed_form(o64, grid, 2, ref["beta"], ref["zinv"], g, lc.ACTS[act], mr, 1.0)
    tol = 1e-9 * np.abs(closed).max()
    assert np.abs(mine - closed).max() <= tol
    ot = torch.from_numpy(o64).requires_grad_(True)
    b, _ = lo.wls_forward(lo.activate_and_mask(ot, lc.ACTS[act], mr), torch.from_numpy(grid), 2, 1.0, skip_rows=mr)
    (b * torch.from_numpy(g)).sum().backward()
    assert np.abs(mine - ot.grad.numpy()).max() <= 1e-7 * np.abs(closed).max()


EDGE_ULPS = [(-2, -1), (-2, 1), (2, -1), (2, 1)]        # (expf, log1pf) results at the edge of their documented bounds


@pytest.mark.parametrize("act", [4, 5], ids=["sigmoid", "softplus"])
def test_activation_table_covers_the_math_library_bounds(act):
    o = np.concatenate([np.linspace(-110, 110, 200001), [19.9, 20, 20.1, -88.7, -88.8, 88.7, -87.3, -103.9, 103.9]])
    o = o.astype(np.float32)
    o64 = o.astype(np.float64)
    a, phi = lc.act64(o64, act)
    ea, ephi = lc.act_err(o64, act)
    use = 0.0
    for ulps in EDGE_ULPS + [(None, None)]:
        for got, ref, bound in ((lc._act_f32(o, act, *ulps), a, ea), (lc._dact_f32(o, act, *ulps), phi, ephi)):
            err = np.abs(got.astype(np.float64) - ref)
            assert np.all(err <= bound), (ulps, float(np.max(err[err > 0] / bound[err > 0])))
            use = max(use, float(np.max(err[err > 0] / bound[err > 0])))
    assert use >= 0.5                                                   # the bound is reached, not just respected


def _ops(c):
    o, xtab, ytab, yrow = lc.case_operands(c)
    return o, xtab, ytab, yrow


@pytest.mark.parametrize("case", lc.COVERAGE, ids=[c[0] for c in lc.COVERAGE])
def test_emulation_passes_and_mutations_fail(case):
    c = lc.case_dict(case)
    o, xtab, ytab, yrow = _ops(c)
    H, W, d, mr, act, dt = c["H"], c["W"], c["order"], c["mask_rows"], c["act"], c["dtype"]
    pf, pb = _plan(c, 0), _plan(c, 1)
    o64 = o.astype(np.float64)
    yf = yrow if pf["rowsep"] else ytab
    args = (o64, xtab, yf, H, W, d, mr, act, c["reg_ls"], pf["rowsep"], pf["nchunks"], dt)
    ref = lc.forward_reference(*args)
    assert float(ref["rho"].max()) <= lc.RHO_MAX                      # in the linear regime: the gate means something
    if pf["rowsep"]:
        b, z = lc.emulate_forward_rowsep(o, xtab, yrow, H, W, d, mr, act, c["reg_ls"], dt)
        assert lc.forward_excess(b, z, ref) <= 0.5                     # >= 2x headroom
        if lc.ACTS[act] in ("sigmoid", "softplus"):
            for ulps in EDGE_ULPS:
                assert lc.forward_excess(*lc.emulate_forward_rowsep(o, xtab, yrow, H, W, d, mr, act, c["reg_ls"], dt, ulps),
                                         ref) <= 1.0, ulps
        got_b, got_z = b, z
    else:
        got_b, got_z = ref["beta"], ref["zinv"]
    for m in lc.forward_mutations(c, pf):
        r2 = lc.forward_reference(*args, mut=m)
        x = lc.forward_excess(got_b, got_z, dict(r2, bound_beta=ref["bound_beta"], bound_zinv=ref["bound_zinv"]))
        assert x > 1.0, (m, x)
    beta, zinv, g = lc.nonsymmetric_backward_inputs(c["B"], c["L"], d, float(np.abs(yrow).max()), 0)
    yb = yrow if pb["rowsep"] else ytab
    em = lc.emulate_backward(o, xtab, yb, H, W, d, mr, act, beta, zinv, g, pb["rowsep"])
    if dt == lc.LF_BF16:
        em = torch.from_numpy(em).bfloat16().float().numpy()
    em = em.astype(np.float64)
    bargs = (o64, xtab, yb, H, W, d, mr, act, beta, zinv, g, pb["rowsep"], dt, em)
    bref, bound = lc.backward_reference(*bargs)
    assert lc.excess(em, bref, bound) <= 1.0
    hu = lc.bf16_half_ulp(em) if dt == lc.LF_BF16 else 0.0
    assert lc.gate_use(em, bref, bound, hu) <= 0.5                      # >= 2x headroom beyond the bf16 rounding
    for m in lc.backward_mutations(c):
        r2, _ = lc.backward_reference(*bargs, mut=m)
        assert lc.excess(em, r2, bound) > 1.0, m
    if lc.ACTS[act] in ("sigmoid", "softplus"):
        for ulps in EDGE_ULPS:
            e2 = lc.emulate_backward(o, xtab, yb, H, W, d, mr, act, beta, zinv, g, pb["rowsep"], ulps)
            if dt == lc.LF_BF16:
                e2 = torch.from_numpy(e2).bfloat16().float().numpy()
            e2 = e2.astype(np.float64)
            _, b2 = lc.backward_reference(*bargs[:-1], e2)
            assert lc.excess(e2, bref, b2) <= 1.0, ulps


def test_coverage_reaches_every_instance_and_the_chunk_edges():
    seen, partial, nch_one = set(), set(), set()
    for case in lc.COVERAGE:
        c = lc.case_dict(case)
        for b in (0, 1):
            pl = _plan(c, b)
            seen.add(lc.instance(b, c["dtype"], pl))
            if pl["rowsep"] and c["L"] % pl["nl"]:
                partial.add(b)
            if pl["nchunks"] == 1:
                nch_one.add(b)
    assert seen == lc.all_instances() and len(seen) == 40
    assert partial == {0, 1} and nch_one == {0, 1}
    # the cap ceil(H / 8) on a case where it is more than one chunk: one image, one lane, 256 unmasked rows -- the score
    # grows with the chunk count up to the cap for any device of 16 SMs or more
    c = lc.case_dict(next(k for k in lc.COVERAGE if k[0] == "sq_f32_nl1_cap"))
    for b in (0, 1):
        assert _plan(c, b)["nchunks"] == (c["H"] + 7) // 8 == 32


def test_plan_matches_the_restatement():
    rng = np.random.default_rng(0)
    Bs = [1, 2, 3, 5, 8, 16, 31, 32, 33, 64, 100, 128, 1000, 4096, 16384, 16385, 65535, 65536]
    Ls = list(range(1, 12)) + [16, 17]
    Hs = [1, 2, 7, 8, 9, 16, 17, 64, 255, 256, 320, 1000]
    Ws = [1, 4, 8, 12, 98, 100, 132, 136, 512, 640]
    for _ in range(20000):
        B, L, H, W = (int(rng.choice(v)) for v in (Bs, Ls, Hs, Ws))
        mr = int(rng.choice([0, 1, H // 3, H - 1, H, H + 1, -1]))
        args = (int(rng.integers(0, 2)), int(rng.integers(0, 2)), bool(rng.integers(0, 2)), bool(rng.integers(0, 2)),
                B, L, H, W, int(rng.integers(0, 6)), mr, int(rng.integers(0, 6)))
        rc, pl = lc.query_plan(*args)
        rc2, pl2 = lc.plan_py(*args)
        assert (rc, pl) == (rc2, pl2), (args, rc, pl, rc2, pl2)


def test_plan_reports_alignment_and_refuses_like_the_entry_points():
    assert lc.query_plan(0, 0, True, True, 2, 2, 16, 64, 2, 3, 1)[1]["align"] == 16
    assert lc.query_plan(0, 0, False, True, 2, 2, 16, 64, 2, 3, 1)[1]["align"] == 0
    assert lc.query_plan(0, 0, False, False, 2, 2, 16, 64, 2, 3, 1)[0] == lc.INVALID
    assert lc.query_plan(0, 0, True, False, 2, 2, 16, 62, 2, 3, 1)[0] == lc.INVALID     # W % 4 != 0, no ytab
    assert lc.query_plan(0, 0, True, True, 16385, 1, 16, 64, 2, 3, 1)[0] == lc.UNSUPPORTED
    assert lc.query_plan(1, 0, True, True, 16385, 1, 16, 64, 2, 3, 1)[0] == 0            # the backward has no tickets
    info = (ctypes.c_int * 7)()
    assert _lib().lf_lsq_plan(2, 0, 1, 1, 2, 2, 16, 64, 2, 3, 1, info) == lc.INVALID
    assert _lib().lf_lsq_plan(0, 0, 1, 1, 2, 2, 16, 64, 2, 3, 1, None) == lc.INVALID


# ---------------------------------------------------------------------------------------------------------------------
# argument refusals of the entry points (no launch happens: no device needed)
# ---------------------------------------------------------------------------------------------------------------------
class _Bufs:
    """Host buffers standing in for device pointers: every call below is refused before anything reads them."""

    def __init__(self):
        self.mem = np.zeros(1 << 16, np.float64)
        base = self.mem.ctypes.data
        self.p = lambda k: base + 64 * k + (64 - base % 64) % 64


def _fwd(b, **kw):
    a = dict(o=b.p(0), dt=0, xtab=b.p(1), ytab=b.p(2), yrow=b.p(3), B=2, L=2, H=16, W=64, order=2, mr=3, act=1, reg=0.0,
             solver=0, beta=b.p(4), zinv=b.p(5), masked=b.p(6), status=b.p(7), ws=b.p(8), wsb=None)
    a.update(kw)
    if a["wsb"] is None:
        a["wsb"] = _lib().lf_lsq_workspace_bytes(a["B"], a["L"], a["H"], a["W"], a["order"])
    return _lib().lf_lsq_fwd(a["o"], a["dt"], a["xtab"], a["ytab"], a["yrow"], a["B"], a["L"], a["H"], a["W"], a["order"],
                             a["mr"], a["act"], a["reg"], a["solver"], a["beta"], a["zinv"], a["masked"], a["status"],
                             a["ws"], a["wsb"], None)


def _bwd(b, **kw):
    a = dict(o=b.p(0), dt=0, xtab=b.p(1), ytab=b.p(2), yrow=b.p(3), B=2, L=2, H=16, W=64, order=2, mr=3, act=1,
             beta=b.p(4), zinv=b.p(5), g=b.p(6), d_o=b.p(7))
    a.update(kw)
    return _lib().lf_lsq_bwd(a["o"], a["dt"], a["xtab"], a["ytab"], a["yrow"], a["B"], a["L"], a["H"], a["W"], a["order"],
                             a["mr"], a["act"], a["beta"], a["zinv"], a["g"], a["d_o"], None)


no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="host addresses as device pointers: CPU-only machines")

COMMON_BAD = [dict(o=None), dict(xtab=None), dict(ytab=None, yrow=None), dict(B=0), dict(L=0), dict(H=0), dict(W=0),
              dict(B=-1), dict(B=65536), dict(L=65536), dict(order=5), dict(order=-1), dict(mr=-1), dict(mr=17),
              dict(act=6), dict(act=-1), dict(dt=2), dict(ytab=None, W=62), dict(ytab=None, dt=1, W=68)]


@no_device
@pytest.mark.parametrize("bad", COMMON_BAD + [dict(beta=None), dict(zinv=None), dict(status=None), dict(ws=None),
                                              dict(solver=2), dict(solver=-1)])
def test_forward_refuses_bad_arguments(bad):
    assert _fwd(_Bufs(), **bad) == lc.INVALID


@no_device
@pytest.mark.parametrize("bad", COMMON_BAD + [dict(beta=None), dict(zinv=None), dict(g=None), dict(d_o=None)])
def test_backward_refuses_bad_arguments(bad):
    assert _bwd(_Bufs(), **bad) == lc.INVALID


@no_device
def test_forward_refuses_a_short_workspace_and_too_many_systems():
    b = _Bufs()
    need = _lib().lf_lsq_workspace_bytes(2, 2, 16, 64, 2)
    assert _fwd(b, wsb=need - 1) == -3
    assert _fwd(b, B=16385, L=1, wsb=1 << 40) == lc.UNSUPPORTED
    assert _fwd(b, B=128, L=129, wsb=1 << 40) == lc.UNSUPPORTED


@no_device
@pytest.mark.parametrize("which", ["o", "xtab", "masked"])
def test_row_separable_forward_refuses_misaligned_pointers(which):
    b = _Bufs()
    assert _fwd(b, **{which: b.p(9) + 4}) == lc.INVALID


@no_device
@pytest.mark.parametrize("which", ["o", "xtab", "d_o"])
def test_row_separable_backward_refuses_misaligned_pointers(which):
    b = _Bufs()
    assert _bwd(b, **{which: b.p(9) + 4}) == lc.INVALID
