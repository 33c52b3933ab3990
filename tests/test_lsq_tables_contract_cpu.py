"""The contract of the least-squares layer's table entry points (tests/lsq_tables_contract.py) checked without a GPU:
  * the grid-gradient formula of the header is the float64 autograd gradient of the restated fit with respect to each
    row's (alpha, gamma, y'), with reg_ls != 0, a keep map and masked rows;
  * kernel-order emulations -- fp32 row sums (the kernel's single accumulator and UNR split ones), the fp64 grid
    gradient, the fits on per-image tables and the prefix fits -- pass their gates with 2x headroom on every coverage
    case, and every mutation breaks them;
  * the coverage table reaches all 338 instances behind the table entry points, through lf_lsq_plan, and the shapes the
    kernels' edges need;
  * the restated instance selection agrees with the one built from lf_lsq_plan.
"""
import numpy as np
import pytest
import torch

import lsq_contract as lc
import lsq_tables_contract as tc

EDGE_ULPS = [(-2, -1), (-2, 1), (2, -1), (2, 1)]


def _bf16(v):
    return torch.from_numpy(np.ascontiguousarray(v, np.float32)).bfloat16().float().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the header's formula against autograd
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [0, 1, 2, 3, 4])
def test_grid_grad_formula_is_the_autograd_gradient(order):
    """dL/d(alpha_r, gamma_r, y'_r) of L = g . beta, beta the fit on x[r][c] = alpha_r c + gamma_r, y_r = 1 - y'_r, in
    float64 autograd, against the header's formula (grid_grad_reference, exact) on fp64 row sums."""
    B, L, H, W, mr, reg, act = 2, 2, 12, 16, 3, 0.25, 5
    rng = np.random.default_rng(order)
    o = rng.standard_normal((B, L, H, W)) * 1.5 + 0.3
    keep = tc.keep_map(H, W, order)
    alpha = torch.tensor(0.5 + 0.1 * rng.standard_normal(H), dtype=torch.float64, requires_grad=True)
    gamma = torch.tensor(rng.standard_normal(H), dtype=torch.float64, requires_grad=True)
    yp = torch.tensor(np.linspace(0.1, 0.9, H) + 0.01 * rng.standard_normal(H), dtype=torch.float64, requires_grad=True)
    g = rng.standard_normal((B, L, order + 1))
    a, _ = lc.act64(tc.zeroed(o, keep, act), act)
    w = torch.from_numpy(a * a)[:, :, mr:]                                             # [B, L, R, W]
    cols = torch.arange(W, dtype=torch.float64)
    x = alpha[mr:, None] * cols + gamma[mr:, None]
    y = 1.0 - yp[mr:]
    n = order + 1
    phi = torch.stack([y ** (order - i) for i in range(n)], -1)                         # [R, n]
    Ar, Br = w.sum(-1), (w * x).sum(-1)
    Z = torch.einsum("blr,ri,rj->blij", Ar, phi, phi) + reg * torch.eye(n, dtype=torch.float64)
    X = torch.einsum("blr,ri->bli", Br, phi)
    beta = torch.linalg.solve(Z, X)
    (beta * torch.from_numpy(g)).sum().backward()
    want = torch.stack([alpha.grad, gamma.grad, yp.grad], -1).numpy()
    # the formula, on fp64 row sums of the same maps and tables
    xt = (alpha.detach()[:, None] * cols + gamma.detach()[:, None]).numpy().reshape(-1)
    rs_ref, _ = tc.rowsums_reference(o, xt, H, W, mr, act, lc.LF_F32, keep)
    rs = np.zeros((B, L, H, 3))
    rs[:, :, mr:] = rs_ref
    zinv = torch.linalg.inv(Z).detach().numpy()
    yrow = (1.0 - yp.detach()).numpy()
    got, _ = tc.grid_grad_reference(rs, yrow, beta.detach().numpy(), zinv, g, B, L, H, order, mr, False)
    assert not got[:mr].any() and not want[:mr].any()
    scale = np.abs(want).max(0)
    assert (np.abs(got - want) <= 1e-9 * scale).all(), np.abs(got - want).max(0) / scale


# ---------------------------------------------------------------------------------------------------------------------
# emulations and mutations on every coverage case
# ---------------------------------------------------------------------------------------------------------------------
def _plans(c):
    args = (c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"], c["act"])
    return lc.plan_py(0, *args, sms=132)[1], lc.plan_py(1, *args, sms=132)[1]


def _rows_full(rs, H, mr):
    B, L = rs.shape[:2]
    out = np.full((B, L, H, 3), np.nan)
    out[:, :, mr:] = rs
    return out


def _check_rowsums(c, o, xtab, keep):
    H, W, mr, act, dt = c["H"], c["W"], c["mask_rows"], c["act"], c["dtype"]
    o64 = o.astype(np.float64)
    ref, bound = tc.rowsums_reference(o64, xtab, H, W, mr, act, dt, keep)
    unr = 4 if c["L"] <= 2 else 2
    V = 8 if dt == lc.LF_BF16 else 4
    steps = -(-(W // V) // 32)
    # split over UNR accumulators, a term passes ceil(steps / UNR) step adds and min(UNR, steps) - 1 adds of the partials
    assert tc.nadd(W, dt) == V + steps + 5 >= V + -(-steps // unr) + min(unr, steps) - 1 + 5
    em = tc.emulate_rowsums(o, xtab, H, W, mr, act, dt, keep)
    for split in (1, unr):
        e = tc.emulate_rowsums(o, xtab, H, W, mr, act, dt, keep, split=split)
        assert lc.excess(e, ref, bound) <= 0.5, split
    if lc.ACTS[act] in ("sigmoid", "softplus"):
        for ulps in EDGE_ULPS:
            assert lc.excess(tc.emulate_rowsums(o, xtab, H, W, mr, act, dt, keep, ulps=ulps), ref, bound) <= 1.0, ulps
    if mr < H:
        r2, _ = tc.rowsums_reference(o64, xtab, H, W, mr, act, dt, keep, mut=("col_shift",))
        assert lc.excess(em, r2, bound) > 1.0
    return em


def _check_grid_grad(c, rs, yv, o, xv, per_image, keep):
    B, L, H, W, d, mr = c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"]
    beta, zinv, g = lc.nonsymmetric_backward_inputs(B, L, d, float(np.abs(yv).max()), 3)
    args = (_rows_full(rs, H, mr), yv, beta, zinv, g, B, L, H, d, mr, per_image)
    ref, bound = tc.grid_grad_reference(*args)
    em = tc.emulate_grid_grad(*args)
    assert lc.excess(em, ref, bound) <= 0.5
    muts = tc.grid_grad_mutations(c, per_image)
    below = tc.row_below_mask(o, xv, H, W, mr, c["act"], c["dtype"], keep) if mr > 0 else None
    for m in muts:
        assert lc.excess(em, tc.emulate_grid_grad(*args, mut=m, below=below), bound) > 1.0, m


@pytest.mark.parametrize("case", tc.COVERAGE, ids=[c[0] for c in tc.COVERAGE])
def test_emulation_passes_and_mutations_fail(case):
    c = tc.case_dict(case)
    o, xtab, ytab, yrow, xs, ys, keep = tc.case_operands(c)
    B, L, H, W, d, mr, act, dt = c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"], c["act"], c["dtype"]
    pf, pb = _plans(c)
    ol = np.ascontiguousarray(o[:, :L])
    o64 = ol.astype(np.float64)
    # prefix fit: the plain fit of o[:, :L]; the stride-L read is outside the gate
    yf = yrow if pf["rowsep"] else ytab
    args = (o64, xtab, yf, H, W, d, mr, act, c["reg_ls"], pf["rowsep"], pf["nchunks"], dt)
    ref = lc.forward_reference(*args)
    assert float(ref["rho"].max()) <= lc.RHO_MAX
    if pf["rowsep"]:
        got = lc.emulate_forward_rowsep(ol, xtab, yrow, H, W, d, mr, act, c["reg_ls"], dt)
        assert lc.forward_excess(*got, ref) <= 0.5
    else:
        got = ref["beta"], ref["zinv"]
    bounds = dict(bound_beta=ref["bound_beta"], bound_zinv=ref["bound_zinv"])
    if mr < H:
        r2 = lc.forward_reference(tc.stride_l_view(o, L).astype(np.float64), *args[1:])
        assert lc.forward_excess(*got, dict(r2, **bounds)) > 1.0
    beta, zinv, g = lc.nonsymmetric_backward_inputs(B, L, d, float(np.abs(yrow).max()), 0)
    yb = yrow if pb["rowsep"] else ytab
    em = lc.emulate_backward(ol, xtab, yb, H, W, d, mr, act, beta, zinv, g, pb["rowsep"])
    em = (_bf16(em) if dt == lc.LF_BF16 else em).astype(np.float64)
    bargs = (o64, xtab, yb, H, W, d, mr, act, beta, zinv, g, pb["rowsep"], dt, em)
    bref, bbound = lc.backward_reference(*bargs)
    assert lc.gate_use(em, bref, bbound, lc.bf16_half_ulp(em) if dt == lc.LF_BF16 else 0.0) <= 0.5
    if mr < H:
        r2, _ = lc.backward_reference(tc.stride_l_view(o, L).astype(np.float64), *bargs[1:])
        assert lc.excess(em, r2, bbound) > 1.0
    if not pf["rowsep"]:
        return
    # row sums, shared tables, with and without the keep map; the grid gradient on the emulated row sums
    for km in (None, keep):
        rs = _check_rowsums(c, ol, xtab, km)
        _check_grid_grad(c, rs, yrow, o64, xtab, False, km)
    # per-image tables: the row sums and grid gradient per image, the fit on each image's tables
    rs = np.concatenate([_check_rowsums(c, ol[b:b + 1], xs[b], None) for b in range(B)])
    _check_grid_grad(c, rs, ys, o64, xs, True, None)
    pref = tc.per_image_forward_reference(o64, xs, ys, H, W, d, mr, act, c["reg_ls"], pf["nchunks"], dt)
    assert float(pref["rho"].max()) <= lc.RHO_MAX
    pgot = tc.emulate_per_image_forward(ol, xs, ys, H, W, d, mr, act, c["reg_ls"], dt)
    assert lc.forward_excess(*pgot, pref) <= 0.5
    pem = tc.emulate_per_image_backward(ol, xs, ys, H, W, d, mr, act, beta, zinv, g)
    pem = (_bf16(pem) if dt == lc.LF_BF16 else pem).astype(np.float64)
    pbref, pbound = tc.per_image_backward_reference(o64, xs, ys, H, W, d, mr, act, beta, zinv, g, dt, pem)
    assert lc.gate_use(pem, pbref, pbound, lc.bf16_half_ulp(pem) if dt == lc.LF_BF16 else 0.0) <= 0.5
    if mr < H:
        m = ("image0",)
        r2 = tc.per_image_forward_reference(o64, xs, ys, H, W, d, mr, act, c["reg_ls"], pf["nchunks"], dt, mut=m)
        assert lc.forward_excess(*pgot, dict(r2, bound_beta=pref["bound_beta"], bound_zinv=pref["bound_zinv"])) > 1.0
        r2, _ = tc.per_image_backward_reference(o64, xs, ys, H, W, d, mr, act, beta, zinv, g, dt, pem, mut=m)
        assert lc.excess(pem, r2, pbound) > 1.0


# ---------------------------------------------------------------------------------------------------------------------
# coverage and the instance selection
# ---------------------------------------------------------------------------------------------------------------------
def test_coverage_reaches_every_instance_and_edge():
    seen = set()
    cases = [tc.case_dict(k) for k in tc.COVERAGE]
    nch = {0: set(), 1: set()}
    for c in cases:
        for call in tc.case_calls(c):
            rc, inst = tc.case_instance(c, call, plan=lc.query_plan)
            assert rc == 0, (c["name"], call)
            assert inst == tc.case_instance(c, call)[1], (c["name"], call)
            seen.add(inst)
        for b in (0, 1):
            pl = lc.query_plan(b, c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"],
                               c["mask_rows"], c["act"])[1]
            if pl["rowsep"]:
                nch[b].add("one" if pl["nchunks"] == 1 else "cap" if pl["nchunks"] == (c["H"] + 7) // 8 else "mid")
    assert seen == tc.all_instances() and len(seen) == 338
    assert nch[0] >= {"one", "cap"} and nch[1] >= {"one", "cap"}
    assert {c["order"] for c in cases} == {0, 1, 2, 3, 4}
    assert {c["act"] for c in cases} == set(range(6))
    assert {5, 6, 7} <= {c["L"] for c in cases}
    assert all(c["L"] < c["Lmap"] and c["B"] >= 3 for c in cases)
    assert max(c["Lmap"] for c in cases) >= 9
    assert {1, 127, 129, 320} <= {c["H"] for c in cases}
    assert {"zero", "all", "inside"} == {"zero" if c["mask_rows"] == 0 else "all" if c["mask_rows"] == c["H"] else
                                         "inside" for c in cases}
    widths = {(c["dtype"], c["W"]) for c in cases if c["yrow"]}
    assert {(lc.LF_F32, 4), (lc.LF_BF16, 8), (lc.LF_F32, 132), (lc.LF_BF16, 136)} <= widths
    # softplus and sigmoid carry the planted values of lc.case_operands on the fitted lanes
    for c in cases:
        if lc.ACTS[c["act"]] in ("sigmoid", "softplus") and c["W"] >= 4:
            o = tc.case_operands(c)[0]
            planted = [19.9, 20.0, 20.1] if lc.ACTS[c["act"]] == "softplus" else [30.0, -30.0, 100.0, -100.0]
            planted = _bf16(planted) if c["dtype"] == lc.LF_BF16 else np.float32(planted)
            assert (o[..., :len(planted)] == planted).all(), c["name"]


def test_instance_selection_matches_the_plan_query():
    """launched() from the restated plan and from lf_lsq_plan: the same instance or the same refusal, for every table
    entry point over a sweep of shapes."""
    rng = np.random.default_rng(0)
    entries = sorted({tc.entry_name(b, pi, rs, kp, ln) for b in (0, 1) for pi in (False, True) for rs in (False, True)
                      for kp in (False, True) for ln in (False, True)} | {"lf_lsq_grid_grad", "lf_lsq_grid_grad_per_image"})
    sms = lc.device_sms()
    for _ in range(6000):
        entry = entries[int(rng.integers(len(entries)))]
        L = int(rng.choice([1, 2, 3, 4, 5, 6, 7, 8, 9, 17]))
        args = (entry, int(rng.integers(0, 2)), int(rng.integers(0, 6)), int(rng.choice([1, 2, 3, 8, 100, 16385])), L,
                L + int(rng.choice([-1, 0, 0, 1, 5])), int(rng.choice([1, 7, 127, 129, 320])),
                int(rng.choice([4, 8, 12, 98, 100, 132, 136, 640])), int(rng.integers(0, 5)), int(rng.choice([0, 1, 52])),
                bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), bool(rng.integers(0, 2)))
        want = tc.launched(*args, plan=lambda *a: lc.plan_py(*a, sms=sms))
        assert tc.launched(*args, plan=lc.query_plan) == want, args
