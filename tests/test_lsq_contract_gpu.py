"""lf_lsq_fwd and lf_lsq_bwd driven directly through their C entry points, entry by entry against the fp64 / exact
restatement of their contract (tests/lsq_contract.py).

Every case builds xtab, ytab and yrow by hand (ytab exactly constant along rows) and launches into sentinel-filled
buffers with guard regions on both sides of beta, zinv, masked and d_o, and a workspace of exactly
lf_lsq_workspace_bytes bytes between guard bytes.  Every entry must be written, every guard must stay intact and the
ticket region must be zero after every launch.  beta and Z^-1 are held to the forward gate, `masked` to torch-CPU float32
(bit for bit, or within the activation's error for sigmoid / softplus; +0.0 in the masked rows), d_o -- from a
hand-built beta, non-symmetric Z^-1 and g -- to the backward gate.  Cases:
  * coverage: one launch per kernel instance and direction (lsq_contract.COVERAGE), asserted through lf_lsq_plan;
  * production: the back-projection grids of get_homography(256) / (320) (at 320 the masked rows hold the vanishing
    line's non-finite y) and the BEV grid, L = 2 and 4, orders 2 and 3, with the training shapes' plans pinned;
  * the header's promises: non-finite values in masked rows change nothing, one workspace reused across shapes,
    repeated launches, independence of the systems, and the status bits;
  * per case, in fp64: every mutation of lsq_contract (dropped chunk-boundary row, mask_rows +- 1, a neighbour's y, the
    last lane of a partial group from the lane before, x one column off, w = a, reg_ls dropped; factor 2 dropped, Z^-1
    transposed, a masked row left unzeroed, the residual's sign flipped) must break the gate.
The largest |err| / gate per entry point and dtype is printed at the end (pytest -s).
"""
import numpy as np
import pytest
import torch

import lsq_contract as lc

pytestmark = pytest.mark.gpu

DEV = "cuda"
GUARD = 256                          # elements of sentinel before and after every output
SENT = -1.2345e30                    # sentinel of the fp32 / bf16 outputs
SENT64 = -1.2345e300                 # sentinel of beta and zinv
WS_GUARD = 4096                      # guard bytes around the workspace
MEASURED = {}                        # (entry point, dtype) -> largest |err| / gate


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (entry, dt), exc in sorted(MEASURED.items()):
        print("%s %s: max |err| / gate %.3e, headroom %.1fx%s" % (entry, dt, exc, 1.0 / max(exc, 1e-30),
                                                               " (beyond d_o's bf16 rounding)" if entry == "lf_lsq_bwd" and dt == "bf16" else ""))


def _record(entry, dtype, exc):
    k = (entry, "bf16" if dtype == lc.LF_BF16 else "f32")
    MEASURED[k] = max(MEASURED.get(k, 0.0), exc)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _guarded(n, dtype, sent):
    return torch.full((2 * GUARD + n,), sent, dtype=dtype, device=DEV)


def _check(buf, sent, tag, name, written=True):
    s = torch.tensor(sent, dtype=buf.dtype, device=DEV)
    assert bool((buf[:GUARD] == s).all()) and bool((buf[-GUARD:] == s).all()), "%s: wrote outside %s" % (tag, name)
    if written:
        assert not bool((buf[GUARD:-GUARD] == s).any()), "%s: an entry of %s was not written" % (tag, name)


class Workspace:
    """lf_lsq_workspace_bytes bytes, zeroed, between guard bytes."""

    def __init__(self, nbytes):
        self.n = nbytes
        self.buf = torch.full((2 * WS_GUARD + nbytes,), 0xA5, dtype=torch.uint8, device=DEV)
        self.buf[WS_GUARD:WS_GUARD + nbytes] = 0

    def ptr(self):
        return self.buf[WS_GUARD:].data_ptr()

    def check(self, tag):
        g = self.buf[:WS_GUARD], self.buf[WS_GUARD + self.n:]
        assert all(bool((t == 0xA5).all()) for t in g), "%s: wrote outside the workspace" % tag
        assert bool((self.buf[WS_GUARD:WS_GUARD + 65536] == 0).all()), "%s: tickets left non-zero" % tag


def _dev(o, dtype):
    t = torch.from_numpy(np.ascontiguousarray(o, np.float32)).to(DEV)
    return t.bfloat16() if dtype == lc.LF_BF16 else t


def fwd(o_t, dtype, xtab, ytab, yrow, B, L, H, W, order, mask_rows, act, reg, solver, ws=None, status0=0, tag=""):
    """One lf_lsq_fwd launch into guarded buffers: (beta, zinv, masked, status) on the CPU."""
    c = _capi()
    n = order + 1
    beta = _guarded(B * L * n, torch.float64, SENT64)
    zinv = _guarded(B * L * n * n, torch.float64, SENT64)
    masked = _guarded(B * L * H * W, torch.float32, SENT)
    status = torch.full((1,), status0, dtype=torch.int32, device=DEV)
    need = c.lib().lf_lsq_workspace_bytes(B, L, H, W, order)
    ws = ws or Workspace(need)
    rc = c.lib().lf_lsq_fwd(o_t.data_ptr(), dtype, xtab.data_ptr(), None if ytab is None else ytab.data_ptr(),
                            None if yrow is None else yrow.data_ptr(), B, L, H, W, order, mask_rows, act, reg, solver,
                            beta[GUARD:].data_ptr(), zinv[GUARD:].data_ptr(), masked[GUARD:].data_ptr(),
                            status.data_ptr(), ws.ptr(), need, c.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (tag, rc)
    _check(beta, SENT64, tag, "beta")
    _check(zinv, SENT64, tag, "zinv")
    _check(masked, SENT, tag, "masked")
    ws.check(tag)
    return (beta[GUARD:-GUARD].cpu().numpy().reshape(B, L, n), zinv[GUARD:-GUARD].cpu().numpy().reshape(B, L, n, n),
            masked[GUARD:-GUARD].cpu().view(B, L, H, W), int(status.item()))


def bwd(o_t, dtype, xtab, ytab, yrow, B, L, H, W, order, mask_rows, act, beta, zinv, g, tag=""):
    c = _capi()
    odt = torch.bfloat16 if dtype == lc.LF_BF16 else torch.float32
    d_o = _guarded(B * L * H * W, odt, SENT)
    bt, zt, gt = (torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(DEV) for v in (beta, zinv, g))
    rc = c.lib().lf_lsq_bwd(o_t.data_ptr(), dtype, xtab.data_ptr(), None if ytab is None else ytab.data_ptr(),
                            None if yrow is None else yrow.data_ptr(), B, L, H, W, order, mask_rows, act, bt.data_ptr(),
                            zt.data_ptr(), gt.data_ptr(), d_o[GUARD:].data_ptr(), c.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (tag, rc)
    _check(d_o, SENT, tag, "d_o")
    return d_o[GUARD:-GUARD].float().cpu().numpy().reshape(B, L, H, W).astype(np.float64)


def check_masked(masked, o32, act, mask_rows, tag):
    top = masked[:, :, :mask_rows]
    assert bool((top.view(torch.int32) == 0).all()), "%s: masked rows are not +0.0" % tag
    want = lc.act_f32_torch(o32[:, :, mask_rows:], act)
    got = masked[:, :, mask_rows:]
    if lc.ACTS[act] in ("sigmoid", "softplus"):
        ea, _ = lc.act_err(np.asarray(o32[:, :, mask_rows:], np.float64), act)
        a64, _ = lc.act64(np.asarray(o32[:, :, mask_rows:], np.float64), act)
        assert bool(np.all(np.abs(got.double().numpy() - a64) <= ea)), "%s: masked outside e_a" % tag
    else:
        assert torch.equal(got, want), "%s: masked differs from torch float32" % tag


def run_forward(c, o, xtab, ytab, yrow, plan, tag, mutations=True):
    B, L, H, W = c["B"], c["L"], c["H"], c["W"]
    dt, mr = c["dtype"], c["mask_rows"]
    o_t = _dev(o, dt)
    xt, ytt = torch.from_numpy(xtab).to(DEV), torch.from_numpy(ytab).to(DEV)
    yrt = torch.from_numpy(yrow).to(DEV) if c["yrow"] else None
    beta, zinv, masked, st = fwd(o_t, dt, xt, ytt, yrt, B, L, H, W, c["order"], mr, c["act"], c["reg_ls"], c["solver"],
                                 tag=tag)
    assert st == 0, (tag, st)
    o_exact = o_t.float().cpu().numpy().astype(np.float64)
    args = (o_exact, xtab, yrow if plan["rowsep"] else ytab, H, W, c["order"], mr, c["act"], c["reg_ls"],
            plan["rowsep"], plan["nchunks"], dt)
    ref = lc.forward_reference(*args)
    assert float(ref["rho"].max()) <= lc.RHO_MAX, (tag, float(ref["rho"].max()))
    exc = lc.forward_excess(beta, zinv, ref)
    _record("lf_lsq_fwd", dt, exc)
    assert exc <= 1.0, "%s: beta / Z^-1 outside the gate (%.3g)" % (tag, exc)
    check_masked(masked, o_t.float().cpu(), c["act"], mr, tag)
    if mutations:
        for m in lc.forward_mutations(c, plan):
            r2 = lc.forward_reference(*args, mut=m)
            x = lc.forward_excess(beta, zinv, dict(r2, bound_beta=ref["bound_beta"], bound_zinv=ref["bound_zinv"]))
            assert x > 1.0, "%s: mutation %s stays within the gate (%.3g)" % (tag, m, x)
    return o_t, xt, ytt, yrt, beta, zinv


def run_backward(c, o_t, xt, ytt, yrt, plan, tag, ymax, mutations=True, seed=0):
    B, L, H, W, d = c["B"], c["L"], c["H"], c["W"], c["order"]
    dt, mr = c["dtype"], c["mask_rows"]
    beta, zinv, g = lc.nonsymmetric_backward_inputs(B, L, d, ymax, seed)
    got = bwd(o_t, dt, xt, ytt, yrt, B, L, H, W, d, mr, c["act"], beta, zinv, g, tag=tag)
    o_exact = o_t.float().cpu().numpy().astype(np.float64)
    yv = (yrt if plan["rowsep"] else ytt).cpu().numpy()
    args = (o_exact, xt.cpu().numpy(), yv, H, W, d, mr, c["act"], beta, zinv, g, plan["rowsep"], dt, got)
    ref, bound = lc.backward_reference(*args)
    exc = lc.excess(got, ref, bound)
    assert exc <= 1.0, "%s: d_o outside the gate (%.3g)" % (tag, exc)
    _record("lf_lsq_bwd", dt, lc.gate_use(got, ref, bound, lc.bf16_half_ulp(got) if dt == lc.LF_BF16 else 0.0))
    if mutations and mr < H:
        for m in lc.backward_mutations(c):
            r2, _ = lc.backward_reference(*args, mut=m)
            x = lc.excess(got, r2, bound)
            assert x > 1.0, "%s: mutation %s stays within the gate (%.3g)" % (tag, m, x)


# ---------------------------------------------------------------------------------------------------------------------
# coverage
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", lc.COVERAGE, ids=[c[0] for c in lc.COVERAGE])
def test_every_instance_against_fp64(case):
    c = lc.case_dict(case)
    o, xtab, ytab, yrow = lc.case_operands(c)
    plans = []
    for b in (0, 1):
        rc, pl = lc.query_plan(b, c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"],
                               c["act"])
        assert rc == 0
        want = lc.plan_py(b, c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"],
                          c["act"], _sms())[1]
        assert pl == want, (pl, want)
        plans.append(pl)
    tag = c["name"]
    o_t, xt, ytt, yrt, _, _ = run_forward(c, o, xtab, ytab, yrow, plans[0], tag)
    ymax = float(np.abs(yrow).max())
    run_backward(c, o_t, xt, ytt, yrt, plans[1], tag, ymax)


# ---------------------------------------------------------------------------------------------------------------------
# production grids
# ---------------------------------------------------------------------------------------------------------------------
def _bp_tables(R):
    from oracle import lsq_oracle as lo
    from lanedetection_end2end_b200 import ops_lsq
    M, _ = lo.get_homography(R)
    grid = lo.projective_grid(R, 2 * R, M.astype(np.float32))
    t = ops_lsq.GridTables(grid, R, 2 * R, 255.0)
    assert t.rowsep
    return t.xtab.numpy(), t.ytab.numpy(), t.yrow.numpy()


def _bev_tables(R):
    from oracle import lsq_oracle as lo
    from lanedetection_end2end_b200 import ops_lsq
    M, _ = lo.get_homography_bev()
    grid = lo.projective_grid(R, 2 * R, M.astype(np.float32), normalised=True)
    t = ops_lsq.GridTables(grid, R, 2 * R, 1.0)
    assert t.rowsep
    return t.xtab.numpy(), t.ytab.numpy(), t.yrow.numpy()


# (grid, resize, L, order, mask_rows, dtype, act, production batch) ; launched at B = 2
PRODUCTION = [("bp", 256, 2, 2, 77, lc.LF_F32, 1, 32), ("bp", 256, 4, 3, 52, lc.LF_BF16, 1, 64),
              ("bp", 320, 4, 3, 64, lc.LF_F32, 1, 32), ("bev", 256, 2, 2, 77, lc.LF_F32, 1, 16),
              ("bev", 256, 4, 3, 52, lc.LF_BF16, 4, 16)]
# plans of the training shapes on 132 SMs: (B, L, H, W, order, mask_rows) -> (fwd nchunks, bwd nchunks), NL = L, 1 group
PINNED = {(1, 2, 256, 512, 2, 77): (22, 22), (32, 2, 256, 512, 2, 77): (8, 16), (64, 4, 256, 512, 3, 52): (4, 8),
          (32, 4, 320, 640, 3, 64): (8, 16)}


def test_training_shapes_keep_their_plan():
    for (B, L, H, W, order, mr), (nf, nb) in PINNED.items():
        for dt in (lc.LF_F32, lc.LF_BF16):
            for b, n in ((0, nf), (1, nb)):
                rc, pl = lc.query_plan(b, dt, True, True, B, L, H, W, order, mr, 1)
                assert rc == 0 and pl["rowsep"] == 1 and pl["nl"] == L and pl["groups"] == 1
                assert pl == lc.plan_py(b, dt, True, True, B, L, H, W, order, mr, 1, _sms())[1]
                if _sms() == 132:
                    assert pl["nchunks"] == n, ((B, L, H, W, order, mr, dt, b), pl)


@pytest.mark.parametrize("prod", PRODUCTION, ids=["%s%d_L%d_d%d_%s" % (p[0], p[1], p[2], p[3], "bf16" if p[5] else "f32")
                                                  for p in PRODUCTION])
def test_production_grids_against_fp64(prod):
    kind, R, L, order, mr, dt, act, _ = prod
    H, W, B = R, 2 * R, 2
    xtab, ytab, yrow = _bp_tables(R) if kind == "bp" else _bev_tables(R)
    if R == 320:
        assert not np.isfinite(yrow[:mr]).all()       # the vanishing line lies in the masked rows
    assert np.isfinite(yrow[mr:]).all()
    c = dict(name="%s%d" % (kind, R), dtype=dt, act=act, L=L, H=H, W=W, B=B, order=order, solver=0, reg_ls=0.0,
             mask_rows=mr, grid="bev", yrow=True)
    o, _, _, _ = lc.case_operands(c)
    o = np.abs(o) if act == 1 else o
    rc, pf = lc.query_plan(0, dt, True, True, B, L, H, W, order, mr, act)
    rc2, pb = lc.query_plan(1, dt, True, True, B, L, H, W, order, mr, act)
    assert rc == 0 and rc2 == 0 and pf["rowsep"] == 1
    o_t, xt, ytt, yrt, _, _ = run_forward(c, o, xtab, ytab, yrow, pf, c["name"])
    run_backward(c, o_t, xt, ytt, yrt, pb, c["name"], float(np.abs(yrow[mr:]).max()))


# ---------------------------------------------------------------------------------------------------------------------
# the header's promises
# ---------------------------------------------------------------------------------------------------------------------
def _small(dt=lc.LF_F32, act=1, B=3, L=3, H=40, W=64, order=2, mr=9, name="promise"):
    c = dict(name=name, dtype=dt, act=act, L=L, H=H, W=W, B=B, order=order, solver=0, reg_ls=0.0, mask_rows=mr,
             grid="bev", yrow=True)
    o, xtab, ytab, yrow = lc.case_operands(c)
    return c, o, xtab, ytab, yrow


def _all(c, o, xtab, ytab, yrow, general=False, ws=None, status0=0):
    """(beta, zinv, masked, status, d_o) of one forward and one backward launch."""
    dt = c["dtype"]
    o_t = _dev(o, dt)
    xt, ytt = torch.from_numpy(xtab).to(DEV), torch.from_numpy(ytab).to(DEV)
    yrt = None if general else torch.from_numpy(yrow).to(DEV)
    args = (c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"], c["act"])
    beta, zinv, masked, st = fwd(o_t, dt, xt, ytt, yrt, *args, c["reg_ls"], c["solver"], ws=ws, status0=status0,
                                 tag=c["name"])
    bb, zz, gg = lc.nonsymmetric_backward_inputs(c["B"], c["L"], c["order"], 1.0, 5)
    d_o = bwd(o_t, dt, xt, ytt, yrt, *args, bb, zz, gg, tag=c["name"])
    return beta, zinv, masked, st, d_o


def _same(r1, r2, what):
    for a, b, n in zip(r1, r2, ("beta", "zinv", "masked", "status", "d_o")):
        if isinstance(a, torch.Tensor):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "%s: %s differs" % (what, n)
        elif isinstance(a, np.ndarray):
            assert np.array_equal(a.view(np.int64), b.view(np.int64)), "%s: %s differs" % (what, n)
        else:
            assert a == b, "%s: %s differs" % (what, n)


@pytest.mark.parametrize("general", [False, True])
@pytest.mark.parametrize("dt", [lc.LF_F32, lc.LF_BF16])
def test_masked_rows_are_never_read(general, dt):
    c, o, xtab, ytab, yrow = _small(dt=dt, act=5)
    base = _all(c, o, xtab, ytab, yrow, general)
    mr, W = c["mask_rows"], c["W"]
    o2, x2, yt2, yr2 = o.copy(), xtab.copy(), ytab.copy(), yrow.copy()
    o2[:, :, :mr] = np.nan
    o2[:, :, 0, 0] = np.inf
    x2[:mr * W] = np.inf
    yt2[:mr * W] = np.nan
    yr2[:mr] = -np.inf
    _same(base, _all(c, o2, x2, yt2, yr2, general), "non-finite masked rows")


def test_repeated_launches_and_one_workspace_for_every_shape():
    shapes = [_small(B=3, L=5, H=40, W=64, order=2, mr=9, name="reuse0"),
              _small(B=7, L=2, H=24, W=128, order=4, mr=3, name="reuse1"),
              _small(B=1, L=1, H=9, W=8, order=0, mr=0, name="reuse2"),
              _small(B=16, L=4, H=64, W=32, order=3, mr=60, name="reuse3")]
    fresh = [_all(*s) for s in shapes]
    _same(fresh[0], _all(*shapes[0]), "repeated launch")
    c = _capi()
    big = max(c.lib().lf_lsq_workspace_bytes(s[0]["B"], s[0]["L"], s[0]["H"], s[0]["W"], s[0]["order"]) for s in shapes)
    ws = Workspace(big)
    for rnd in range(2):
        for s, f in zip(shapes, fresh):
            _same(f, _all(*s, ws=ws), "shared workspace, round %d, %s" % (rnd, s[0]["name"]))


def test_systems_are_independent():
    c, o, xtab, ytab, yrow = _small(B=3, L=5)
    base = _all(c, o, xtab, ytab, yrow)
    o2 = o.copy()
    j = (1, 3)
    o2[j] = o2[j] * 1.5 + 0.25
    pert = _all(c, o2, xtab, ytab, yrow)
    keep = np.ones((c["B"], c["L"]), bool)
    keep[j] = False
    assert not np.array_equal(base[0][j], pert[0][j])
    assert np.array_equal(base[0][keep].view(np.int64), pert[0][keep].view(np.int64))
    assert np.array_equal(base[1][keep].view(np.int64), pert[1][keep].view(np.int64))
    assert np.array_equal(base[4][keep].view(np.int64), pert[4][keep].view(np.int64))


# ---------------------------------------------------------------------------------------------------------------------
# status
# ---------------------------------------------------------------------------------------------------------------------
def test_status_bits():
    c, o, xtab, ytab, yrow = _small(B=2, L=3)
    assert _all(c, o, xtab, ytab, yrow)[3] == 0
    assert _all(c, o, xtab, ytab, yrow, status0=lc_bits()["nonfinite"])[3] == lc_bits()["nonfinite"]   # kept
    # SINGULAR: one all-zero system, only its beta NaN
    o1 = o.copy()
    o1[1, 2] = 0
    beta, _, _, st, _ = _all(c, o1, xtab, ytab, yrow)
    assert st & lc_bits()["singular"]
    assert np.isnan(beta[1, 2]).all()
    others = np.ones((2, 3), bool)
    others[1, 2] = False
    assert np.isfinite(beta[others]).all()
    # SINGULAR: every row masked, no regularisation
    cm = dict(c, mask_rows=c["H"])
    beta, _, masked, st, d_o = _all(cm, o, xtab, ytab, yrow)
    assert st & lc_bits()["singular"] and np.isnan(beta).all()
    assert bool((masked.view(torch.int32) == 0).all()) and not d_o.any()
    # NOT_POSDEF: Cholesky with a negative reg_ls
    cc = dict(c, solver=1, reg_ls=-1e30)
    assert _all(cc, o, xtab, ytab, yrow)[3] & lc_bits()["not_posdef"]
    # NONFINITE: an Inf in an unmasked pixel; fp32 overflow of w
    o2 = o.copy()
    o2[0, 0, c["mask_rows"] + 1, 5] = np.inf
    assert _all(c, o2, xtab, ytab, yrow)[3] & lc_bits()["nonfinite"]
    o3 = o.copy()
    o3[1, 1, c["H"] - 1, 3] = 1e10                      # a = 1e20 is finite, w = a^2 = 1e40 overflows fp32
    assert _all(c, o3, xtab, ytab, yrow)[3] & lc_bits()["nonfinite"]


def lc_bits():
    c = _capi()
    return dict(singular=c.STATUS_SINGULAR, nonfinite=c.STATUS_NONFINITE, not_posdef=c.STATUS_NOT_POSDEF)
