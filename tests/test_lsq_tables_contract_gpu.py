"""The least-squares layer's table entry points -- row sums, grid gradient, per-image tables and prefix fits -- driven
through their C entry points, entry by entry against the fp64 / exact contract of tests/lsq_tables_contract.py.

Every output goes into a sentinel-filled buffer with guard regions (test_lsq_contract_gpu's _guarded / _check) and the
forward's workspace has guard bytes around it: no write may land outside an output, every entry must be written except
the row sums of rows < mask_rows (which must still hold the sentinel), and the tickets must be left at zero.  The grid
gradient reads the row-sum buffer as the forward left it, sentinel rows included.
  * coverage: every case of tc.COVERAGE through every table entry point (tc.case_calls), the instance of each call
    checked through lf_lsq_plan; beta / Z^-1, masked, row sums, g_rowp and d_o against their gates, d_o of the unfitted
    lanes +0.0 bit for bit, and per case the mutations (lanes read with stride L, image 0's tables for every image, the
    row sums' column index one off, and the grid gradient's six) outside the gates;
  * production: the fixed warp, hg.LearnedHomography with non-zero offsets and _PredictedWarpFunction's per-image
    tables at R = 256 and 320, B = 8, L = 4 and a prefix of K = 2 of 4 lanes.
The largest |err| / gate of each family is printed at the end (pytest -s).
"""
import numpy as np
import pytest
import torch

import lsq_contract as lc
import lsq_tables_contract as tc
from test_lsq_contract_gpu import GUARD, SENT, SENT64, Workspace, _bp_tables, _check, _guarded

pytestmark = pytest.mark.gpu

DEV = "cuda"
MEASURED = {}                       # family -> largest |err| / gate
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam, exc in sorted(MEASURED.items()):
        print("%s: max |err| / gate %.3e, headroom %.1fx" % (fam, exc, 1.0 / max(exc, 1e-30)))


def _record(fam, exc):
    MEASURED[fam] = max(MEASURED.get(fam, 0.0), exc)


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


def _p(t):
    return None if t is None else t.data_ptr()


def _g(buf):
    return buf[GUARD:].data_ptr()


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t.bfloat16() if dtype == lc.LF_BF16 else t


# ---------------------------------------------------------------------------------------------------------------------
# launches into guarded buffers
# ---------------------------------------------------------------------------------------------------------------------
def fwd(o_t, dt, tabs, keep_t, B, L, Lmap, H, W, order, mr, act, reg, solver, rowsums, per_image, lanes, tag):
    """One forward table entry point: (beta, zinv, masked [B, L, H, W] cpu, status, rowsums device buffer or None)."""
    c = _capi()
    xtab, ytab, yrow = tabs
    name = tc.entry_name(0, per_image, rowsums, keep_t is not None, lanes)
    n = order + 1
    beta = _guarded(B * L * n, torch.float64, SENT64)
    zinv = _guarded(B * L * n * n, torch.float64, SENT64)
    masked = _guarded(B * L * H * W, torch.float32, SENT)
    rs = _guarded(B * L * H * 3, torch.float32, SENT) if rowsums else None
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    need = c.lib().lf_lsq_workspace_bytes(B, L, H, W, order)
    ws = Workspace(need)
    args = [_p(o_t), dt, _p(xtab)]
    if per_image:
        args += [_p(yrow), _p(keep_t)]
    else:
        args += ([] if rowsums else [_p(ytab)]) + [_p(yrow)] + ([] if keep_t is None else [_p(keep_t)])
    args += [B, L] + ([Lmap] if lanes else []) + [H, W, order, mr, act, reg, solver, _g(beta), _g(zinv), _g(masked),
                                                 status.data_ptr()]
    if per_image or rowsums:
        args.append(None if rs is None else _g(rs))
    rc = getattr(c.lib(), name)(*args, ws.ptr(), need, c.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (tag, name, rc)
    for buf, s, what in ((beta, SENT64, "beta"), (zinv, SENT64, "zinv"), (masked, SENT, "masked")):
        _check(buf, s, "%s %s" % (tag, name), what)
    ws.check("%s %s" % (tag, name))
    if rs is not None:
        _check(rs, SENT, tag, "rowsums", written=False)
        v = rs[GUARD:-GUARD].view(B, L, H, 3)
        assert bool((v[:, :, :mr] == SENT).all()), "%s %s: a row sum of a masked row was written" % (tag, name)
        assert not bool((v[:, :, mr:] == SENT).any()), "%s %s: a row sum was not written" % (tag, name)
    return (beta[GUARD:-GUARD].cpu().numpy().reshape(B, L, n), zinv[GUARD:-GUARD].cpu().numpy().reshape(B, L, n, n),
            masked[GUARD:-GUARD].cpu().view(B, L, H, W), int(status.item()), rs)


def bwd(o_t, dt, tabs, keep_t, B, L, Lmap, H, W, order, mr, act, beta, zinv, g, per_image, lanes, tag):
    """One backward table entry point: d_o [B, Lmap if lanes else L, H, W] as a cpu tensor of o's dtype."""
    c = _capi()
    xtab, ytab, yrow = tabs
    name = tc.entry_name(1, per_image, False, keep_t is not None, lanes)
    Lm = Lmap if lanes else L
    d_o = _guarded(B * Lm * H * W, o_t.dtype, SENT)
    bt, zt, gt = (torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(DEV) for v in (beta, zinv, g))
    args = [_p(o_t), dt, _p(xtab)]
    if per_image:
        args += [_p(yrow), _p(keep_t)]
    else:
        args += [_p(ytab), _p(yrow)] + ([] if keep_t is None else [_p(keep_t)])
    args += [B, L] + ([Lmap] if lanes else []) + [H, W, order, mr, act, bt.data_ptr(), zt.data_ptr(), gt.data_ptr(),
                                                 _g(d_o), c.stream_ptr()]
    rc = getattr(c.lib(), name)(*args)
    torch.cuda.synchronize()
    assert rc == 0, (tag, name, rc)
    _check(d_o, SENT, "%s %s" % (tag, name), "d_o")
    return d_o[GUARD:-GUARD].cpu().view(B, Lm, H, W)


def grid_grad(rs, yrow_t, beta, zinv, g, B, L, H, order, mr, per_image, tag):
    c = _capi()
    out = _guarded((B if per_image else 1) * H * 3, torch.float64, SENT64)
    bt, zt, gt = (torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(DEV) for v in (beta, zinv, g))
    name = "lf_lsq_grid_grad_per_image" if per_image else "lf_lsq_grid_grad"
    rc = getattr(c.lib(), name)(_g(rs), _p(yrow_t), bt.data_ptr(), zt.data_ptr(), gt.data_ptr(), B, L, H, order, mr,
                                _g(out), c.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (tag, name, rc)
    _check(out, SENT64, "%s %s" % (tag, name), "g_rowp")
    v = out[GUARD:-GUARD].cpu().numpy()
    return v.reshape(B, H, 3) if per_image else v.reshape(H, 3)


def check_masked(masked, o32, act, mr, keep, tag):
    """masked: +0.0 in the masked rows and where keep is 0, the activation (torch float32, or within e_a) elsewhere."""
    H, W = o32.shape[-2:]
    live = np.zeros((H, W), bool)
    live[mr:] = True if keep is None else keep[mr:] != 0
    mk = masked.numpy()
    assert (mk[..., ~live].view(np.int32) == 0).all(), "%s: masked is not +0.0 where it must be" % tag
    if lc.ACTS[act] in ("sigmoid", "softplus"):
        o64 = o32.numpy().astype(np.float64)
        ea, _ = lc.act_err(o64, act)
        a64, _ = lc.act64(o64, act)
        assert (np.abs(mk - a64)[..., live] <= ea[..., live]).all(), "%s: masked outside e_a" % tag
    else:
        assert np.array_equal(mk[..., live], lc.act_f32_torch(o32, act).numpy()[..., live]), "%s: masked" % tag


def bwd_gate(o64, xtab, yv, H, W, d, mr, act, beta, zinv, g, rowsep, dt, got, keep, per_image, mut=None):
    """(ref, bound) of d_o: lc.backward_reference (per image on its own tables), zero where keep is 0."""
    if per_image:
        ref, bound = tc.per_image_backward_reference(o64, xtab, yv, H, W, d, mr, act, beta, zinv, g, dt, got, mut=mut)
    else:
        ref, bound = lc.backward_reference(o64, xtab, yv, H, W, d, mr, act, beta, zinv, g, rowsep, dt, got)
    if keep is not None:
        ref[..., keep == 0] = 0.0
        bound[..., keep == 0] = 0.0
    return ref, bound


def rowsums_gate(o64, xtab, H, W, mr, act, dt, keep, per_image, mut=None):
    if not per_image:
        return tc.rowsums_reference(o64, xtab, H, W, mr, act, dt, keep, mut=mut)
    parts = [tc.rowsums_reference(o64[b:b + 1], xtab[b], H, W, mr, act, dt, keep, mut=mut) for b in range(len(o64))]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


# ---------------------------------------------------------------------------------------------------------------------
# coverage
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", tc.COVERAGE, ids=[c[0] for c in tc.COVERAGE])
def test_every_table_entry_point_against_fp64(case):
    c = tc.case_dict(case)
    o, xtab, ytab, yrow, xs, ys, keep = tc.case_operands(c)
    B, L, Lmap, H, W, d, mr, act, dt = (c[k] for k in ("B", "L", "Lmap", "H", "W", "order", "mask_rows", "act", "dtype"))
    tag = c["name"]
    calls = tc.case_calls(c)
    for call in calls:
        rc, inst = tc.case_instance(c, call, plan=lc.query_plan)
        assert rc == 0 and inst == tc.case_instance(c, call, plan=lambda *a: lc.plan_py(*a, sms=lc.device_sms()))[1]
    pf = lc.query_plan(0, dt, c["yrow"], True, B, L, H, W, d, mr, act)[1]
    pb = lc.query_plan(1, dt, c["yrow"], True, B, L, H, W, d, mr, act)[1]
    o_t = _dev(o, dt)                                            # [B, Lmap, H, W]
    o_exact = o_t.float().cpu().numpy().astype(np.float64)
    o64 = np.ascontiguousarray(o_exact[:, :L])
    o32 = torch.from_numpy(o64.astype(np.float32))
    shared = (_dev(xtab), _dev(ytab), _dev(yrow) if c["yrow"] else None)
    per_img = (_dev(xs), None, _dev(ys))
    keep_t = _dev(keep)
    beta_b, zinv_b, g_b = lc.nonsymmetric_backward_inputs(B, L, d, float(np.abs(yrow).max()), 0)
    refs, rowsum_bufs, mutated = {}, {}, set()

    def fit_ref(pi, km, o_in=o64, mut=None):
        key = (pi, km is not None)
        if mut is None and o_in is o64 and key in refs:
            return refs[key]
        oz = o_in if km is None else tc.zeroed(o_in, km, act)
        if pi:
            r = tc.per_image_forward_reference(oz, xs, ys, H, W, d, mr, act, c["reg_ls"], pf["nchunks"], dt, mut=mut)
        else:
            r = lc.forward_reference(oz, xtab, yrow if pf["rowsep"] else ytab, H, W, d, mr, act, c["reg_ls"],
                                     pf["rowsep"], pf["nchunks"], dt)
        if mut is None and o_in is o64:
            assert float(r["rho"].max()) <= lc.RHO_MAX, tag
            refs[key] = r
        return r

    for entry, kp, rs_on in calls:
        km = keep if kp else None
        kt = keep_t if kp else None
        pi = "per_image" in entry
        lanes = entry.endswith("_lanes")
        tabs = per_img if pi else shared
        what = "%s %s%s%s" % (tag, entry, " keep" if kp else "", " rowsums" if rs_on and pi else "")
        if entry.startswith("lf_lsq_grid_grad"):
            continue
        ot = o_t if lanes else o_t[:, :L].contiguous()
        if "_bwd" in entry:
            got_t = bwd(ot, dt, tabs, kt, B, L, Lmap, H, W, d, mr, act, beta_b, zinv_b, g_b, pi, lanes, what)
            if lanes:
                rest = got_t[:, L:].contiguous().view(_INT[got_t.dtype])
                assert bool((rest == 0).all()), "%s: d_o of the unfitted lanes is not +0.0" % what
            got = got_t[:, :L].double().numpy()
            yv = ys if pi else (yrow if pb["rowsep"] else ytab)
            xv = xs if pi else xtab
            ref, bound = bwd_gate(o64, xv, yv, H, W, d, mr, act, beta_b, zinv_b, g_b, pb["rowsep"], dt, got, km, pi)
            exc = lc.excess(got, ref, bound)
            assert exc <= 1.0, "%s: d_o outside the gate (%.3g)" % (what, exc)
            _record("d_o " + ("per_image" if pi else "lanes"),
                    lc.gate_use(got, ref, bound, lc.bf16_half_ulp(got) if dt == lc.LF_BF16 else 0.0))
            if mr < H and lanes and ("bwd_lanes", pi) not in mutated:
                mutated.add(("bwd_lanes", pi))
                r2, _ = bwd_gate(tc.stride_l_view(o_exact, L), xv, yv, H, W, d, mr, act, beta_b, zinv_b, g_b,
                                 pb["rowsep"], dt, got, km, pi)
                assert lc.excess(got, r2, bound) > 1.0, "%s: lanes read with stride L stay within the gate" % what
            if mr < H and pi and "bwd_image0" not in mutated:
                mutated.add("bwd_image0")
                r2, _ = bwd_gate(o64, xv, yv, H, W, d, mr, act, beta_b, zinv_b, g_b, True, dt, got, km, True,
                                 mut=("image0",))
                assert lc.excess(got, r2, bound) > 1.0, "%s: image 0's tables stay within the gate" % what
            continue
        beta, zinv, masked, st, rs = fwd(ot, dt, tabs, kt, B, L, Lmap, H, W, d, mr, act, c["reg_ls"], c["solver"],
                                         rs_on, pi, lanes, what)
        assert st == 0, (what, st)
        ref = fit_ref(pi, km)
        exc = lc.forward_excess(beta, zinv, ref)
        assert exc <= 1.0, "%s: beta / Z^-1 outside the gate (%.3g)" % (what, exc)
        _record("beta, Z^-1 " + ("per_image" if pi else "lanes" if lanes else "rowsums"), exc)
        check_masked(masked, o32, act, mr, km, what)
        bounds = dict(bound_beta=ref["bound_beta"], bound_zinv=ref["bound_zinv"])
        if mr < H and lanes and ("fwd_lanes", pi) not in mutated:
            mutated.add(("fwd_lanes", pi))
            r2 = fit_ref(pi, km, tc.stride_l_view(o_exact, L), mut=())
            assert lc.forward_excess(beta, zinv, dict(r2, **bounds)) > 1.0, "%s: stride L within the gate" % what
        if mr < H and pi and "fwd_image0" not in mutated:
            mutated.add("fwd_image0")
            r2 = fit_ref(True, km, o64, mut=("image0",))
            assert lc.forward_excess(beta, zinv, dict(r2, **bounds)) > 1.0, "%s: image 0's tables within the gate" % what
        if rs is None:
            continue
        xv = xs if pi else xtab
        got = rs[GUARD:-GUARD].view(B, L, H, 3)[:, :, mr:].double().cpu().numpy()
        ref_rs, bound_rs = rowsums_gate(o64, xv, H, W, mr, act, dt, km, pi)
        exc = lc.excess(got, ref_rs, bound_rs)
        assert exc <= 1.0, "%s: row sums outside the gate (%.3g)" % (what, exc)
        _record("rowsums", exc)
        if mr < H and ("col", pi) not in mutated:
            mutated.add(("col", pi))
            r2, _ = rowsums_gate(o64, xv, H, W, mr, act, dt, km, pi, mut=("col_shift",))
            assert lc.excess(got, r2, bound_rs) > 1.0, "%s: the column index one off within the gate" % what
        if not kp and not lanes:
            rowsum_bufs[pi] = rs
    # the grid gradient, on the row sums the forward left (sentinel rows included)
    if not pf["rowsep"]:
        return
    for pi in (False, True):
        rs = rowsum_bufs[pi]
        yv, xv = (ys, xs) if pi else (yrow, xtab)
        got = grid_grad(rs, _dev(yv), beta_b, zinv_b, g_b, B, L, H, d, mr, pi, tag)
        rsn = rs[GUARD:-GUARD].view(B, L, H, 3).double().cpu().numpy()
        args = (rsn, yv, beta_b, zinv_b, g_b, B, L, H, d, mr, pi)
        ref, bound = tc.grid_grad_reference(*args)
        exc = lc.excess(got, ref, bound)
        assert exc <= 1.0, "%s: g_rowp%s outside the gate (%.3g)" % (tag, " per image" if pi else "", exc)
        _record("grid_grad" + (" per_image" if pi else ""), exc)
        below = tc.row_below_mask(o64, xv, H, W, mr, act, dt) if mr > 0 else None
        for m in tc.grid_grad_mutations(c, pi):
            x = lc.excess(got, tc.emulate_grid_grad(*args, mut=m, below=below), bound)
            assert x > 1.0, "%s: grid gradient mutation %s stays within the gate (%.3g)" % (tag, m, x)


# ---------------------------------------------------------------------------------------------------------------------
# production tables
# ---------------------------------------------------------------------------------------------------------------------
# (warp, R, mask_rows, dtype); B = 8, order 3, square; every case fits all 4 lanes and the prefix K = 2 of 4
PRODUCTION = [("fixed", 256, 52, lc.LF_F32), ("fixed", 320, 96, lc.LF_BF16), ("learned", 256, 77, lc.LF_BF16),
              ("learned", 320, 77, lc.LF_F32), ("predicted", 256, 77, lc.LF_F32), ("predicted", 320, 96, lc.LF_BF16)]


def _production_tables(warp, R, mr, B):
    """(xtab, yrow) numpy fp32: [R*2R] and [R] for a shared warp, [B, R*2R] and [B, R] per image."""
    from lanedetection_end2end_b200 import homography as hg
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    if warp == "fixed":
        xtab, _, yrow = _bp_tables(R)
        return xtab, yrow
    if warp == "learned":
        mod = hg.LearnedHomography(R, mr).cuda()
        with torch.no_grad():
            mod.offsets.copy_(torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01]))
        t = mod(st)
        out = t.xtab.cpu().numpy(), t.yrow.cpu().numpy()
    else:
        z = (torch.randn(B, 3, generator=torch.Generator().manual_seed(R)) * 0.5).to(DEV)
        t = hg._PredictedWarpFunction.apply(z, R, mr, 255.0, st)
        out = t[4].cpu().numpy(), t[5].cpu().numpy()
        assert not np.array_equal(out[1][0], out[1][1])
    assert int(st.item()) == 0
    return out


@pytest.mark.parametrize("prod", PRODUCTION, ids=["%s%d_m%d_%s" % (p[0], p[1], p[2], "bf16" if p[3] else "f32")
                                                  for p in PRODUCTION])
def test_production_tables_against_fp64(prod):
    from oracle import inputs
    warp, R, mr, dt = prod
    B, Lmap, H, W, d, act = 8, 4, R, 2 * R, 3, 1
    pi = warp == "predicted"
    xtab, yrow = _production_tables(warp, R, mr, B)
    assert np.isfinite(yrow[..., mr:]).all()
    o = inputs.make_lane_maps(B, Lmap, H, W, seed=R + mr)
    o_t = _dev(o, dt)
    o_exact = o_t.float().cpu().numpy().astype(np.float64)
    tabs = (_dev(xtab), None, _dev(yrow))
    for L in (4, 2):
        tag = "%s%d L%d of %d" % (warp, R, L, Lmap)
        lanes = L < Lmap
        o64 = np.ascontiguousarray(o_exact[:, :L])
        beta, zinv, masked, st, rs = fwd(o_t, dt, tabs, None, B, L, Lmap, H, W, d, mr, act, 0.0, 0, True, pi, lanes,
                                         tag)
        assert st == 0, (tag, st)
        pf = lc.query_plan(0, dt, True, False, B, L, H, W, d, mr, act)[1]
        pb = lc.query_plan(1, dt, True, False, B, L, H, W, d, mr, act)[1]
        if pi:
            ref = tc.per_image_forward_reference(o64, xtab, yrow, H, W, d, mr, act, 0.0, pf["nchunks"], dt)
        else:
            ref = lc.forward_reference(o64, xtab, yrow, H, W, d, mr, act, 0.0, True, pf["nchunks"], dt)
        assert float(ref["rho"].max()) <= lc.RHO_MAX
        exc = lc.forward_excess(beta, zinv, ref)
        assert exc <= 1.0, "%s: beta / Z^-1 outside the gate (%.3g)" % (tag, exc)
        _record("beta, Z^-1 production", exc)
        got = rs[GUARD:-GUARD].view(B, L, H, 3)[:, :, mr:].double().cpu().numpy()
        ref_rs, bound_rs = rowsums_gate(o64, xtab, H, W, mr, act, dt, None, pi)
        exc = lc.excess(got, ref_rs, bound_rs)
        assert exc <= 1.0, "%s: row sums outside the gate (%.3g)" % (tag, exc)
        _record("rowsums production", exc)
        gbeta = np.random.default_rng(L).standard_normal((B, L, d + 1))
        gg = grid_grad(rs, tabs[2], beta, zinv, gbeta, B, L, H, d, mr, pi, tag)
        rsn = rs[GUARD:-GUARD].view(B, L, H, 3).double().cpu().numpy()
        gref, gbound = tc.grid_grad_reference(rsn, yrow, beta, zinv, gbeta, B, L, H, d, mr, pi)
        exc = lc.excess(gg, gref, gbound)
        assert exc <= 1.0, "%s: g_rowp outside the gate (%.3g)" % (tag, exc)
        _record("grid_grad production", exc)
        d_t = bwd(o_t if lanes else o_t[:, :L].contiguous(), dt, tabs, None, B, L, Lmap, H, W, d, mr, act, beta, zinv,
                  gbeta, pi, lanes, tag)
        if lanes:
            assert bool((d_t[:, L:].contiguous().view(_INT[d_t.dtype]) == 0).all()), tag
        got = d_t[:, :L].double().numpy()
        ref, bound = bwd_gate(o64, xtab, yrow, H, W, d, mr, act, beta, zinv, gbeta, pb["rowsep"], dt, got, None, pi)
        exc = lc.excess(got, ref, bound)
        assert exc <= 1.0, "%s: d_o outside the gate (%.3g)" % (tag, exc)
        _record("d_o production", lc.gate_use(got, ref, bound, lc.bf16_half_ulp(got) if dt == lc.LF_BF16 else 0.0))
