"""lf_conv_f32, lf_wgrad_f32 and the split reductions (lf_wgrad_reduce, lf_reduce_multi, lf_vec_reduce, lf_colsum) driven
directly through their C entry points, entry by entry against the fp64 restatement of their contracts
(tests/f32_contract.py).

Every case builds the args struct by hand over strided NHWC views, launches once into sentinel-filled buffers and holds
every entry the contract writes to |got - ref| <= (k_steps + c) * 2^-24 * S, and every other entry to the sentinel:
  * lf_conv_f32: each N-tile instantiation with Cout at, 1 below and 3 below the padded width (vector and scalar epilogue,
    with and without bias / ReLU / mask_src / add_src / add_mask), every production phase table of net_plans at pixel
    counts off the tile size, channel-slice strides on both sides, permuted weight slots, K tails, four operand classes,
    bitwise determinism and exact power-of-two equivariance;
  * lf_wgrad_f32: every production weight-gradient plan, one shape per branch of the small-channel kernel's plan, the four
    tile instantiations over odd channel counts, split counts 1 / preferred / non-dividing / more than there are steps,
    each split's partial on its own pixel range, then the reductions bit for bit against each other and against fp64;
  * per family, in fp64: dropping the last pixels, shifting a tap by one pixel, swapping oy0 / ox0 or ignoring out_coff
    must each break the gate, so the case would see those bugs.
The largest |err| / gate per kernel is printed at the end (pytest -s)."""
import ctypes

import pytest
import torch

import f32_contract as fc
from lanedetection_end2end_b200 import net_plans as plans

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -1.2345e30                     # sentinel: a value no kernel here produces
GUARD = 1024                          # floats of sentinel after every output
MEASURED = {}                         # kernel -> largest |err| / gate seen


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(MEASURED.items()):
        print("%-28s max |err| / gate %.3f" % (k, v))


def _hold(kern, what, got, ref, bound):
    x = fc.excess(got, ref, bound)
    MEASURED[kern] = max(MEASURED.get(kern, 0.0), x)
    assert x <= 1.0, "%s: |err| reaches %.3g x the gate" % (what, x)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _operand(n, cls, g):
    t = torch.randn(n, generator=g, device=DEV)
    if cls == "relu":
        return t.clamp_min(0)
    if cls == "heavy":
        return t * torch.exp(2 * torch.randn(n, generator=g, device=DEV))
    return t


def _buf(n):
    return torch.full((n + GUARD,), SENT, dtype=torch.float32, device=DEV)


def _untouched(buf, off):
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    keep[off.reshape(-1)] = False
    return bool((buf[keep] == SENT).all())


def _p(t, off=0):
    return None if t is None else t.data_ptr() + 4 * off


# =====================================================================================================================
# lf_conv_f32
# =====================================================================================================================
def launch_conv(s, inp, wmat, out, bias=None, mask_src=None, add_src=None, add_mask=None):
    c = _capi()
    a = c.LfConvArgs()
    a.inp, a.wmat, a.bias, a.out = _p(inp), _p(wmat), _p(bias), _p(out)
    a.mask_src, a.add_src, a.add_mask = _p(mask_src), _p(add_src), _p(add_mask)
    for k in ("N", "Hin", "Win", "Cin", "in_cstride", "Hout", "Wout", "out_cstride", "out_coff", "Cout", "CoutPad", "Hs", "Ws",
              "osy", "osx", "oy0", "ox0", "isy", "isx", "ntaps", "relu"):
        setattr(a, k, getattr(s, k))
    for t in range(s.ntaps):
        a.dy[t], a.dx[t], a.wtap[t] = s.dy[t], s.dx[t], s.wtap[t]
    c.call("lf_conv_f32", ctypes.byref(a), c.stream_ptr())


def run_conv_case(s, cls="randn", epi=False, seed=0, zero_group=False, repeat=False, scale=False, mutate=()):
    g = _gen(seed)
    inp = _operand(s.N * s.Hin * s.Win * s.in_cstride, cls, g)
    if zero_group:
        inp.view(-1, s.in_cstride)[:, :4] = 0
    wmat = torch.randn((max(s.wtap) + 1) * s.Cin * s.CoutPad, generator=g, device=DEV)
    n_out = s.N * s.Hout * s.Wout * s.out_cstride
    extra = {}
    if epi:
        extra = dict(bias=torch.randn(s.Cout, generator=g, device=DEV),
                     mask_src=torch.randn(n_out, generator=g, device=DEV).clamp_min(0),      # half the gates are exact zeros
                     add_src=torch.randn(n_out, generator=g, device=DEV))
        if epi == "add_mask":
            extra["add_mask"] = torch.randn(n_out, generator=g, device=DEV)
    out = _buf(n_out)
    launch_conv(s, inp, wmat, out, **extra)
    ref, S, off = fc.conv_f32(s, inp, wmat, **extra)
    bound = fc.gate(fc.conv_ksteps(s), S)
    what = "conv Cin %d Cout %d/%d taps %d M %d %s" % (s.Cin, s.Cout, s.CoutPad, s.ntaps, s.N * s.Hs * s.Ws, cls)
    _hold("lf_conv_f32 BN=%d" % conv_bn(s.CoutPad), what, out[off], ref, bound)
    assert _untouched(out, off), what + ": wrote outside the phase's entries"
    if repeat:
        out2 = _buf(n_out)
        launch_conv(s, inp, wmat, out2, **extra)
        assert torch.equal(out, out2), what + ": not deterministic"
    if scale:
        o1, o2 = _buf(n_out), _buf(n_out)
        launch_conv(s, inp, wmat, o1)
        launch_conv(s, inp * 8.0, wmat, o2)
        assert torch.equal(o1[off] * 8.0, o2[off]), what + ": not equivariant under a power-of-two scale"
    ref0 = torch.zeros(out.numel(), dtype=torch.float64, device=DEV)
    ref0[off] = ref
    for m in mutate:
        if m == "swap_phase":
            s2 = fc.NS(**dict(vars(s), oy0=s.ox0, ox0=s.oy0))
            r2, _, o2 = fc.conv_f32(s2, inp, wmat, **extra)
        else:
            kw = dict(drop_tile=dict(m_limit=ref.shape[0] - 1 - (ref.shape[0] - 1) % 128), shift_tap=dict(tap_shift=(s.ntaps // 2, 1)),
                      ignore_coff=dict(ignore_coff=True))[m]
            r2, _, o2 = fc.conv_f32(s, inp, wmat, **dict(extra, **kw))
        mut = torch.zeros_like(ref0)
        mut[o2] = r2
        assert fc.excess(mut[off], ref, bound) > 1.0, what + ": the gate would not see mutation " + m
    return out


def conv_bn(pad):
    return 128 if pad % 128 == 0 else (64 if pad % 64 == 0 else (32 if pad % 32 == 0 else 16))


TAPS3 = [(0, -2, 0), (0, 0, 1), (0, 2, 2)]


@pytest.mark.parametrize("pad", [16, 32, 64, 128, 48, 96])
@pytest.mark.parametrize("below", [0, 1, 3])
def test_conv_instantiations_and_both_epilogue_branches(pad, below):
    """N = 2, 9 x 15 (M = 270: a partial last tile for BM 128 and 256), K = 3*8 = 24 (half a K step), output in a slice."""
    cout = pad - below
    cs = -(-cout // 4) * 4 + 8
    ph = plans._phase(9, 15, TAPS3)
    for epi in (False, True, "add_mask"):
        s = fc.conv_spec(2, 9, 15, 8, 9, 15, cout, pad, ph, in_cstride=12, out_cstride=cs, out_coff=4, relu=int(bool(epi)))
        run_conv_case(s, epi=epi, seed=pad + below, mutate=("drop_tile", "shift_tap", "ignore_coff") if epi is True else ())


def _production_conv_cases():
    """(id, N, Hin, Win, Cin, in_cstride, Hout, Wout, Cout, CoutPad, out_cstride, out_coff, phases)."""
    out = []
    for name, ci, cs_in, cc, ctot, H, W in (("stem", 4, 4, 13, 16, 18, 22), ("down16_64", 16, 16, 48, 64, 14, 18),
                                            ("down64_128", 64, 64, 64, 128, 10, 14)):
        ph, (Ho, Wo) = plans.conv_fwd_plan(H, W, 3, 3, 2, 1, 1)
        out.append((name, 3, H, W, ci, cs_in, Ho, Wo, cc, plans.cout_pad(cc), ctot, 0, ph))
        dph, _ = plans.transposed_gather_plan(Ho, Wo, H, W, 3, 1)                       # its input gradient: 4 phases
        cip = plans.pad_to(cc, 4)
        out.append((name + "_dgrad", 3, Ho, Wo, cip, ctot, H, W, ci, plans.cout_pad(ci), ci, 0, dph))
    for name, ci, co, H, W in (("up128_64", 128, 64, 5, 7), ("up64_16", 64, 16, 9, 11)):
        ph, (Hb, Wb) = plans.transposed_gather_plan(H, W, 2 * H, 2 * W, 3, 1)
        out.append((name, 3, H, W, ci, ci, Hb, Wb, co, plans.cout_pad(co), co, 0, ph))
        dph, _ = plans.convT_dgrad_plan(Hb, Wb, H, W, 3, 1)
        out.append((name + "_dgrad", 3, Hb, Wb, co, co, H, W, ci, plans.cout_pad(ci), ci, 0, dph))
    for C, dil in ((64, 1), (128, 2), (128, 16), (16, 1), (64, 16)):
        for vert in (True, False):
            kh, kw, p, d = (3, 1, (dil, 0), (dil, 1)) if vert else (1, 3, (0, dil), (1, dil))
            ph, _ = plans.conv_fwd_plan(9, 11, kh, kw, 1, p[0], p[1], d[0], d[1])
            out.append(("%s_c%d_d%d" % ("v" if vert else "h", C, dil), 3, 9, 11, C, C, 9, 11, C, plans.cout_pad(C), C, 0, ph))
            dph, _ = plans.conv_dgrad_plan_s1(9, 11, kh, kw, p[0], p[1], d[0], d[1])
            out.append(("%s_c%d_d%d_dgrad" % ("v" if vert else "h", C, dil), 3, 9, 11, C, C, 9, 11, C, plans.cout_pad(C), C, 0, dph))
    ph, _ = plans.conv_fwd_plan(5, 7, 3, 3, 1, 1, 1)
    out.append(("head3x3_small_M", 1, 5, 7, 64, 64, 5, 7, 64, 64, 64, 0, ph))           # M = 35 < 128
    return out


PROD_CONV = _production_conv_cases()


@pytest.mark.parametrize("case", PROD_CONV, ids=[c[0] for c in PROD_CONV])
def test_conv_production_phase_tables(case):
    name, N, Hin, Win, Cin, cs_in, Hout, Wout, Cout, pad, cs_out, coff, phases = case
    n_out = N * Hout * Wout * cs_out
    seen = torch.zeros(n_out + GUARD, dtype=torch.int32, device=DEV)
    for k, ph in enumerate(phases):
        s = fc.conv_spec(N, Hin, Win, Cin, Hout, Wout, Cout, pad, ph, in_cstride=cs_in, out_cstride=cs_out, out_coff=coff,
                         relu=k % 2)
        assert (N * s.Hs * s.Ws) % 256 != 0
        multi = len(phases) > 1
        run_conv_case(s, cls=("randn", "relu", "heavy")[k % 3], epi=("add_mask" if k % 2 else False), seed=len(name) + k,
                      repeat=(k == 0), mutate=(("swap_phase",) if multi and ph["oy0"] != ph["ox0"] else ("shift_tap",)))
        seen[fc.conv_out_offsets(s, DEV).reshape(-1)] += 1
    if len(phases) > 1:                       # the phases of a transposed convolution tile the output exactly once
        v = seen[:n_out].view(-1, cs_out)
        assert bool((v[:, coff:coff + Cout] == 1).all()) and int(seen.sum()) == N * Hout * Wout * Cout


@pytest.mark.parametrize("ntaps,Cin", [(1, 4), (3, 4), (9, 4), (3, 16)])
@pytest.mark.parametrize("cls", ["randn", "relu", "heavy", "zero_group"])
def test_conv_k_tails_slices_permuted_slots_and_operand_classes(ntaps, Cin, cls):
    taps = [(a - 1, b - 1, 0) for a in range(3) for b in range(3)][:ntaps] if ntaps > 1 else [(0, 0, 0)]
    slots = [(5 * t + 2) % 11 for t in range(ntaps)]                                  # wtap[t] != t, slots up to 10
    ph = plans._phase(7, 13, [(dy, dx, sl) for (dy, dx, _), sl in zip(taps, slots)])
    s = fc.conv_spec(3, 7, 13, Cin, 7, 13, 20, 32, ph, in_cstride=Cin + 8, out_cstride=28, out_coff=8)
    run_conv_case(s, cls="randn" if cls == "zero_group" else cls, zero_group=(cls == "zero_group"), seed=ntaps * Cin,
                  repeat=True, scale=True,
                  mutate=() if cls == "zero_group" else ("ignore_coff",) + (("shift_tap",) if ntaps > 1 else ()))


# =====================================================================================================================
# lf_wgrad_f32 and the reductions
# =====================================================================================================================
def fill_wgrad(s, P, Q, partial, qpart, nsplit, p_off=0, q_off=0):
    c = _capi()
    a = c.LfWgradArgs()
    for k in ("N", "Hs", "Ws", "Hp", "Wp", "Cp", "p_cstride", "p_coff", "psy", "psx", "Hq", "Wq", "Cq", "q_cstride", "q_coff",
              "qsy", "qsx", "ntaps", "CpPad", "CqPad"):
        setattr(a, k, getattr(s, k))
    for t in range(s.ntaps):
        a.pdy[t], a.pdx[t], a.qdy[t], a.qdx[t] = s.pdy[t], s.pdx[t], s.qdy[t], s.qdx[t]
    a.P, a.Q, a.partial, a.qsum_partial, a.nsplit = _p(P), _p(Q), _p(partial), _p(qpart), nsplit
    return a


def run_wgrad_case(s, nsplits, qsum, cls="randn", seed=0, expect_small=None, mutate=False):
    """nsplits: split counts; "pref" = the library's preference, "over" = more splits than PXS-pixel steps."""
    c = _capi()
    g = _gen(seed)
    P = _operand(s.N * s.Hp * s.Wp * s.p_cstride, cls, g)
    Q = _operand(s.N * s.Hq * s.Wq * s.q_cstride, cls, g)
    plan, why = fc.ws_plan(s, qsum)
    if expect_small is not None:
        assert (plan is not None) == expect_small, why
    kern = "lf_wgrad_f32 small" if plan else "lf_wgrad_f32 tile %dx%d" % (16 if s.Cp <= 16 else 64, 16 if s.Cq <= 16 else 64)
    PXS = plan.PXS if plan else fc.tile_pxs(s)
    M = s.N * s.Hs * s.Ws
    a0 = fill_wgrad(s, P, Q, P, P if qsum else None, 1)
    pref = int(c.lib().lf_wgrad_f32_nsplit(ctypes.byref(a0)))
    assert (pref > 0) == (plan is not None)
    Gt, St, qt, Sqt = fc.wgrad_f32(s, P, Q)
    for ns in nsplits:
        ns = {"pref": pref if pref > 0 else max(1, M // 256), "over": -(-M // PXS) + 3}.get(ns, ns)
        what = "%s Cp %d Cq %d taps %d M %d nsplit %d %s" % (kern, s.Cp, s.Cq, s.ntaps, M, ns, cls)
        n_part = ns * s.ntaps * s.CpPad * s.CqPad
        partial, qpart = _buf(n_part), (_buf(ns * s.CqPad) if qsum else None)
        c.call("lf_wgrad_f32", ctypes.byref(fill_wgrad(s, P, Q, partial, qpart, ns)), c.stream_ptr())
        assert bool((partial[n_part:] == SENT).all()), what + ": wrote past the partial"
        pv = partial[:n_part].view(ns, s.ntaps, s.CpPad, s.CqPad)
        body = pv[:, :, :s.Cp, :s.Cq]
        pad = torch.ones_like(pv, dtype=torch.bool)
        pad[:, :, :s.Cp, :s.Cq] = False
        assert bool(((pv[pad] == SENT) | (pv[pad] == 0)).all()), what + ": padding holds neither zero nor the sentinel"
        ranges = fc.split_ranges(M, ns, PXS)
        assert ranges[-1][1] == M
        for k, (m0, m1) in enumerate(ranges):
            if m0 == m1:
                assert bool((body[k] == 0).all()), what + ": an empty split must write exact zeros"
                if qsum:
                    assert bool((qpart[k * s.CqPad:k * s.CqPad + s.Cq] == 0).all())
                continue
            G, S, q, Sq = fc.wgrad_f32(s, P, Q, m0, m1)
            _hold(kern, what + " split %d" % k, body[k], G, fc.gate(m1 - m0, S))
            if qsum:
                _hold(kern + " qsum", what + " qsum split %d" % k, qpart[k * s.CqPad:k * s.CqPad + s.Cq], q, fc.gate(m1 - m0, Sq))
        # the reduction: into a [Cq][Cp][ntaps] weight layout, then against the sum of the partials and against fp64
        st, sp, sq = 1, s.ntaps, s.ntaps * s.Cp
        dst = _buf(s.ntaps * s.Cp * s.Cq)
        c.call("lf_wgrad_reduce", _p(partial), ns, s.ntaps, s.Cp, s.Cq, s.CpPad, s.CqPad, _p(dst), st, sp, sq, c.stream_ptr())
        off = fc.reduce_offsets(s.ntaps, s.Cp, s.Cq, st, sp, sq, DEV)
        assert _untouched(dst, off)
        rr, Sr = fc.reduce_ref(partial, ns, s.ntaps, s.Cp, s.Cq, s.CpPad, s.CqPad)
        _hold("lf_wgrad_reduce", what + " reduce", dst[off], rr, fc.gate(ns, Sr))
        _hold(kern + " reduced", what + " reduced vs fp64", dst[off], Gt, fc.gate(-(-M // ns) + PXS + ns, St))
        if qsum:
            db = _buf(s.Cq)
            c.call("lf_vec_reduce", _p(qpart), ns, s.Cq, s.CqPad, _p(db), c.stream_ptr())
            assert bool((db[s.Cq:] == SENT).all())
            _hold("lf_vec_reduce", what + " qsum reduced", db[:s.Cq], qt, fc.gate(-(-M // ns) + PXS + ns, Sqt))
    if mutate:
        bound = fc.gate(M, St)
        assert fc.excess(fc.wgrad_f32(s, P, Q, 0, M - 1)[0], Gt, bound) > 1.0
        if s.ntaps > 1:
            assert fc.excess(fc.wgrad_f32(s, P, Q, tap_shift=(s.ntaps // 2, 1))[0], Gt, bound) > 1.0


PROD_WGRAD = fc.production_wgrads(N=2, H=64, W=96)


@pytest.mark.parametrize("case", PROD_WGRAD, ids=[c[0] for c in PROD_WGRAD])
def test_wgrad_production_plans(case):
    name, plan, Hp, Wp, Cp, Hq, Wq, Cq, qs = case
    s = fc.wgrad_spec(2, plan, Hp, Wp, Cp, Hq, Wq, Cq)
    small = name in ("stem", "down16_64", "up64_16", "v3x1_c16_d1", "h1x3_c16_d1")
    run_wgrad_case(s, ("pref", 3), qs, cls=("randn", "relu", "heavy")[len(name) % 3], seed=len(name), expect_small=small,
                   mutate=True)


BRANCHES = [b for b in fc.PLAN_BRANCHES]


@pytest.mark.parametrize("key,want", BRANCHES, ids=["%d_%d_%d_%s_%d" % k for k, _ in BRANCHES])
def test_wgrad_every_plan_branch_and_refusal(key, want):
    """One shape per branch of the small-channel plan (taps on P / on Q, G = 1, 2..7, >= 8) and per refusal reason (those run
    on the tile kernel), at split counts 1, preferred, non-dividing and more than there are steps."""
    s = fc.branch_spec(key)
    run_wgrad_case(s, (1, "pref", 7, "over"), key[4], seed=sum(key[:3]), expect_small=not isinstance(want, str), mutate=True)


def test_wgrad_small_kernel_several_fetch_passes():
    s = fc.branch_spec((16, 48, 9, "p", True))
    plan, _ = fc.ws_plan(s, True)
    assert plan.passes > 1 and 2 <= plan.G <= 7
    s = fc.branch_spec((4, 16, 9, "p", True))
    plan, _ = fc.ws_plan(s, True)
    assert plan.G >= 8


@pytest.mark.parametrize("Cp,Cq", [(4, 4), (12, 16), (16, 20), (20, 12), (64, 68), (68, 128), (128, 4), (16, 64)])
@pytest.mark.parametrize("qsum", [False, True])
def test_wgrad_tile_instantiations_with_slices_and_strided_gathers(Cp, Cq, qsum):
    """Two taps gathered on both sides (so the tile kernel runs), P read with stride 2 and Q with stride 1, both operands
    channel slices of wider tensors."""
    plan = dict(Hs=11, Ws=13, psy=2, psx=2, qsy=1, qsx=1, ptaps=[(-1, 0), (0, 1)], qtaps=[(0, 0), (1, -1)])
    s = fc.wgrad_spec(3, plan, 22, 26, Cp, 11, 13, Cq, p_cstride=Cp + 8, p_coff=4, q_cstride=Cq + 12, q_coff=8)
    run_wgrad_case(s, (1, 5, "over"), qsum, seed=Cp + Cq, expect_small=False, mutate=True)


def test_wgrad_gathered_q_with_stride_two():
    """ConvTranspose2d form on the tile kernel (Cp = 64 > 16 and Cq = 32 > 16) and on the small kernel (Cq = 16)."""
    for Cq, small in ((32, False), (16, True)):
        s = fc.wgrad_spec(2, plans.convT_wgrad_plan(9, 11, 3, 1), 9, 11, 64, 18, 22, Cq, q_cstride=Cq + 4, q_coff=4)
        run_wgrad_case(s, (1, "pref", 4), False, cls="relu", seed=Cq, expect_small=small, mutate=True)


def test_reduce_multi_matches_the_single_reductions_bit_for_bit():
    c = _capi()
    g = _gen(5)
    shapes = [(7, 3, 64, 64, 64, 64), (33, 3, 16, 16, 64, 64), (5, 9, 4, 13, 64, 64), (40, 1, 1, 64, 1, 64), (1, 1, 1, 13, 1, 64),
              (12, 9, 16, 48, 64, 64), (3, 1, 128, 20, 128, 64), (9, 1, 1, 128, 1, 128)]   # (nsplit, ntaps, Cp, Cq, CpPad, CqPad)
    for njobs in (1, 8):
        jobs = (c.LfReduceJob * njobs)()
        keep = []
        for i, (ns, nt, Cp, Cq, CpPad, CqPad) in enumerate(shapes[:njobs]):
            part = torch.randn(ns * nt * CpPad * CqPad, generator=g, device=DEV)
            st, sp, sq = (Cp * Cq, Cq, 1) if i % 2 else (1, nt, nt * Cp)
            dst, single = _buf(nt * Cp * Cq), _buf(nt * Cp * Cq)
            j = jobs[i]
            j.partial, j.dst = part.data_ptr(), dst.data_ptr()
            j.nsplit, j.ntaps, j.Cp, j.Cq, j.CpPad, j.CqPad, j.st, j.sp, j.sq = ns, nt, Cp, Cq, CpPad, CqPad, st, sp, sq
            if nt == 1 and Cp == 1 and CpPad == 1:          # a bias job: what lf_vec_reduce computes
                c.call("lf_vec_reduce", _p(part), ns, Cq, CqPad, _p(single), c.stream_ptr())
            else:
                c.call("lf_wgrad_reduce", _p(part), ns, nt, Cp, Cq, CpPad, CqPad, _p(single), st, sp, sq, c.stream_ptr())
            keep.append((part, dst, single, (ns, nt, Cp, Cq, CpPad, CqPad, st, sp, sq)))
        c.call("lf_reduce_multi", jobs, njobs, c.stream_ptr())
        for part, dst, single, (ns, nt, Cp, Cq, CpPad, CqPad, st, sp, sq) in keep:
            off = fc.reduce_offsets(nt, Cp, Cq, st, sp, sq, DEV)
            assert _untouched(dst, off) and _untouched(single, off)
            rr, Sr = fc.reduce_ref(part, ns, nt, Cp, Cq, CpPad, CqPad)
            _hold("lf_reduce_multi", "reduce_multi job %s" % ((ns, nt, Cp, Cq),), dst[off], rr, fc.gate(ns, Sr))
            _hold("lf_wgrad_reduce", "single reduce %s" % ((ns, nt, Cp, Cq),), single[off], rr, fc.gate(ns, Sr))
            if not (nt == 1 and Cp == 1):                   # lf_vec_reduce sums the splits in one chain: same value, other order
                assert torch.equal(dst, single), "lf_reduce_multi differs from lf_wgrad_reduce"


@pytest.mark.parametrize("C", [1, 3, 13, 16, 128, 300])
@pytest.mark.parametrize("npix", [1, 127, 3000])
def test_colsum(C, npix):
    _colsum_case(C, npix)


def test_colsum_at_the_block_cap():
    c = _capi()
    npix = 128 * c.lib().lf_colsum_blocks(1 << 40) * 3 + 77
    assert c.lib().lf_colsum_blocks(npix) == c.lib().lf_colsum_blocks(1 << 40)
    _colsum_case(16, npix)


def _colsum_case(C, npix):
    c = _capi()
    g = _gen(C + npix)
    cstride, coff, Cpad = C + 5, 3, C + 2
    src = torch.randn(npix * cstride, generator=g, device=DEV) + 0.5
    nblk = int(c.lib().lf_colsum_blocks(npix))
    part = _buf(nblk * Cpad)
    c.call("lf_colsum", _p(src), npix, C, cstride, coff, _p(part), Cpad, c.stream_ptr())
    assert bool((part[nblk * Cpad:] == SENT).all())
    pv = part[:nblk * Cpad].view(nblk, Cpad)
    assert bool((pv[:, C:] == SENT).all()), "padding columns are not the kernel's to write"
    per = -(-npix // nblk)
    x = src.view(npix, cstride)[:, coff:coff + C].double()
    for b in range(nblk):
        rows = x[b * per:min(npix, (b + 1) * per)]
        _hold("lf_colsum", "colsum C %d npix %d block %d" % (C, npix, b), pv[b, :C], rows.sum(0), fc.gate(per, rows.abs().sum(0)))
    dst = _buf(C)
    c.call("lf_vec_reduce", _p(part), nblk, C, Cpad, _p(dst), c.stream_ptr())
    assert bool((dst[C:] == SENT).all())
    _hold("lf_vec_reduce", "colsum reduced C %d npix %d" % (C, npix), dst[:C], x.sum(0), fc.gate(per + nblk, x.abs().sum(0)))
