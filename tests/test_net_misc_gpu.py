"""The bandwidth-bound kernels of csrc/net_misc.cu driven directly through their C entry points against the fp64
restatements of tests/f32_contract.py: the BatchNorm forward chain (lf_bn_stats -> lf_bn_finalize -> lf_bn_apply /
lf_bn_apply_bf16, lf_bn_eval_prepare) and backward chain (lf_bn_bwd_reduce -> lf_bn_bwd_finalize -> lf_bn_bwd_apply /
_gated), the 2x2 max pool, its eval form and its gradient, the output ConvTranspose2d, the layout changes and
lf_pack_gather.

Outputs are pre-filled with a sentinel and followed by a sentinel guard.  The BatchNorm statistics are held to the
closed-form bound f32_contract.bn_stat_bounds derives from the kernels' arithmetic (fp32 per-thread sums of T terms,
fp64 after), on inputs whose |mean| / sigma is 0, 3, 30 and 300; the elementwise kernels are held entry by entry to a few
fp32 roundings of their own inputs; pooling, layout and packing to exact equality, on inputs full of ties.
The largest |err| / gate per kernel and the measured BatchNorm error per |mean| / sigma are printed at the end
(pytest -s)."""
import ctypes

import pytest
import torch

import f32_contract as fc

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -1.2345e30
GUARD = 1024
MEASURED = {}
ENVELOPE = {}                         # |mean|/sigma -> [largest |y - fp64| of ours, of torch's fp32 BatchNorm, of the derived bound]
U = fc.U
EPS, MOM = 1e-3, 0.1


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(MEASURED.items()):
        print("%-28s max |err| / gate %.3f" % (k, v))
    for r, (ours, ref32, bound) in sorted(ENVELOPE.items()):
        print("BatchNorm |mean|/sigma %5g: max |y - fp64| ours %.2e, torch fp32 %.2e, derived bound %.2e" % (r, ours, ref32, bound))


def _hold(kern, what, got, ref, bound):
    x = fc.excess(got, ref, bound)
    MEASURED[kern] = max(MEASURED.get(kern, 0.0), x)
    assert x <= 1.0, "%s: |err| reaches %.3g x the gate" % (what, x)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g):
    return torch.randn(shape, generator=g, device=DEV)


def _buf(n, dtype=torch.float32):
    return torch.full((n + GUARD,), SENT, dtype=dtype, device=DEV)


def _guard_ok(buf, n):
    return bool((buf[n:] == SENT).all())


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return _capi().stream_ptr()


# =====================================================================================================================
# BatchNorm
# =====================================================================================================================
def bn_case(C, npix, ratio, nimg, drop, res, relu, ymask, running, gamma_kind, seed):
    c = _capi()
    h = c.lib()
    g = _gen(seed)
    sigma = 1.5
    sign = torch.where(torch.arange(C, device=DEV) % 2 == 0, 1.0, -1.0)
    x = (_randn((npix, C), g) * sigma + ratio * sigma * sign).contiguous()
    gamma = _randn((C,), g)
    if gamma_kind == "negzero":
        gamma[0::3] = -gamma[0::3].abs()
        gamma[1::3] = 0.0
    beta = _randn((C,), g)
    ppi = npix // nimg
    assert ppi * nimg == npix
    what = "bn C %d npix %d ratio %g" % (C, npix, ratio)
    nblk = int(h.lf_bn_blocks(npix, C))
    T = fc.bn_terms_per_thread(npix, C, nblk)
    per = -(-npix // nblk)
    f = ctypes.c_float

    # ---- statistics: every block's partial on its own pixel range
    part = _buf(nblk * 2 * C, torch.float64)
    c.call("lf_bn_stats", _p(x), npix, C, _p(part), _st())
    assert _guard_ok(part, nblk * 2 * C), what
    xd = x.double()
    edges = torch.tensor([min(npix, b * per) for b in range(nblk + 1)], device=DEV)
    zero = torch.zeros(1, C, dtype=torch.float64, device=DEV)
    cs = [torch.cat([zero, t.cumsum(0)])[edges] for t in (xd, xd * xd, xd.abs())]
    b1, b2, ba = (t[1:] - t[:-1] for t in cs)
    pv = part[:nblk * 2 * C].view(nblk, 2, C)
    slack = 1e-13 * cs[2][-1][None, :]                                   # the fp64 prefix sums' own rounding
    _hold("lf_bn_stats", what + " sum x", pv[:, 0], b1, (T + 1) * U * ba + slack)
    _hold("lf_bn_stats", what + " sum x^2", pv[:, 1], b2, (T + 1) * U * b2 + 1e-13 * cs[1][-1][None, :])

    # ---- finalize
    rm0, rv0 = _randn((C,), g), _randn((C,), g).abs() + 0.5
    rm, rv = (rm0.clone(), rv0.clone()) if running else (None, None)
    st = _buf(4 * C)
    sv = st[:4 * C].view(4, C)
    c.call("lf_bn_finalize", _p(part), nblk, npix, C, _p(gamma), _p(beta), f(EPS), f(MOM), _p(rm), _p(rv), _p(sv[0]), _p(sv[1]),
           _p(sv[2]), _p(sv[3]), _st())
    assert _guard_ok(st, 4 * C)
    mean, invstd, scale, shift = sv[0], sv[1], sv[2], sv[3]
    r = fc.bn_forward(x, gamma, beta, EPS, MOM, rm0, rv0)
    dmean, dvar, rel_is = fc.bn_stat_bounds(x, T, EPS)
    dscale = gamma.double().abs() * r["invstd"] * (rel_is + 2 * U)
    dshift = r["scale"].abs() * dmean + r["mean"].abs() * dscale + 4 * U * ((r["mean"] * r["scale"]).abs() + beta.double().abs())
    _hold("lf_bn_finalize mean", what, mean, r["mean"], dmean + U * r["mean"].abs())
    _hold("lf_bn_finalize invstd", what, invstd, r["invstd"], r["invstd"] * rel_is)
    _hold("lf_bn_finalize scale", what, scale, r["scale"], dscale + 1e-300)
    _hold("lf_bn_finalize shift", what, shift, r["shift"], dshift)
    if running:
        unb = npix / max(npix - 1, 1)
        brm = MOM * dmean + 4 * U * (rm0.double().abs() + r["mean"].abs())
        brv = MOM * dvar * unb + 4 * U * (rv0.double().abs() + r["var"] * unb)
        _hold("lf_bn_finalize running", what + " running_mean", rm, r["running_mean"], brm)
        _hold("lf_bn_finalize running", what + " running_var", rv, r["running_var"], brv)
        if npix == 127 and ratio <= 3:                                   # the biased variance would be seen
            rb = fc.bn_forward(x, gamma, beta, EPS, MOM, rm0, rv0, biased_running=True)
            assert fc.excess(rb["running_var"], r["running_var"], brv) > 1.0

    # ---- apply, against the kernel's own scale / shift (a few roundings) and against the true BatchNorm (the envelope)
    dr = ((torch.rand((nimg, C), generator=g, device=DEV) > 0.3).float() / 0.7) if drop else None
    rs = _randn((npix, C), g) if res else None
    y = _buf(npix * C)
    c.call("lf_bn_apply", _p(x), npix, C, ppi, _p(scale), _p(shift), _p(dr), _p(rs), int(relu), _p(y), _st())
    assert _guard_ok(y, npix * C)
    yv = y[:npix * C].view(npix, C)
    yr, Ty = fc.bn_apply(x, scale, shift, ppi, dr, rs, relu)
    _hold("lf_bn_apply", what, yv, yr, 4 * U * Ty)
    ybf = torch.full((npix * C + GUARD,), -7.0, dtype=torch.bfloat16, device=DEV)
    c.call("lf_bn_apply_bf16", _p(x), npix, C, ppi, _p(scale), _p(shift), _p(dr), _p(rs), int(relu), _p(ybf), _st())
    assert bool((ybf[npix * C:] == -7.0).all())
    assert torch.equal(ybf[:npix * C].view(npix, C), yv.to(torch.bfloat16)), what + ": bf16 store differs from .to(bfloat16)"
    yt, Tt = fc.bn_apply(x, r["scale"], r["shift"], ppi, dr, rs, relu)
    dsc = (xd.abs() * dscale + dshift) * (1.0 if dr is None else fc._per_image(dr, npix, ppi).abs())
    _hold("lf_bn_apply vs true BN", what, yv, yt, dsc + 4 * U * Tt)
    if 1 < npix <= 4096 and not (drop or res or relu):     # the yardstick: torch's own fp32 BatchNorm on the same input
        ref32 = torch.nn.functional.batch_norm(x.cpu().t().contiguous().view(1, C, npix, 1), None, None, gamma.cpu(), beta.cpu(),
                                               True, MOM, EPS)[0, :, :, 0].t().to(DEV)
        e = ENVELOPE.setdefault(ratio, [0.0, 0.0, 0.0])
        e[0] = max(e[0], float((yv.double() - yt).abs().max()))
        e[1] = max(e[1], float((ref32.double() - yt).abs().max()))
        e[2] = max(e[2], float((dsc + 4 * U * Tt).max()))

    # ---- backward
    dy = _randn((npix, C), g)
    ym = yv.clone() if ymask else None
    bpart = _buf(nblk * 2 * C, torch.float64)
    c.call("lf_bn_bwd_reduce", _p(dy), _p(ym), _p(dr), _p(x), npix, C, ppi, _p(mean), _p(invstd), _p(bpart), _st())
    assert _guard_ok(bpart, nblk * 2 * C)
    bs = _buf(4 * C)
    bv = bs[:4 * C].view(4, C)
    c.call("lf_bn_bwd_finalize", _p(bpart), nblk, npix, C, _p(bv[0]), _p(bv[1]), _p(bv[2]), _p(bv[3]), _st())
    assert _guard_ok(bs, 4 * C)
    s1, s2, a1, a2 = fc.bn_backward_sums(dy, x, mean, invstd, ppi, ym, dr)
    g1, g2 = (T + 3) * U * a1, (T + 8) * U * a2
    _hold("lf_bn_bwd_finalize", what + " dbeta", bv[1], s1, g1)
    _hold("lf_bn_bwd_finalize", what + " dgamma", bv[0], s2, g2)
    _hold("lf_bn_bwd_finalize", what + " c1", bv[2], s1 / npix, g1 / npix)
    _hold("lf_bn_bwd_finalize", what + " c2", bv[3], s2 / npix, g2 / npix)
    dxr, gated_r, Tdx = fc.bn_backward_dx(dy, x, mean, invstd, gamma, bv[2], bv[3], ppi, ym, dr)
    dx, dx2, gated = _buf(npix * C), _buf(npix * C), _buf(npix * C)
    c.call("lf_bn_bwd_apply", _p(dy), _p(ym), _p(dr), _p(x), npix, C, ppi, _p(mean), _p(invstd), _p(gamma), _p(bv[2]), _p(bv[3]),
           _p(dx), _st())
    c.call("lf_bn_bwd_apply_gated", _p(dy), _p(ym), _p(dr), _p(x), npix, C, ppi, _p(mean), _p(invstd), _p(gamma), _p(bv[2]),
           _p(bv[3]), _p(dx2), _p(gated), _st())
    assert _guard_ok(dx, npix * C) and _guard_ok(gated, npix * C)
    _hold("lf_bn_bwd_apply", what, dx[:npix * C].view(npix, C), dxr, 8 * U * Tdx)
    assert torch.equal(dx, dx2)
    assert torch.equal(gated[:npix * C].view(npix, C).double(), gated_r), what + ": gated"


@pytest.mark.parametrize("C", [4, 12, 16, 20, 64, 128, 516, 1024])
@pytest.mark.parametrize("npix,nimg", [(1, 1), (127, 1), (385, 5), (1155, 3)])
def test_bn_chains_over_channel_counts_and_flags(C, npix, nimg):
    """Every combination of drop / res / relu / ymask is met across the grid (the flags cycle with the case number);
    385 = 128*3 + 1 pixels in 5 images of 77, so images end inside a block's pixel range."""
    k = [4, 12, 16, 20, 64, 128, 516, 1024].index(C) * 4 + [1, 127, 385, 1155].index(npix)
    bn_case(C, npix, (0, 3)[k % 2], nimg, drop=bool(k & 1), res=bool(k & 2), relu=bool(k & 4), ymask=bool(k & 8),
            running=bool((k >> 1) & 1) or npix == 127, gamma_kind=("randn", "negzero")[(k >> 2) & 1], seed=k)


@pytest.mark.parametrize("flags", range(16))
def test_bn_every_flag_combination(flags):
    bn_case(16, 385, 0, 5, drop=bool(flags & 1), res=bool(flags & 2), relu=bool(flags & 4), ymask=bool(flags & 8), running=True,
            gamma_kind="negzero", seed=100 + flags)


@pytest.mark.parametrize("ratio", [0, 3, 30, 300])
@pytest.mark.parametrize("C,npix,nimg", [(16, 127, 1), (64, 1155, 3), (128, 4096, 2), (64, 32 * 64 * 128, 32), (16, 32 * 128 * 256, 32)])
def test_bn_mean_to_sigma_envelope(ratio, C, npix, nimg):
    """Inputs with |mean| / sigma of 0, 3, 30, 300: every statistic inside the derived bound, at small sizes and at the
    two largest BatchNorm inputs of a batch-32 256 x 512 training step."""
    bn_case(C, npix, ratio, nimg, drop=False, res=False, relu=False, ymask=False, running=True, gamma_kind="randn",
            seed=ratio + C)


def test_bn_eval_prepare():
    c = _capi()
    g = _gen(3)
    for C in (1, 13, 128, 300):
        gamma, beta, rm = (_randn((C,), g) for _ in range(3))
        rv = _randn((C,), g).abs()
        out = _buf(2 * C)
        c.call("lf_bn_eval_prepare", C, _p(gamma), _p(beta), ctypes.c_float(EPS), _p(rm), _p(rv), _p(out[:C]), _p(out[C:2 * C]), _st())
        assert _guard_ok(out, 2 * C)
        sc = gamma.double() / torch.sqrt(rv.double() + EPS)
        _hold("lf_bn_eval_prepare", "scale C %d" % C, out[:C], sc, 4 * U * sc.abs() + 1e-300)
        sh = beta.double() - rm.double() * sc
        _hold("lf_bn_eval_prepare", "shift C %d" % C, out[C:2 * C], sh, 6 * U * ((rm.double() * sc).abs() + beta.double().abs()))


# =====================================================================================================================
# 2x2 max pool
# =====================================================================================================================
def _tie_input(N, H, W, cs, g):
    """post-ReLU map (half zeros) with an all-equal window, a +-0 window and the maximum at each of the four positions."""
    x = _randn((N, H, W, cs), g).clamp_min(0)
    x[:, 0:2, 0:2] = 1.5
    x[:, 0:2, 2:4] = 0.0
    x[:, 0, 2] = -0.0
    x[:, 1, 3, 0::2] = -0.0
    for k, (a, b) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        x[:, 2:4, 2 * k:2 * k + 2] = 0.25
        x[:, 2 + a, 2 * k + b] = 2.0
        x[:, 2 + a, 2 * k + b, 0] = 0.25
    return x


@pytest.mark.parametrize("C", [3, 16, 64])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_maxpool_forward_eval_form_and_first_maximum_gradient(C, accumulate):
    c = _capi()
    g = _gen(C + accumulate)
    N, H, W = 2, 12, 16
    ics, ocs, ocoff, dcs = C + 4, 2 * C + 5, C + 1, C + 2
    x = _tie_input(N, H, W, ics, g).reshape(-1)
    assert float((x == 0).float().mean()) >= 0.4
    npo = N * (H // 2) * (W // 2)
    out = _buf(npo * ocs)
    c.call("lf_maxpool2_fwd", _p(x), N, H, W, C, ics, _p(out), ocs, ocoff, _st())
    ref, off = fc.maxpool2_fwd(x, N, H, W, C, ics, ocs, ocoff)
    assert torch.equal(out[off].double(), ref), "pool forward"
    keep = torch.ones(out.numel(), dtype=torch.bool, device=DEV)
    keep[off.reshape(-1)] = False
    assert bool((out[keep] == SENT).all()), "pool forward wrote outside its channel slice"
    sc, sh = _randn((ocs,), g), _randn((ocs,), g)
    oute = _buf(npo * ocs)
    c.call("lf_maxpool2_affine_relu", _p(x), N, H, W, C, ics, _p(sc), _p(sh), _p(oute), ocs, ocoff, _st())
    refe, _ = fc.maxpool2_fwd(x, N, H, W, C, ics, ocs, ocoff, sc, sh)
    cc = torch.arange(C, device=DEV) + ocoff
    _hold("lf_maxpool2_affine_relu", "C %d" % C, oute[off], refe, 2 * U * ((ref * sc.double()[cc]).abs() + sh.double()[cc].abs()))
    assert bool((oute[keep] == SENT).all())
    # gradient: d_out is the slice of a wider tensor, d_in has its own stride
    dout = _randn((npo * ocs,), g)
    vals, offs = fc.maxpool2_bwd(x, N, H, W, C, ics, dout, ocs, ocoff, dcs)
    base = _randn((N * H * W * dcs + GUARD,), g) if accumulate else _buf(N * H * W * dcs)
    din = base.clone()
    c.call("lf_maxpool2_bwd", _p(x), N, H, W, C, ics, _p(dout), ocs, ocoff, _p(din), dcs, accumulate, _st())
    want = base.clone()
    want[offs.reshape(-1)] = (base[offs.reshape(-1)] if accumulate else 0) + vals.reshape(-1).float()
    assert torch.equal(din, want), "pool gradient (first maximum wins), untouched channels and guard"
    lastv, _ = fc.maxpool2_bwd(x, N, H, W, C, ics, dout, ocs, ocoff, dcs, last_wins=True)
    assert not torch.equal(lastv, vals)


# =====================================================================================================================
# output ConvTranspose2d(16 -> L, 2, stride 2)
# =====================================================================================================================
@pytest.mark.parametrize("L", range(1, 9))
@pytest.mark.parametrize("N,H,W", [(1, 1, 1), (1, 4095, 1), (1, 1, 4097), (2, 24, 40)])
def test_outconv(L, N, H, W):
    c = _capi()
    g = _gen(L * 7 + H)
    bias = _randn((L,), g) if (L + H) % 2 else None
    x, w = _randn((N, H, W, 16), g), _randn((16, L, 2, 2), g)
    what = "outconv L %d %dx%dx%d" % (L, N, H, W)
    n_out = N * L * 4 * H * W
    out = _buf(n_out)
    c.call("lf_outconv_fwd", _p(x), _p(w), _p(bias), N, H, W, 16, L, _p(out), _st())
    assert _guard_ok(out, n_out)
    ref, S = fc.outconv_fwd(x, w, bias)
    _hold("lf_outconv_fwd", what, out[:n_out].view_as(ref), ref, fc.gate(17, S))
    dout = _randn((N, L, 2 * H, 2 * W), g)
    dx = _buf(N * H * W * 16)
    c.call("lf_outconv_bwd_data", _p(dout), _p(w), N, H, W, 16, L, _p(dx), _st())
    assert _guard_ok(dx, N * H * W * 16)
    rdx, Sdx = fc.outconv_bwd_data(dout, w)
    _hold("lf_outconv_bwd_data", what, dx[:N * H * W * 16].view_as(rdx), rdx, fc.gate(4 * L + 4, Sdx))
    npix = N * H * W
    nblk = int(c.lib().lf_outconv_wgrad_blocks(npix))
    assert nblk == -(-npix // 4096)
    row = 16 * L * 4 + L
    part = _buf(nblk * row)
    c.call("lf_outconv_bwd_weight", _p(x), _p(dout), N, H, W, 16, L, _p(part), _st())
    assert _guard_ok(part, nblk * row)
    tw, tsw, tb, tsb = 0, 0, 0, 0
    for b in range(nblk):
        dw, Sw, db, Sb = fc.outconv_bwd_weight(x, dout, b * 4096, min(npix, (b + 1) * 4096))
        pb = part[b * row:(b + 1) * row]
        _hold("lf_outconv_bwd_weight", what + " block %d" % b, pb[:16 * L * 4].view_as(dw), dw, fc.gate(32, Sw))
        _hold("lf_outconv_bwd_weight", what + " bias block %d" % b, pb[16 * L * 4:], db, fc.gate(34, Sb))
        tw, tsw, tb, tsb = tw + dw, tsw + Sw, tb + db, tsb + Sb
    tot = part[:nblk * row].view(nblk, row).double().sum(0)
    assert fc.excess(tot[:16 * L * 4].view_as(tw), tw, fc.gate(32, tsw)) <= 1 and fc.excess(tot[16 * L * 4:], tb, fc.gate(34, tsb)) <= 1


def test_outconv_unsupported_shapes_write_nothing():
    c = _capi()
    h = c.lib()
    x, w = torch.zeros(4096, device=DEV), torch.zeros(4096, device=DEV)
    for Cin, L in ((8, 2), (16, 9)):
        out = _buf(4096)
        assert h.lf_outconv_fwd(_p(x), _p(w), None, 1, 4, 4, Cin, L, _p(out), _st()) == -2
        assert h.lf_outconv_bwd_data(_p(x), _p(w), 1, 4, 4, Cin, L, _p(out), _st()) == -2
        assert h.lf_outconv_bwd_weight(_p(x), _p(w), 1, 4, 4, Cin, L, _p(out), _st()) == -2
        torch.cuda.synchronize()
        assert bool((out == SENT).all())


# =====================================================================================================================
# layouts and packing
# =====================================================================================================================
@pytest.mark.parametrize("C,Cpad", [(3, 4), (1, 4), (4, 4)])
def test_nchw_to_nhwc_pad(C, Cpad):
    c = _capi()
    x = _randn((3, C, 7, 9), _gen(C))
    out = _buf(3 * 7 * 9 * Cpad)
    c.call("lf_nchw_to_nhwc_pad", _p(x), 3, C, 7, 9, Cpad, _p(out), _st())
    want = torch.zeros(3, 7, 9, Cpad, device=DEV)
    want[..., :C] = x.permute(0, 2, 3, 1)
    assert torch.equal(out[:want.numel()].view_as(want), want) and _guard_ok(out, want.numel())


@pytest.mark.parametrize("N,C,H,W", [(2, 13, 5, 7), (3, 40, 33, 3), (1, 1, 1, 1), (2, 64, 8, 12)])
def test_layout_round_trip(N, C, H, W):
    c = _capi()
    x = _randn((N, C, H, W), _gen(C + H))
    n = x.numel()
    nhwc, back = _buf(n), _buf(n)
    c.call("lf_nchw_to_nhwc", _p(x), N, C, H, W, _p(nhwc), _st())
    assert torch.equal(nhwc[:n].view(N, H, W, C), x.permute(0, 2, 3, 1)) and _guard_ok(nhwc, n)
    c.call("lf_nhwc_to_nchw", _p(nhwc), N, H, W, C, _p(back), _st())
    assert torch.equal(back[:n].view(N, C, H, W), x) and _guard_ok(back, n)


class LfPackJob(ctypes.Structure):
    _fields_ = [("src", ctypes.c_void_p), ("dst", ctypes.c_void_p), ("idx", ctypes.c_void_p), ("n", ctypes.c_longlong),
                ("dst_dtype", ctypes.c_int), ("pad", ctypes.c_int)]


@pytest.mark.parametrize("blocks_per_job", [1, 64])
def test_pack_gather(blocks_per_job):
    c = _capi()
    g = _gen(blocks_per_job)
    src = _randn((5000,), g) * torch.exp(_randn((5000,), g))
    src[3], src[4], src[5] = 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8        # TF32 and bf16 rounding ties
    src[6], src[7] = -(1.0 + 2.0 ** -11), 0.0
    jobs, keep = (LfPackJob * 5)(), []
    for k, (n, flag, bf) in enumerate(((1, 0, False), (300, fc.PACK_TF32_HI, False), (5000, fc.PACK_TF32_LO, False),
                                       (70001, 0, True), (4097, 0, False))):
        idx = torch.randint(0, 5000, (n,), generator=g, device=DEV, dtype=torch.int32)
        idx[:min(n, 8)] = torch.arange(min(n, 8), device=DEV, dtype=torch.int32)
        idx = idx | flag
        idx[n // 2::7] = -1
        dst = torch.full((n + GUARD,), -7.0, dtype=torch.bfloat16 if bf else torch.float32, device=DEV)
        jobs[k].src, jobs[k].dst, jobs[k].idx, jobs[k].n, jobs[k].dst_dtype = _p(src), _p(dst), _p(idx), n, int(bf)
        keep.append((idx, dst, n, flag, bf))
    assert ctypes.sizeof(LfPackJob) == 40
    dev_jobs = torch.frombuffer(bytearray(bytes(jobs)), dtype=torch.uint8).to(DEV)
    c.call("lf_pack_gather", _p(dev_jobs), 5, blocks_per_job, _st())
    for idx, dst, n, flag, bf in keep:
        want = fc.pack_gather(src, idx, bf16=bf)
        assert torch.equal(dst[:n], want), "pack job n %d flag %x" % (n, flag)
        assert bool((dst[n:] == -7.0).all())
        if flag:
            assert bool(((dst[:n].view(torch.int32) & 0x1fff) == 0).all())
    # hi + lo reproduces the value to 2^-22 relative
    hi = fc.pack_gather(src, torch.arange(5000, device=DEV, dtype=torch.int32) | fc.PACK_TF32_HI)
    lo = fc.pack_gather(src, torch.arange(5000, device=DEV, dtype=torch.int32) | fc.PACK_TF32_LO)
    assert bool(((hi.double() + lo.double() - src.double()).abs() <= 2.0 ** -22 * src.double().abs()).all())


# =====================================================================================================================
# per-image max |x| (the activation scale of an fp8 convolution whose input is not an fp8 convolution's output)
# =====================================================================================================================
AMAX_GUARD = 2.0 ** -149     # atomicMax on the float bits only raises an entry: any stray maximum overwrites this


def _amax_input(N, per_image, g):
    """[N, per_image] fp32: images at scales 10^-3 .. 10^3 with -0.0 entries; the only image of N = 1 and image 1 of
    N >= 4 hold only subnormals (of fp32 and of bf16) and -0.0, image 2 a +inf, image N // 2 only zeros (half of them
    -0.0); the last image's maximum is its last element, negative"""
    x = _randn((N, per_image), g) * (10.0 ** torch.linspace(-3, 3, N, device=DEV)).view(-1, 1)
    sub = 1 if N >= 4 else 0 if N == 1 else None
    if sub is not None:
        x[sub] = _randn((per_image,), g).clamp(-3.9, 3.9) * 2.0 ** -128
    x[:, 1::5] = -0.0
    if N >= 4:
        x[2, per_image // 3] = float("inf")
        x[N // 2] = 0.0
        x[N // 2, ::2] = -0.0
    x[-1, -1] = -2 * x[-1].abs().max()
    return x


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("N,per_image", [(1, 8), (7, 8), ("many", 8), (1, 2048 * 3 + 8), (7, 2048 * 5 + 8),
                                         ("many", 2048 + 8), (1, 4 * 1024 * 1024 + 8), (7, 4 * 1024 * 1024)])
def test_amax_per_image_exact(N, per_image, dtype):
    """lf_amax_per_image == x.abs().flatten(1).amax(1) exactly: one element per image, a tail past a multiple of the
    8 x 256 elements a CTA covers per step, several CTAs per image (4M elements), and more images than 4 x the SM count
    (one CTA each); -0.0, fp32 subnormals, +inf and an all-zero image (which keeps its 0)"""
    c = _capi()
    if N == "many":
        N = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 5
    x = _amax_input(N, per_image, _gen(N + per_image)).to(dtype)
    want = x.float().abs().flatten(1).amax(1)
    buf = torch.full((2 * GUARD + N,), AMAX_GUARD, device=DEV)
    buf[GUARD:GUARD + N] = 0
    c.call("lf_amax_per_image", _p(x), c.dtype_id(x), per_image, N, _p(buf[GUARD:]), _st())
    torch.cuda.synchronize()
    assert bool((buf[:GUARD] == AMAX_GUARD).all()) and bool((buf[GUARD + N:] == AMAX_GUARD).all()), "wrote outside amax"
    got = buf[GUARD:GUARD + N]
    assert torch.equal(got, want), (got.tolist()[:8], want.tolist()[:8])
    if N >= 4:
        assert got[N // 2] == 0 and got[2] == float("inf") and 0 < float(got[1]) < 2.0 ** -126
    if N == 1:
        assert 0 < float(got[0]) < 2.0 ** -125
    # amax[n] = max(amax[n], ...): a second pass over the same input changes nothing
    c.call("lf_amax_per_image", _p(x), c.dtype_id(x), per_image, N, _p(buf[GUARD:]), _st())
    torch.cuda.synchronize()
    assert torch.equal(buf[GUARD:GUARD + N], want)
