"""The fp64 restatements of tests/f32_contract.py checked without a GPU: against torch's own float64 convolutions,
BatchNorm, pooling and autograd; the mutations the GPU cases rely on move the fp64 result by more than the gate; the
host-side argument checks of the CUDA-core entry points refuse what they guard (no launch); and the kernel choice of
lf_wgrad_f32 for every production weight-gradient shape is pinned."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import f32_contract as fc
from lanedetection_end2end_b200 import net_plans as plans

F64 = torch.float64
TOL = 1e-12


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rand(shape, g):
    return torch.randn(shape, generator=g, dtype=F64)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _run_phases(phases, x_nhwc, wmat, Cout, Hout, Wout, bias=None):
    """Every phase of a plan through fc.conv_f32 into one NHWC fp64 output (unwritten entries stay NaN)."""
    N, Hin, Win, Cin = x_nhwc.shape
    out = torch.full((N * Hout * Wout * Cout,), float("nan"), dtype=F64)
    for ph in phases:
        s = fc.conv_spec(N, Hin, Win, Cin, Hout, Wout, Cout, wmat.shape[2], ph)
        ref, _, off = fc.conv_f32(s, x_nhwc.reshape(-1), wmat.reshape(-1), bias)
        out[off] = ref
    return out.view(N, Hout, Wout, Cout)


def _pad_cols(w, pad):
    return F.pad(w, (0, pad - w.shape[2])).contiguous()


# layer kinds of ERFNet: (name, Cin, Cout, kh, kw, stride, ph, pw, dh, dw, H, W)
CONVS = [("stem", 3, 13, 3, 3, 2, 1, 1, 1, 1, 12, 14), ("down", 16, 48, 3, 3, 2, 1, 1, 1, 1, 10, 8),
         ("head3x3", 8, 6, 3, 3, 1, 1, 1, 1, 1, 7, 9), ("head1x1", 8, 8, 1, 1, 1, 0, 0, 1, 1, 5, 6)]
CONVS += [("v3x1_d%d" % d, 8, 8, 3, 1, 1, d, 0, d, 1, 9, 11) for d in (1, 2, 4, 8, 16)]
CONVS += [("h1x3_d%d" % d, 8, 8, 1, 3, 1, 0, d, 1, d, 9, 11) for d in (1, 2, 4, 8, 16)]


@pytest.mark.parametrize("case", CONVS, ids=[c[0] for c in CONVS])
def test_conv_restatement_matches_torch_forward_and_input_gradient(case):
    _, Ci, Co, kh, kw, st, ph, pw, dh, dw, H, W = case
    g = _g(len(case[0]) + Ci)
    x = _rand((2, Ci, H, W), g).requires_grad_()
    w, b = _rand((Co, Ci, kh, kw), g), _rand((Co,), g)
    y = F.conv2d(x, w, b, stride=st, padding=(ph, pw), dilation=(dh, dw))
    phases, (Ho, Wo) = plans.conv_fwd_plan(H, W, kh, kw, st, ph, pw, dh, dw)
    assert (Ho, Wo) == tuple(y.shape[2:])
    wf = _pad_cols(w.permute(2, 3, 1, 0).reshape(kh * kw, Ci, Co), 64)
    got = _run_phases(phases, _nhwc(x.detach()), wf, Co, Ho, Wo, b)
    assert (got - _nhwc(y.detach())).abs().max() < TOL
    dy = _rand(y.shape, g)
    dx, = torch.autograd.grad(y, x, dy)
    wd = _pad_cols(w.permute(2, 3, 0, 1).reshape(kh * kw, Co, Ci), 64)
    if st == 1:
        dphases, _ = plans.conv_dgrad_plan_s1(H, W, kh, kw, ph, pw, dh, dw)
    else:
        dphases, _ = plans.transposed_gather_plan(Ho, Wo, H, W, kh, ph)
    gd = _run_phases(dphases, _nhwc(dy), wd, Ci, H, W)
    assert not torch.isnan(gd).any(), "the phases cover every input pixel"
    assert (gd - _nhwc(dx)).abs().max() < TOL


@pytest.mark.parametrize("H,W", [(5, 6), (4, 7)])
def test_conv_restatement_matches_conv_transpose(H, W):
    g = _g(H * 10 + W)
    Ci, Co = 8, 5
    x = _rand((2, Ci, H, W), g).requires_grad_()
    w, b = _rand((Ci, Co, 3, 3), g), _rand((Co,), g)
    y = F.conv_transpose2d(x, w, b, stride=2, padding=1, output_padding=1)
    phases, (Hb, Wb) = plans.transposed_gather_plan(H, W, 2 * H, 2 * W, 3, 1)
    assert len(phases) == 4 and (Hb, Wb) == tuple(y.shape[2:])
    wf = _pad_cols(w.permute(2, 3, 0, 1).reshape(9, Ci, Co), 16)
    got = _run_phases(phases, _nhwc(x.detach()), wf, Co, Hb, Wb, b)
    assert not torch.isnan(got).any()
    assert (got - _nhwc(y.detach())).abs().max() < TOL
    dy = _rand(y.shape, g)
    dx, = torch.autograd.grad(y, x, dy)
    dphases, _ = plans.convT_dgrad_plan(Hb, Wb, H, W, 3, 1)
    wd = _pad_cols(w.permute(2, 3, 1, 0).reshape(9, Co, Ci), 16)
    gd = _run_phases(dphases, _nhwc(dy), wd, Ci, H, W)
    assert (gd - _nhwc(dx)).abs().max() < TOL


def test_conv_restatement_epilogue_order_and_slices():
    """+bias, ReLU, *(mask_src > 0), +add_src*(add_mask > 0), into a channel slice of a wider tensor."""
    g = _g(5)
    N, H, W, Ci, Co, cs, coff = 2, 4, 5, 4, 6, 12, 4
    x, w, b = _rand((N, H, W, Ci), g), _rand((1, Ci, 16), g), _rand((Co,), g)
    mask, add, amask = (_rand((N * H * W * cs,), g) for _ in range(3))
    ph = plans.conv_fwd_plan(H, W, 1, 1)[0][0]
    s = fc.conv_spec(N, H, W, Ci, H, W, Co, 16, ph, out_cstride=cs, out_coff=coff, relu=1)
    ref, S, off = fc.conv_f32(s, x.reshape(-1), w.reshape(-1), b, mask, add, amask)
    conv = (x.reshape(-1, Ci) @ w[0, :, :Co] + b).clamp_min(0)
    m3, a3, am3 = (t.view(-1, cs)[:, coff:coff + Co] for t in (mask, add, amask))
    want = conv * (m3 > 0) + a3 * (am3 > 0)
    assert (ref - want).abs().max() < TOL
    assert torch.equal(off, (torch.arange(N * H * W)[:, None] * cs + coff + torch.arange(Co)[None, :]))
    assert (S >= ref.abs() - 1e-12).all()


@pytest.mark.parametrize("case", CONVS, ids=[c[0] for c in CONVS])
def test_wgrad_restatement_matches_autograd(case):
    _, Ci, Co, kh, kw, st, ph, pw, dh, dw, H, W = case
    g = _g(77 + Ci + kh)
    x = _rand((2, Ci, H, W), g)
    w = _rand((Co, Ci, kh, kw), g).requires_grad_()
    b = _rand((Co,), g).requires_grad_()
    y = F.conv2d(x, w, b, stride=st, padding=(ph, pw), dilation=(dh, dw))
    dy = _rand(y.shape, g)
    dw_, db_ = torch.autograd.grad(y, (w, b), dy)
    plan = plans.conv_wgrad_plan(H, W, kh, kw, st, ph, pw, dh, dw)
    s = fc.wgrad_spec(2, plan, H, W, Ci, y.shape[2], y.shape[3], Co)
    G, S, qsum, _ = fc.wgrad_f32(s, _nhwc(x).reshape(-1), _nhwc(dy).reshape(-1))
    assert (G - dw_.permute(2, 3, 1, 0).reshape(kh * kw, Ci, Co)).abs().max() < 1e-11
    assert (qsum - db_).abs().max() < 1e-11
    # summed over any split of the pixels it is the same gradient
    M = 2 * s.Hs * s.Ws
    parts = [fc.wgrad_f32(s, _nhwc(x).reshape(-1), _nhwc(dy).reshape(-1), a, b_)[0] for a, b_ in fc.split_ranges(M, 3, 16)]
    assert (sum(parts) - G).abs().max() < 1e-11


def test_wgrad_restatement_matches_conv_transpose_autograd():
    g = _g(9)
    Ci, Co, H, W = 8, 4, 5, 6
    x = _rand((2, Ci, H, W), g)
    w = _rand((Ci, Co, 3, 3), g).requires_grad_()
    y = F.conv_transpose2d(x, w, None, stride=2, padding=1, output_padding=1)
    dy = _rand(y.shape, g)
    dw_, = torch.autograd.grad(y, w, dy)
    s = fc.wgrad_spec(2, plans.convT_wgrad_plan(H, W, 3, 1), H, W, Ci, 2 * H, 2 * W, Co)
    G, _, _, _ = fc.wgrad_f32(s, _nhwc(x).reshape(-1), _nhwc(dy).reshape(-1))
    assert (G - dw_.permute(2, 3, 0, 1).reshape(9, Ci, Co)).abs().max() < 1e-11


def test_reduce_restatement_and_layout():
    g = _g(3)
    ns, nt, Cp, Cq = 5, 3, 6, 7
    part = _rand((ns, nt, 64, 64), g).float()
    ref, S = fc.reduce_ref(part.reshape(-1), ns, nt, Cp, Cq, 64, 64)
    assert (ref - part.double()[:, :, :Cp, :Cq].sum(0)).abs().max() < TOL and (S >= ref.abs()).all()
    off = fc.reduce_offsets(nt, Cp, Cq, 1, nt * Cq, nt)          # [Cp][Cq][nt] destination
    dst = torch.zeros(nt * Cp * Cq, dtype=F64)
    dst[off] = ref
    assert torch.equal(dst.view(Cp, Cq, nt), ref.permute(1, 2, 0))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("npix,C", [(1, 4), (37, 12), (200, 20)])
def test_batchnorm_restatement_matches_torch(npix, C):
    g = _g(npix + C)
    x = (_rand((npix, C), g) * 2 + 3).requires_grad_()
    bn = torch.nn.BatchNorm2d(C, eps=1e-3, momentum=0.1).double().train()
    with torch.no_grad():
        bn.weight.copy_(_rand((C,), g))
        bn.bias.copy_(_rand((C,), g))
        bn.running_mean.copy_(_rand((C,), g))
        bn.running_var.copy_(_rand((C,), g).abs() + 0.5)
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    xin = x.t().contiguous().view(1, C, npix, 1)          # contiguous: ATen's CPU backward misreads a transposed gradient
    if npix == 1:
        r = fc.bn_forward(x.detach(), bn.weight, bn.bias, 1e-3, 0.1, rm0, rv0)       # torch refuses one value per channel
        assert r["var"].abs().max() == 0 and (r["running_var"] - 0.9 * rv0).abs().max() < TOL
        return
    res, drop = _rand((npix, C), g), (torch.rand((1, C), generator=g, dtype=F64) > 0.3).double() / 0.7
    y = F.relu(bn(xin)[0, :, :, 0].t() * drop + res)
    r = fc.bn_forward(x.detach(), bn.weight, bn.bias, 1e-3, 0.1, rm0, rv0)
    assert (r["running_mean"] - bn.running_mean).abs().max() < TOL and (r["running_var"] - bn.running_var).abs().max() < TOL
    got, _ = fc.bn_apply(x.detach(), r["scale"], r["shift"], npix, drop, res, relu=True)
    assert (got - y.detach()).abs().max() < 1e-11
    dy = _rand((npix, C), g)
    dx, dgam, dbet = torch.autograd.grad(y, (x, bn.weight, bn.bias), dy)
    s1, s2, _, _ = fc.bn_backward_sums(dy, x.detach(), r["mean"], r["invstd"], npix, ymask=y.detach(), drop=drop)
    assert (s1 - dbet).abs().max() < 1e-10 and (s2 - dgam).abs().max() < 1e-10
    gdx, gated, _ = fc.bn_backward_dx(dy, x.detach(), r["mean"], r["invstd"], bn.weight.detach(), s1 / npix, s2 / npix, npix,
                                      ymask=y.detach(), drop=drop)
    assert (gdx - dx).abs().max() < 1e-10
    assert torch.equal(gated, dy * (y.detach() > 0))
    # the mutation: the biased variance in the running statistic is off by var/(n-1) * momentum
    rb = fc.bn_forward(x.detach(), bn.weight, bn.bias, 1e-3, 0.1, rm0, rv0, biased_running=True)
    assert ((rb["running_var"] - r["running_var"]).abs() > 1e-3 * r["running_var"].abs() / npix).all()


def _tie_input(N, H, W, C, g):
    """post-ReLU-like map: >= 50 % zeros, all-equal windows, -0 / +0, the maximum in each of the four positions."""
    x = torch.randn((N, H, W, C), generator=g).clamp_min(0)
    x[:, 0:2, 0:2] = 1.5                       # all-equal window
    x[:, 0:2, 2:4] = 0.0
    x[:, 0, 2] = -0.0                          # +-0 window
    for k, (a, b) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        x[:, 2:4, 2 * k:2 * k + 2] = 0.25
        x[:, 2 + a, 2 * k + b] = 2.0           # unique maximum at position k
        x[:, 2 + a, 2 * k + b, 0] = 0.25       # ... and channel 0 all equal
    return x


@pytest.mark.parametrize("C", [3, 16])
def test_pool_restatement_matches_aten_on_ties(C):
    g = _g(C)
    N, H, W = 2, 6, 8
    x = _tie_input(N, H, W, C, g).double()
    assert (x == 0).double().mean() >= 0.3
    xt = x.permute(0, 3, 1, 2).contiguous().requires_grad_()
    y = F.max_pool2d(xt, 2, 2)
    got, off = fc.maxpool2_fwd(x.reshape(-1), N, H, W, C, C, C, 0)
    assert torch.equal(got.view(N, H // 2, W // 2, C), _nhwc(y.detach()))
    dy = _rand(y.shape, g)
    dx, = torch.autograd.grad(y, xt, dy)
    vals, offs = fc.maxpool2_bwd(x.reshape(-1), N, H, W, C, C, _nhwc(dy).reshape(-1), C, 0, C)
    din = torch.zeros(N * H * W * C, dtype=F64)
    din[offs.reshape(-1)] = vals.reshape(-1)
    assert torch.equal(din.view(N, H, W, C), _nhwc(dx))
    lv, _ = fc.maxpool2_bwd(x.reshape(-1), N, H, W, C, C, _nhwc(dy).reshape(-1), C, 0, C, last_wins=True)
    assert not torch.equal(lv, vals), "the input has ties, so the last-maximum mutation is visible"
    # eval form
    sc, sh = _rand((C + 4,), g), _rand((C + 4,), g)
    ga, _ = fc.maxpool2_fwd(x.reshape(-1), N, H, W, C, C, C + 4, 4, sc, sh)
    assert (ga.view(N, H // 2, W // 2, C) - (_nhwc(y.detach()) * sc[4:] + sh[4:]).clamp_min(0)).abs().max() < TOL


@pytest.mark.parametrize("L", [1, 4, 8])
def test_outconv_restatement_matches_torch(L):
    g = _g(L)
    N, H, W, Ci = 2, 3, 5, 16
    x = _rand((N, Ci, H, W), g).requires_grad_()
    w = _rand((Ci, L, 2, 2), g).requires_grad_()
    b = _rand((L,), g).requires_grad_()
    y = F.conv_transpose2d(x, w, b, stride=2)
    o, S = fc.outconv_fwd(_nhwc(x.detach()), w.detach(), b.detach())
    assert (o - y.detach()).abs().max() < TOL and (S >= o.abs() - 1e-12).all()
    dy = _rand(y.shape, g)
    dx, dw, db = torch.autograd.grad(y, (x, w, b), dy)
    gx, _ = fc.outconv_bwd_data(dy, w.detach())
    assert (gx - _nhwc(dx)).abs().max() < 1e-11
    gw, _, gb, _ = fc.outconv_bwd_weight(_nhwc(x.detach()), dy)
    assert (gw - dw).abs().max() < 1e-11 and (gb - db).abs().max() < 1e-11
    a = fc.outconv_bwd_weight(_nhwc(x.detach()), dy, 0, 7)
    c = fc.outconv_bwd_weight(_nhwc(x.detach()), dy, 7, None)
    assert (a[0] + c[0] - dw).abs().max() < 1e-11 and (a[2] + c[2] - db).abs().max() < 1e-11


def test_pack_gather_restatement():
    g = _g(1)
    src = torch.randn(64, generator=g)
    src[3] = 1.0 + 2.0 ** -11                                   # a TF32 tie: exactly half a TF32 ulp above 1
    src[4] = 1.0 + 2.0 ** -8                                    # a bf16 tie (even neighbour below)
    src[5] = 1.0 + 3 * 2.0 ** -8                                # a bf16 tie (even neighbour above)
    idx = torch.arange(64, dtype=torch.int32)
    hi = fc.pack_gather(src, idx | fc.PACK_TF32_HI)
    lo = fc.pack_gather(src, idx | fc.PACK_TF32_LO)
    assert ((hi.view(torch.int32) & 0x1fff) == 0).all() and ((lo.view(torch.int32) & 0x1fff) == 0).all()
    assert ((hi.double() + lo.double() - src.double()).abs() <= 2.0 ** -22 * src.double().abs()).all()
    assert hi[3] == 1.0 + 2.0 ** -10
    plain = fc.pack_gather(src, torch.tensor([2, -1, 7], dtype=torch.int32))
    assert torch.equal(plain, torch.stack([src[2], torch.tensor(0.0), src[7]]))
    bf = fc.pack_gather(src, idx, bf16=True)
    assert bf.dtype == torch.bfloat16 and float(bf[4]) == 1.0 and float(bf[5]) == 1.0 + 2.0 ** -6


# ---------------------------------------------------------------------------------------------------------------------
# the mutations of the GPU cases are visible through the gate
# ---------------------------------------------------------------------------------------------------------------------
def test_conv_mutations_exceed_the_gate():
    g = _g(11)
    N, Hb, Wb, Ci, Co = 2, 10, 12, 8, 12
    phases, _ = plans.transposed_gather_plan(5, 6, Hb, Wb, 3, 1)
    x, w = _rand((N, 5, 6, Ci), g).float(), _rand((9, Ci, 16), g).float()
    ph = [p for p in phases if p["oy0"] != p["ox0"]][0]
    s = fc.conv_spec(N, 5, 6, Ci, Hb, Wb, Co, 16, ph, out_cstride=16, out_coff=4)
    ref, S, off = fc.conv_f32(s, x.reshape(-1), w.reshape(-1))
    bound = fc.gate(fc.conv_ksteps(s), S)
    buf = torch.zeros(N * Hb * Wb * 16, dtype=F64)
    buf[off] = ref

    def moved(**kw):
        r2, _, o2 = fc.conv_f32(s, x.reshape(-1), w.reshape(-1), **kw)
        b2 = torch.zeros_like(buf)
        b2[o2] = r2
        return fc.excess(b2[off], ref, bound)
    assert moved(m_limit=ref.shape[0] - 3) > 1
    assert moved(tap_shift=(0, 1)) > 1
    assert moved(ignore_coff=True) > 1
    s2 = fc.conv_spec(N, 5, 6, Ci, Hb, Wb, Co, 16, dict(ph, oy0=ph["ox0"], ox0=ph["oy0"]), out_cstride=16, out_coff=4)
    r2, _, o2 = fc.conv_f32(s2, x.reshape(-1), w.reshape(-1))
    b2 = torch.zeros_like(buf)
    b2[o2] = r2
    assert fc.excess(b2[off], ref, bound) > 1


def test_wgrad_mutations_exceed_the_gate():
    g = _g(12)
    N, H, W = 2, 9, 10
    plan = plans.conv_wgrad_plan(H, W, 1, 3, 1, 0, 2, 1, 2)
    s = fc.wgrad_spec(N, plan, H, W, 8, H, W, 8)
    P, Q = _rand((N * H * W * 8,), g).float(), _rand((N * H * W * 8,), g).float()
    G, S, _, _ = fc.wgrad_f32(s, P, Q)
    bound = fc.gate(N * H * W, S)
    assert fc.excess(fc.wgrad_f32(s, P, Q, 0, N * H * W - 1)[0], G, bound) > 1       # last pixel dropped
    assert fc.excess(fc.wgrad_f32(s, P, Q, tap_shift=(1, 1))[0], G, bound) > 1


def test_bn_envelope_is_monotone_and_finite():
    assert fc.bn_envelope_ratio(32) > fc.bn_envelope_ratio(128) > 1
    assert fc.bn_terms_per_thread(32 * 64 * 128, 64, 528) == 32
    assert fc.bn_terms_per_thread(127, 1024, 1) == 127


# ---------------------------------------------------------------------------------------------------------------------
# host-side argument checks: refused before any launch
# ---------------------------------------------------------------------------------------------------------------------
def _lib():
    from lanedetection_end2end_b200 import _capi
    return _capi, _capi.lib()


P_ = ctypes.c_void_p(4096)            # a non-NULL pointer that is never dereferenced (every call below is refused first)


def _conv_args(c, **kw):
    a = c.LfConvArgs()
    a.inp = a.wmat = a.out = 4096
    a.N, a.Hin, a.Win, a.Cin, a.in_cstride = 1, 4, 4, 4, 4
    a.Hout, a.Wout, a.out_cstride, a.out_coff, a.Cout, a.CoutPad = 4, 4, 16, 0, 13, 16
    a.Hs, a.Ws, a.osy, a.osx, a.isy, a.isx, a.ntaps = 4, 4, 1, 1, 1, 1, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_conv_f32_refuses_bad_arguments():
    c, h = _lib()
    assert h.lf_conv_f32(None, None) == -1
    for kw in (dict(inp=None), dict(wmat=None), dict(out=None), dict(N=0), dict(Hs=0), dict(Ws=0), dict(Cin=0), dict(Cout=0),
               dict(ntaps=0), dict(ntaps=10), dict(Cin=6), dict(in_cstride=6), dict(out_cstride=18), dict(out_coff=2),
               dict(CoutPad=24), dict(CoutPad=16, Cout=17), dict(N=1 << 15, Hs=1 << 8, Ws=1 << 8)):
        assert h.lf_conv_f32(ctypes.byref(_conv_args(c, **kw)), None) == -1, kw


def _wgrad_args(c, **kw):
    a = c.LfWgradArgs()
    a.P = a.Q = a.partial = 4096
    a.N, a.Hs, a.Ws, a.ntaps, a.nsplit = 1, 4, 4, 1, 1
    a.Hp, a.Wp, a.Cp, a.p_cstride, a.psy, a.psx = 4, 4, 8, 8, 1, 1
    a.Hq, a.Wq, a.Cq, a.q_cstride, a.qsy, a.qsx = 4, 4, 8, 8, 1, 1
    a.CpPad = a.CqPad = 64
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_wgrad_and_reductions_refuse_bad_arguments():
    c, h = _lib()
    assert h.lf_wgrad_f32(None, None) == -1 and h.lf_wgrad_f32_nsplit(None) == 0
    for kw in (dict(P=None), dict(Q=None), dict(partial=None), dict(N=0), dict(Hs=0), dict(Ws=0), dict(ntaps=0), dict(ntaps=10),
               dict(nsplit=0), dict(Cp=6), dict(Cq=6), dict(p_cstride=6), dict(q_cstride=6), dict(p_coff=2), dict(q_coff=2),
               dict(CpPad=32), dict(CqPad=96), dict(Cp=68), dict(Cq=68), dict(N=1 << 15, Hs=1 << 8, Ws=1 << 8)):
        assert h.lf_wgrad_f32(ctypes.byref(_wgrad_args(c, **kw)), None) == -1, kw
    ok = dict(partial=P_, nsplit=1, ntaps=1, Cp=4, Cq=4, CpPad=64, CqPad=64, dst=P_, st=16, sp=4, sq=1)
    for kw in (dict(partial=None), dict(dst=None), dict(nsplit=0), dict(ntaps=0), dict(Cp=0), dict(Cq=0), dict(CqPad=66)):
        v = dict(ok, **kw)
        assert h.lf_wgrad_reduce(v["partial"], v["nsplit"], v["ntaps"], v["Cp"], v["Cq"], v["CpPad"], v["CqPad"], v["dst"],
                                 v["st"], v["sp"], v["sq"], None) == -1, kw
        jobs = (c.LfReduceJob * 2)()
        for j in jobs:
            j.partial = j.dst = 4096
            j.nsplit, j.ntaps, j.Cp, j.Cq, j.CpPad, j.CqPad, j.st, j.sp, j.sq = 1, 1, 4, 4, 64, 64, 16, 4, 1
        for k, val in kw.items():
            setattr(jobs[1], k, val.value if isinstance(val, ctypes.c_void_p) else val)
        assert h.lf_reduce_multi(jobs, 2, None) == -1, kw
    jobs = (c.LfReduceJob * 1)()
    assert h.lf_reduce_multi(None, 1, None) == -1 and h.lf_reduce_multi(jobs, 0, None) == -1
    assert h.lf_reduce_multi(jobs, c.REDUCE_MAX_JOBS + 1, None) == -1
    for a in ((None, 1, 4, 4, P_), (P_, 1, 4, 4, None), (P_, 0, 4, 4, P_), (P_, 1, 0, 4, P_), (P_, 1, 5, 4, P_)):
        assert h.lf_vec_reduce(*a, None) == -1, a
    for a in ((None, 4, 4, 4, 0, P_, 4), (P_, 4, 4, 4, 0, None, 4), (P_, 0, 4, 4, 0, P_, 4), (P_, 4, 0, 4, 0, P_, 4),
              (P_, 4, 5, 8, 0, P_, 4)):
        assert h.lf_colsum(*a, None) == -1, a


def test_net_misc_refuses_bad_arguments():
    c, h = _lib()
    f = ctypes.c_float
    for npix, C in ((0, 16), (8, 0), (8, 6), (8, 1028)):
        assert h.lf_bn_stats(P_, npix, C, P_, None) == -1
        assert h.lf_bn_apply(P_, npix, C, 1, P_, P_, None, None, 0, P_, None) == -1
        assert h.lf_bn_apply_bf16(P_, npix, C, 1, P_, P_, None, None, 0, P_, None) == -1
        assert h.lf_bn_bwd_reduce(P_, None, None, P_, npix, C, 1, P_, P_, P_, None) == -1
        assert h.lf_bn_bwd_apply(P_, None, None, P_, npix, C, 1, P_, P_, P_, P_, P_, P_, None) == -1
        assert h.lf_bn_bwd_apply_gated(P_, None, None, P_, npix, C, 1, P_, P_, P_, P_, P_, P_, P_, None) == -1
        # the finalize kernels divide by npix and size their grid from C
        assert h.lf_bn_finalize(P_, 1, npix, C, P_, P_, f(1e-3), f(0.1), None, None, P_, P_, P_, P_, None) == -1, (npix, C)
        assert h.lf_bn_bwd_finalize(P_, 1, npix, C, P_, P_, P_, P_, None) == -1, (npix, C)
    assert h.lf_bn_stats(None, 8, 16, P_, None) == -1 and h.lf_bn_stats(P_, 8, 16, None, None) == -1
    assert h.lf_bn_apply(P_, 8, 16, 0, P_, P_, None, None, 0, P_, None) == -1            # pix_per_image
    assert h.lf_bn_apply(P_, 8, 16, 1, P_, P_, None, None, 0, None, None) == -1
    assert h.lf_bn_bwd_reduce(P_, None, None, P_, 8, 16, 0, P_, P_, P_, None) == -1
    assert h.lf_bn_bwd_apply_gated(P_, None, None, P_, 8, 16, 1, P_, P_, P_, P_, P_, P_, None, None) == -1
    assert h.lf_bn_finalize(P_, 0, 8, 16, P_, P_, f(1e-3), f(0.1), None, None, P_, P_, P_, P_, None) == -1
    assert h.lf_bn_finalize(P_, 1, 8, 16, P_, P_, f(1e-3), f(0.1), P_, None, P_, P_, P_, P_, None) == -1   # one running_* only
    assert h.lf_bn_bwd_finalize(P_, 0, 8, 16, P_, P_, P_, P_, None) == -1
    assert h.lf_bn_eval_prepare(0, P_, P_, f(1e-3), P_, P_, P_, P_, None) == -1
    assert h.lf_bn_eval_prepare(4, P_, P_, f(1e-3), None, P_, P_, P_, None) == -1
    for N, H, W, C in ((0, 4, 4, 4), (1, 1, 4, 4), (1, 4, 1, 4), (1, 4, 4, 0), (1, 5, 4, 4), (1, 4, 6 + 1, 4)):
        assert h.lf_maxpool2_fwd(P_, N, H, W, C, 4, P_, 4, 0, None) == -1
        assert h.lf_maxpool2_affine_relu(P_, N, H, W, C, 4, P_, P_, P_, 4, 0, None) == -1
        assert h.lf_maxpool2_bwd(P_, N, H, W, C, 4, P_, 4, 0, P_, 4, 0, None) == -1
    assert h.lf_maxpool2_affine_relu(P_, 1, 4, 4, 4, 4, None, P_, P_, 4, 0, None) == -1
    for Cin, L in ((8, 2), (16, 9), (16, 0)):          # refused as unsupported, before any launch
        assert h.lf_outconv_fwd(P_, P_, None, 1, 4, 4, Cin, L, P_, None) == -2
        assert h.lf_outconv_bwd_data(P_, P_, 1, 4, 4, Cin, L, P_, None) == -2
        assert h.lf_outconv_bwd_weight(P_, P_, 1, 4, 4, Cin, L, P_, None) == -2
    assert h.lf_outconv_fwd(None, P_, None, 1, 4, 4, 16, 2, P_, None) == -1
    assert h.lf_outconv_bwd_data(P_, P_, 0, 4, 4, 16, 2, P_, None) == -1
    assert h.lf_outconv_bwd_weight(P_, P_, 1, 4, 0, 16, 2, P_, None) == -1
    assert h.lf_nchw_to_nhwc_pad(P_, 1, 4, 4, 4, 3, P_, None) == -1                      # Cpad < C
    assert h.lf_nchw_to_nhwc_pad(P_, 0, 3, 4, 4, 4, P_, None) == -1
    assert h.lf_nhwc_to_nchw(P_, 0, 4, 4, 4, P_, None) == -1 and h.lf_nchw_to_nhwc(None, 1, 4, 4, 4, P_, None) == -1
    assert h.lf_nhwc_to_nchw(P_, 70000, 4, 4, 4, P_, None) == -1
    assert h.lf_pack_gather(None, 1, 1, None) == -1 and h.lf_pack_gather(P_, 0, 1, None) == -1
    assert h.lf_pack_gather(P_, 1, 0, None) == -1 and h.lf_pack_gather(P_, 70000, 1, None) == -1
    # lf_amax_per_image: 8 elements per step (per_image % 8), one grid row per image (N <= 65535), fp32 / bf16 only
    for a in ((None, 0, 8, 1, P_), (P_, 0, 8, 1, None), (P_, 0, 12, 1, P_), (P_, 1, 4, 1, P_), (P_, 0, 0, 1, P_),
              (P_, 0, -8, 1, P_), (P_, 0, 8, 0, P_), (P_, 0, 8, -1, P_), (P_, 0, 8, 65536, P_), (P_, 2, 8, 1, P_),
              (P_, -1, 8, 1, P_)):
        assert h.lf_amax_per_image(*a, None) == -1, a


# ---------------------------------------------------------------------------------------------------------------------
# which kernel serves each production weight gradient (fp32 convolution mode)
# ---------------------------------------------------------------------------------------------------------------------
SMALL_KERNEL_LAYERS = {"stem", "down16_64", "up64_16", "v3x1_c16_d1", "h1x3_c16_d1"}


def _fill_wgrad(c, s, want_qsum):
    a = c.LfWgradArgs()
    for k in ("N", "Hs", "Ws", "Hp", "Wp", "Cp", "p_cstride", "p_coff", "psy", "psx", "Hq", "Wq", "Cq", "q_cstride", "q_coff",
              "qsy", "qsx", "ntaps", "CpPad", "CqPad", "nsplit"):
        setattr(a, k, getattr(s, k))
    for t in range(s.ntaps):
        a.pdy[t], a.pdx[t], a.qdy[t], a.qdx[t] = s.pdy[t], s.pdx[t], s.qdy[t], s.qdx[t]
    a.qsum_partial = 1 if want_qsum else None
    return a


def test_production_weight_gradients_keep_their_kernel():
    c, h = _lib()
    sms = h.lf_bn_blocks(1 << 40, 4) // 4
    small = set()
    for name, plan, Hp, Wp, Cp, Hq, Wq, Cq, qs in fc.production_wgrads():
        s = fc.wgrad_spec(2, plan, Hp, Wp, Cp, Hq, Wq, Cq)
        pl, why = fc.ws_plan(s, qs)
        pref = h.lf_wgrad_f32_nsplit(ctypes.byref(_fill_wgrad(c, s, qs)))
        assert (pref > 0) == (pl is not None), (name, pref, why)
        if pl is not None:
            small.add(name)
            M = 2 * s.Hs * s.Ws
            assert pref == max(1, min(2 * sms, -(-M // (4 * pl.PXS)))), (name, pref, pl)
    assert small == SMALL_KERNEL_LAYERS, small ^ SMALL_KERNEL_LAYERS


@pytest.mark.parametrize("key,want", fc.PLAN_BRANCHES, ids=["%d_%d_%d_%s_%d" % k for k, _ in fc.PLAN_BRANCHES])
def test_plan_branches(key, want):
    c, h = _lib()
    s = fc.branch_spec(key)
    pl, why = fc.ws_plan(s, key[4])
    pref = h.lf_wgrad_f32_nsplit(ctypes.byref(_fill_wgrad(c, s, key[4])))
    if isinstance(want, str):
        assert pl is None and why == want and pref == 0
    else:
        assert pl is not None and pref > 0
        assert (pl.taps_on_p, pl.G) == (want["taps_on_p"], want["G"]), pl
