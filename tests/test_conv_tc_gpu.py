"""GPU tests of the tensor-core (TF32) 3-tap convolution kernel (csrc/conv_tc.cu) against the fp32 CUDA-core
kernel (csrc/conv_f32.cu) and against torch-CPU fp64.

Two kinds of checks:
  * operands that are exactly representable in TF32 (10 mantissa bits) -> products are exact, both kernels
    accumulate in fp32 -> agreement to ~1e-6 (catches every descriptor / swizzle / tap / phase bug);
  * generic fp32 operands -> agreement within TF32 rounding (rel 2e-3 of the output scale).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def ops():
    from lanedetection_end2end_b200 import ops_net
    return ops_net


def tf32_exact(t):
    """Zero the 13 low mantissa bits so the value is a TF32 number."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def prep(t, mode):
    """tf32 mode is checked with TF32-exact operands (exact products), tf32x3 with generic fp32 operands."""
    return tf32_exact(t) if mode == "tf32" else t


def wop(t, mode):
    """A packed weight operand as the mode's kernels take it (tf32x3: the TF32 hi / lo pair)."""
    return ops().split_tf32(t) if mode == "tf32x3" else t


TC_MODES = ["tf32", "tf32x3"]

CASES = [
    # N, C, H, W, vertical, dil
    (2, 64, 16, 128, True, 1),
    (2, 64, 16, 128, False, 1),
    (3, 128, 32, 64, True, 2),
    (3, 128, 32, 64, False, 4),
    (2, 128, 32, 64, True, 16),
    (2, 128, 32, 64, False, 16),
    (1, 128, 40, 80, True, 8),      # 320x640 geometry: 16x8 patch
    (1, 64, 80, 160, False, 1),
    (5, 64, 64, 128, True, 1),      # more tiles than one wave of a small grid
]


@pytest.fixture(params=[2, 1], ids=["slab", "per_tap"])
def variant(request):
    """Both implementations of lf_conv1d_tc: 2 = halo slab (default), 1 = one TMA box per tap."""
    from lanedetection_end2end_b200 import _capi
    _capi.lib().lf_conv1d_tc_set_variant(request.param)
    yield request.param
    _capi.lib().lf_conv1d_tc_set_variant(2)


@pytest.mark.parametrize("N,C,H,W,vertical,dil", CASES)
@pytest.mark.parametrize("exact", [True, False])
def test_tc_forward_matches_fp32_kernel(N, C, H, W, vertical, dil, exact, variant):
    o = ops()
    g = torch.Generator().manual_seed(N * 1000 + C + dil)
    x = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    if exact:
        x, w = tf32_exact(x), tf32_exact(w)
    assert o.tc_supported(x)
    o.set_conv_mode("fp32")
    ref = o.conv3(x, w, vertical, dil, False, bias=b, relu=False)
    o.set_conv_mode("tf32")
    try:
        got = o.conv3(x, w, vertical, dil, False, bias=b, relu=False)
        torch.cuda.synchronize()
    finally:
        o.set_conv_mode("fp32")
    scale = float(ref.abs().max())
    err = float((got - ref).abs().max()) / scale
    assert err <= (2e-6 if exact else 2e-3), err
    # independent check against torch-CPU fp64 on a slice
    xs, ws = x[:1].double().cpu().permute(0, 3, 1, 2), w.double().cpu()
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    cpu = F.conv2d(xs, ws, b.double().cpu(), 1, pad, dl).permute(0, 2, 3, 1)
    assert float((got[:1].double().cpu() - cpu).abs().max()) / scale <= (2e-6 if exact else 2e-3)


@pytest.mark.parametrize("C,H,W,dil", [(64, 16, 128, 1), (128, 32, 64, 8)])
def test_tc_epilogues_and_dgrad(C, H, W, dil, variant):
    o = ops()
    g = torch.Generator().manual_seed(7)
    N = 2
    x = tf32_exact(torch.randn(N, H, W, C, generator=g).cuda())
    w = tf32_exact((torch.randn(C, C, 1, 3, generator=g) / (3 * C) ** 0.5).cuda())
    b = torch.randn(C, generator=g).cuda()
    mask = torch.randn(N, H, W, C, generator=g).cuda()
    add = torch.randn(N, H, W, C, generator=g).cuda()
    addm = torch.randn(N, H, W, C, generator=g).cuda()
    outs = {}
    for mode in ("fp32", "tf32"):
        o.set_conv_mode(mode)
        try:
            outs[mode] = (o.conv3(x, w, False, dil, False, bias=b, relu=True),
                          o.conv3(x, w, False, dil, True, mask_src=mask),
                          o.conv3(x, w, False, dil, True, add_src=add, add_mask=addm))
            torch.cuda.synchronize()
        finally:
            o.set_conv_mode("fp32")
    for a, r in zip(outs["tf32"], outs["fp32"]):
        assert float((a - r).abs().max()) <= 2e-6 * float(r.abs().max())
    # fused column sums (bias gradient) of the masked input gradient
    o.set_conv_mode("tf32")
    try:
        cs = torch.empty(C, device="cuda")
        d = o.conv3(x, w, False, dil, True, colsum=cs, mask_src=mask)
        torch.cuda.synchronize()
    finally:
        o.set_conv_mode("fp32")
    want = d.double().sum(dim=(0, 1, 2))
    assert float((cs.double() - want).abs().max()) <= 1e-4 * float(want.abs().max())


def test_tc_block_level_tf32_tolerance():
    """non_bottleneck_1d fwd+bwd in tf32 mode vs fp32 mode: agreement within TF32 rounding."""
    from lanedetection_end2end_b200.Networks import ERFNet
    o = ops()
    torch.manual_seed(0)
    blk = ERFNet.non_bottleneck_1d(128, 0.0, 4).cuda().train()
    x = torch.randn(4, 128, 32, 64, device="cuda")
    gy = torch.randn(4, 128, 32, 64, device="cuda")
    res = {}
    for mode in ("fp32", "tf32"):
        o.set_conv_mode(mode)
        try:
            xi = x.clone().requires_grad_(True)
            blk.zero_grad()
            y = blk(xi)
            y.backward(gy)
            torch.cuda.synchronize()
            res[mode] = (y.detach().clone(), xi.grad.clone(), blk.conv3x1_2.weight.grad.clone())
        finally:
            o.set_conv_mode("fp32")
    # TF32 rounding can flip the sign of a near-zero pre-activation, which toggles a ReLU mask and changes
    # isolated gradient entries by O(1) (measured: rel. L2 3e-2, 5 % of the entries off by > 1 % of the max on
    # this random block): gate the L2 error and the FRACTION of large deviations, not the max norm.  The exact
    # checks of the kernels are the TF32-exact-operand tests above.
    for a, r in zip(res["tf32"], res["fp32"]):
        rel_l2 = float((a - r).norm() / r.norm())
        frac_bad = float(((a - r).abs() > 1e-2 * r.abs().max()).float().mean())
        assert rel_l2 <= 8e-2 and frac_bad <= 1e-1, (rel_l2, frac_bad)


@pytest.mark.parametrize("C,H,W,vertical,dil", [(64, 64, 128, False, 1), (128, 32, 64, False, 4), (128, 32, 64, True, 16)])
def test_tc_fused_bn_statistics(C, H, W, vertical, dil):
    """BatchNorm statistics accumulated in the conv epilogue == statistics of the stored output."""
    o = ops()
    g = torch.Generator().manual_seed(3)
    N = 4
    x = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    o.set_conv_mode("tf32")
    try:
        out, s = o.conv3_bn_stats(x, w, vertical, dil, b, gamma, beta, rm, rv, True)
        torch.cuda.synchronize()
    finally:
        o.set_conv_mode("fp32")
    mean = out.double().mean(dim=(0, 1, 2))
    var = out.double().var(dim=(0, 1, 2), unbiased=False)
    assert float((s.mean.double() - mean).abs().max()) <= 1e-5 * float(mean.abs().max() + 1)
    assert float((s.invstd.double() - (var + 1e-3).rsqrt()).abs().max()) <= 1e-5
    assert float((rm.double() - 0.1 * mean).abs().max()) <= 1e-5


@pytest.mark.parametrize("vertical", [True, False])
def test_c16_layers_on_tensor_cores_via_super_pixels(vertical):
    """C = 16 decoder blocks: [N,H,W,16] viewed as [N,H,W/4,64] with packed 64x64 weight blocks
    (ops_net.pack_tc_super).  TF32-exact operands -> agreement with the fp32 kernels to round-off."""
    o = ops()
    g = torch.Generator().manual_seed(11)
    N, C, H, W = 2, 16, 128, 256
    x = tf32_exact(torch.randn(N, H, W, C, generator=g).cuda())
    dy = tf32_exact(torch.randn(N, H, W, C, generator=g).cuda())
    kh, kw = (3, 1) if vertical else (1, 3)
    w = tf32_exact((torch.randn(C, C, kh, kw, generator=g) / 7).cuda())
    b = torch.randn(C, generator=g).cuda()
    mask = torch.randn(N, H, W, C, generator=g).cuda()
    res = {}
    for mode in ("fp32", "tf32"):
        o.set_conv_mode(mode)
        try:
            if mode == "tf32":
                assert o.super_ok(x, 1)
            cs = torch.empty(C, device="cuda")
            res[mode] = (o.conv3(x, w, vertical, 1, False, bias=b, relu=True),
                         o.conv3(dy, w, vertical, 1, True, colsum=cs, mask_src=mask), cs,
                         *o.wgrad3(x, dy, w, vertical, 1))
            torch.cuda.synchronize()
        finally:
            o.set_conv_mode("fp32")
    for i, (a, r) in enumerate(zip(res["tf32"], res["fp32"])):
        tol = 2e-6 if i < 2 else 1e-4
        assert float((a - r).abs().max()) <= tol * float(r.abs().max()), i


# ------------------------------------------------------------------------------------------------
# lf_conv_tcg: the resolution-changing layers (Down / Up blocks) on the tensor cores
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,O,tot,H,W,N", [(16, 48, 64, 128, 256, 2), (64, 64, 128, 64, 128, 3), (16, 48, 64, 32, 64, 1)])
@pytest.mark.parametrize("mode", TC_MODES)
def test_tcg_stride2_conv_and_its_input_gradient(C, O, tot, H, W, N, mode):
    """DownsamplerBlock conv (3x3, stride 2) into the concat buffer and its input gradient (tf32: TF32-exact operands,
    tf32x3: generic operands -> fp32-level agreement with torch fp64)."""
    o = ops()
    o.set_conv_mode(mode)
    try:
        g = torch.Generator().manual_seed(C + O)
        x = prep(torch.randn(N, H, W, C, generator=g).cuda(), mode)
        w = prep((torch.randn(O, C, 3, 3, generator=g) / (9 * C) ** 0.5).cuda(), mode)
        b = torch.randn(O, generator=g).cuda()
        assert o.tcg_s2conv_ok(x, C, O)
        cat = torch.full((N, H // 2, W // 2, tot), 7.0, device="cuda")
        o.run_tcg_s2conv(x, wop(o.pack_tcg_s2conv(w), mode), O, cat, bias=b)
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
        err = float((cat[..., :O].double() - ref).abs().max() / ref.abs().max())
        assert err < 3e-6, err
        assert bool((cat[..., O:] == 7.0).all())
        dcat = prep(torch.randn(N, H // 2, W // 2, tot, generator=g).cuda(), mode)
        assert o.tcg_s2convT_ok(dcat, O, C)
        kc = ((O + 31) // 32) * 32
        dx = torch.full((N, H, W, C), 3.0, device="cuda")
        o.run_tcg_s2convT(dcat, O, (wop(o.pack_tcg_s2convT(w, 0, kc), mode), wop(o.pack_tcg_s2convT(w, 1, kc), mode)), C, dx)
        ref = F.conv_transpose2d(dcat[..., :O].permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=1,
                                 output_padding=1).permute(0, 2, 3, 1)
        err = float((dx.double() - ref).abs().max() / ref.abs().max())
        assert err < 3e-6, err
    finally:
        o.set_conv_mode("fp32")


@pytest.mark.parametrize("I,O,H,W,N", [(128, 64, 32, 64, 2), (64, 16, 64, 128, 3), (64, 16, 16, 32, 1)])
@pytest.mark.parametrize("mode", TC_MODES)
def test_tcg_stride2_transposed_conv_and_its_input_gradient(I, O, H, W, N, mode):
    """UpsamplerBlock ConvTranspose2d (3x3, stride 2, padding 1, output_padding 1) and its input gradient."""
    o = ops()
    o.set_conv_mode(mode)
    try:
        g = torch.Generator().manual_seed(I + O)
        x = prep(torch.randn(N, H, W, I, generator=g).cuda(), mode)
        w = prep((torch.randn(I, O, 3, 3, generator=g) / (9 * I) ** 0.5).cuda(), mode)
        b = torch.randn(O, generator=g).cuda()
        assert o.tcg_s2convT_ok(x, I, O)
        u = torch.zeros(N, 2 * H, 2 * W, O, device="cuda")
        o.run_tcg_s2convT(x, I, (wop(o.pack_tcg_s2convT(w, 0, I), mode), wop(o.pack_tcg_s2convT(w, 1, I), mode)), O, u,
                          bias2=b.repeat(2))
        ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1,
                                 output_padding=1).permute(0, 2, 3, 1)
        err = float((u.double() - ref).abs().max() / ref.abs().max())
        assert err < 3e-6, err
        du = prep(torch.randn(N, 2 * H, 2 * W, O, generator=g).cuda(), mode)
        assert o.tcg_s2conv_ok(du, O, I)
        dx = torch.zeros(N, H, W, I, device="cuda")
        o.run_tcg_s2conv(du, wop(o.pack_tcg_s2conv(w), mode), I, dx)
        xin = x.permute(0, 3, 1, 2).double().requires_grad_(True)
        F.conv_transpose2d(xin, w.double(), stride=2, padding=1, output_padding=1).backward(du.permute(0, 3, 1, 2).double())
        ref = xin.grad.permute(0, 2, 3, 1)
        err = float((dx.double() - ref).abs().max() / ref.abs().max())
        assert err < 3e-6, err
    finally:
        o.set_conv_mode("fp32")


@pytest.mark.parametrize("C,H,W,dil", [(64, 32, 64, 1), (128, 32, 64, 2), (128, 32, 64, 8)])
@pytest.mark.parametrize("mode", TC_MODES)
def test_fused_batchnorm_backward_in_dgrad_epilogue(C, H, W, dil, mode):
    """dgrad_relu_bn_fused: the dgrad launch takes the BatchNorm INPUT x as mask operand, rebuilds the ReLU mask with the
    forward's fma(x, scale, shift) > 0 and accumulates sum g and sum g*x; the result must equal the two-pass route
    (dgrad masked with relu(bn(x)), then lf_bn_bwd_reduce over (g, x)) -- also for a negative and for a ZERO BatchNorm
    weight (round 1 divided by gamma there)."""
    o = ops()
    o.set_conv_mode(mode)
    g = torch.Generator().manual_seed(C + dil)
    N = 3
    x = torch.randn(N, H, W, C, generator=g).cuda() * 2 + 0.3            # pre-BN activations
    gamma = (torch.rand(C, generator=g) + 0.5).cuda()
    gamma[1] = -0.7
    gamma[3] = 0.0
    beta = (torch.randn(C, generator=g) * 0.3).cuda()
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    s = o.bn_forward_stats(x, gamma, beta, rm, rv, True)
    y = o.bn_apply(x, s, relu=True)
    d_out = prep(torch.randn(N, H, W, C, generator=g).cuda(), mode)
    w = prep((torch.randn(C, C, 3, 1, generator=g) / (3 * C) ** 0.5).cuda(), mode)
    fused = o.dgrad_relu_bn_fused(d_out, w, True, dil, x, s, gamma)
    assert fused is not None
    dx_f, dg_f, db_f = fused
    gref = o.conv3(d_out, w, True, dil, True, mask_src=y)
    dx_r, dg_r, db_r = o.bn_backward(gref, None, None, x, s, gamma)
    torch.cuda.synchronize()
    for a_, b_, name in ((dx_f, dx_r, "dx"), (dg_f, dg_r, "dgamma"), (db_f, db_r, "dbeta")):
        err = float((a_.double() - b_.double()).abs().max() / b_.double().abs().max())
        assert err < 2e-5, (name, err)


@pytest.mark.parametrize("kind,C,O,tot,H,W,N", [("conv", 16, 48, 64, 128, 256, 2), ("conv", 64, 64, 128, 64, 128, 3),
                                                ("convT", 64, 128, 0, 32, 64, 2), ("convT", 16, 64, 0, 64, 128, 2)])
@pytest.mark.parametrize("mode", TC_MODES)
def test_tcg_weight_gradients(kind, C, O, tot, H, W, N, mode):
    """lf_wgrad_tcg: weight gradients of the stride-2 Conv2d (A = input, B = output gradient) and of the stride-2
    ConvTranspose2d (A = output gradient, B = input) vs autograd in fp64 (TF32-exact operands)."""
    o = ops()
    o.set_conv_mode(mode)
    try:
        g = torch.Generator().manual_seed(C * 7 + O)
        if kind == "conv":
            x = prep(torch.randn(N, H, W, C, generator=g).cuda(), mode)
            dcat = prep(torch.randn(N, H // 2, W // 2, tot, generator=g).cuda(), mode)
            assert o.wgrad_tcg_ok(x, C, dcat, ((O + 31) // 32) * 32)
            dw = o.wgrad_tcg_conv(x, C, dcat, O)
            w = torch.zeros(O, C, 3, 3, dtype=torch.float64, device="cuda", requires_grad=True)
            F.conv2d(x.permute(0, 3, 1, 2).double(), w, stride=2, padding=1).backward(dcat[..., :O].permute(0, 3, 1, 2).double())
        else:
            # C = Cout_T (channels of the output gradient), O = Cin_T
            x = prep(torch.randn(N, H, W, O, generator=g).cuda(), mode)
            du = prep(torch.randn(N, 2 * H, 2 * W, C, generator=g).cuda(), mode)
            assert o.wgrad_tcg_ok(du, C, x, O)
            dw = o.wgrad_tcg_convT(x, O, du, C)
            w = torch.zeros(O, C, 3, 3, dtype=torch.float64, device="cuda", requires_grad=True)
            F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w, stride=2, padding=1, output_padding=1).backward(
                du.permute(0, 3, 1, 2).double())
        err = float((dw.double() - w.grad).abs().max() / w.grad.abs().max())
        assert err < 2e-5, err
    finally:
        o.set_conv_mode("fp32")


# ------------------------------------------------------------------------------------------------------
# 3xTF32 mode (csrc/conv_tc.cu): fp32-grade products on tensor cores -- GENERIC operands, fp32-level gates
# ------------------------------------------------------------------------------------------------------
X3_CASES = CASES + [
    (2, 128, 32, 64, True, 8),      # tall tile (32 x 4): halo 2d / TA
    (2, 128, 32, 64, False, 8),
    (1, 128, 40, 80, False, 16),    # 320x640 geometry, 48 KB slab: two pipeline stages
    (9, 128, 32, 64, True, 1),      # 9 tiles per CTA pair: several tiles per persistent CTA
    (1, 64, 128, 64, False, 1),     # the super-pixel view of a C=16 decoder layer
]


def _fp64_conv(x, w, b, vertical, dil, n=1):
    xs, ws = x[:n].double().cpu().permute(0, 3, 1, 2), w.double().cpu()
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    return F.conv2d(xs, ws, None if b is None else b.double().cpu(), 1, pad, dl).permute(0, 2, 3, 1)


@pytest.mark.parametrize("N,C,H,W,vertical,dil", X3_CASES)
def test_x3_forward_generic_operands_fp32_accuracy(N, C, H, W, vertical, dil):
    """lf_conv1d_tc_x3 on operands that are NOT TF32-exact: as close to fp64 as the fp32 FFMA kernel is."""
    o = ops()
    g = torch.Generator().manual_seed(N * 1000 + C + dil)
    x = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    o.set_conv_mode("tf32x3")
    assert o.tc_supported(x, vertical, dil)
    got = o.conv3(x, w, vertical, dil, False, bias=b, relu=False)
    o.set_conv_mode("fp32")
    ref = o.conv3(x, w, vertical, dil, False, bias=b, relu=False)
    torch.cuda.synchronize()
    cpu = _fp64_conv(x, w, b, vertical, dil, n=N)
    scale = float(cpu.abs().max())
    e_x3 = float((got.double().cpu() - cpu).abs().max()) / scale
    e_f32 = float((ref.double().cpu() - cpu).abs().max()) / scale
    print("x3 err %.2e  fp32-kernel err %.2e" % (e_x3, e_f32))
    assert e_x3 <= 2e-6, (e_x3, e_f32)
    assert e_x3 <= 2 * e_f32 + 5e-7, (e_x3, e_f32)


@pytest.mark.parametrize("C,H,W,dil,vertical", [(64, 16, 128, 1, False), (128, 32, 64, 8, False), (128, 32, 64, 16, False),
                                                (128, 32, 64, 16, True), (128, 32, 64, 8, True), (128, 40, 80, 8, True)])
def test_x3_epilogues_and_dgrad(C, H, W, dil, vertical):
    o = ops()
    g = torch.Generator().manual_seed(7)
    N = 3
    x = torch.randn(N, H, W, C, generator=g).cuda()
    w = (torch.randn(C, C, *((3, 1) if vertical else (1, 3)), generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    mask = torch.randn(N, H, W, C, generator=g).cuda()
    add = torch.randn(N, H, W, C, generator=g).cuda()
    addm = torch.randn(N, H, W, C, generator=g).cuda()
    outs = {}
    for mode in ("fp32", "tf32x3"):
        o.set_conv_mode(mode)
        cs = torch.empty(C, device="cuda")
        outs[mode] = (o.conv3(x, w, vertical, dil, False, bias=b, relu=True),
                      o.conv3(x, w, vertical, dil, True, mask_src=mask, colsum=cs),
                      o.conv3(x, w, vertical, dil, True, add_src=add, add_mask=addm), cs)
        torch.cuda.synchronize()
    for a, r in zip(outs["tf32x3"][:3], outs["fp32"][:3]):
        assert float((a - r).abs().max()) <= 3e-6 * float(r.abs().max())
    want = outs["tf32x3"][1].double().sum(dim=(0, 1, 2))
    assert float((outs["tf32x3"][3].double() - want).abs().max()) <= 1e-4 * float(want.abs().max())


def test_x3_block_level_matches_fp32_mode():
    """non_bottleneck_1d fwd+bwd (C=128, dilated, and the C=16 super-pixel form) in tf32x3 mode vs fp32 mode."""
    from lanedetection_end2end_b200.Networks import ERFNet
    o = ops()
    for C, dil, H, W in ((128, 4, 32, 64), (64, 1, 64, 128), (16, 1, 128, 256)):
        torch.manual_seed(0)
        blk = ERFNet.non_bottleneck_1d(C, 0.0, dil).cuda().train()
        x = torch.randn(2, C, H, W, device="cuda")
        gy = torch.randn(2, C, H, W, device="cuda")
        res = {}
        for mode in ("fp32", "tf32x3"):
            o.set_conv_mode(mode)
            xi = x.clone().requires_grad_(True)
            blk.zero_grad()
            y = blk(xi)
            y.backward(gy)
            torch.cuda.synchronize()
            res[mode] = [y.detach().clone(), xi.grad.clone()] + [p.grad.clone() for p in blk.parameters()]
        # The forward output is a continuous function of the arithmetic: max-norm gate.  Gradients are not: an fp32-level
        # difference in a pre-activation within ~1e-6 of zero flips one ReLU mask bit (expected: a handful per 1.5 M
        # mask entries), and each flip changes the ~1000 gradient entries downstream of that pixel by O(1) (measured:
        # 2 % of the entries).  A wrong tap / operand / descriptor would corrupt MOST entries: gate the median error at
        # fp32 round-off level and the share of entries beyond it.  The arithmetic of every kernel is gated entry by
        # entry in the operand-level tests above and below.
        assert float((res["tf32x3"][0] - res["fp32"][0]).abs().max()) <= 2e-5 * float(res["fp32"][0].abs().max())
        npix = 2 * H * W
        for a, r in zip(res["tf32x3"][1:], res["fp32"][1:]):
            sc = max(float(r.abs().max()), 1e-6)
            d = (a - r).abs().flatten()
            # the BatchNorm statistics couple EVERY entry behind them to a flip: one flipped bit moves the batch sums by one
            # entry out of `npix`, i.e. all those gradients by ~1/npix of their scale (measured 1.3e-4 at npix = 4096 with one
            # flip, session 7); allow three
            assert float(d.median()) <= (1e-5 + 3.0 / npix) * sc, (C, float(d.median()), sc)
            assert float((d > (1e-4 + 3.0 / npix) * sc).float().mean()) <= 0.05, (C, float((d > 1e-4 * sc).float().mean()))


@pytest.mark.parametrize("N,C,H,W,vertical,dil", [(2, 64, 16, 128, True, 1), (3, 64, 64, 128, False, 1), (3, 128, 32, 64, True, 2),
                                                  (2, 128, 32, 64, False, 16), (1, 128, 40, 80, True, 8), (32, 128, 32, 64, False, 4),
                                                  (3, 128, 32, 64, True, 16), (3, 128, 32, 64, True, 8)])
def test_x3_weight_gradient_generic_operands(N, C, H, W, vertical, dil):
    """lf_wgrad3_tc_x3 on generic fp32 operands vs torch fp64: as accurate as the fp32 split-K kernel."""
    o = ops()
    g = torch.Generator().manual_seed(5 + N + dil)
    x = torch.randn(N, H, W, C, generator=g).cuda()
    dy = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = torch.zeros(C, C, kh, kw, device="cuda")
    res = {}
    for mode in ("fp32", "tf32x3"):
        o.set_conv_mode(mode)
        res[mode] = o.wgrad3(x, dy, w, vertical, dil)[0]
        torch.cuda.synchronize()
    xs = x.double().cpu().permute(0, 3, 1, 2).requires_grad_(False)
    wd = torch.zeros(C, C, kh, kw, dtype=torch.float64, requires_grad=True)
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    F.conv2d(xs, wd, None, 1, pad, dl).backward(dy.double().cpu().permute(0, 3, 1, 2))
    scale = float(wd.grad.abs().max())
    e_x3 = float((res["tf32x3"].double().cpu() - wd.grad).abs().max()) / scale
    e_f32 = float((res["fp32"].double().cpu() - wd.grad).abs().max()) / scale
    print("wgrad x3 err %.2e  fp32-kernel err %.2e" % (e_x3, e_f32))
    # the sum runs over up to 65 536 pixels; the tensor-core accumulator adds 8 products per instruction in fp32 (measured
    # 3.8e-6 at N=32, the split-K FFMA kernel's hierarchical sum 5.7e-7) -- an fp32 dot product of that length
    assert e_x3 <= 1e-5, (e_x3, e_f32)


@pytest.mark.parametrize("vertical", [True, False])
def test_x3_c16_super_pixel_layers(vertical):
    """C = 16 decoder blocks through the 3xTF32 kernels (super-pixel view), generic operands."""
    o = ops()
    g = torch.Generator().manual_seed(11)
    N, C, H, W = 2, 16, 128, 256
    x = torch.randn(N, H, W, C, generator=g).cuda()
    dy = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / 7).cuda()
    b = torch.randn(C, generator=g).cuda()
    mask = torch.randn(N, H, W, C, generator=g).cuda()
    res = {}
    for mode in ("fp32", "tf32x3"):
        o.set_conv_mode(mode)
        if mode == "tf32x3":
            assert o.super_ok(x, 1)
        cs = torch.empty(C, device="cuda")
        res[mode] = (o.conv3(x, w, vertical, 1, False, bias=b, relu=True),
                     o.conv3(dy, w, vertical, 1, True, colsum=cs, mask_src=mask), cs,
                     *o.wgrad3(x, dy, w, vertical, 1))
        torch.cuda.synchronize()
    for i, (a, r) in enumerate(zip(res["tf32x3"], res["fp32"])):
        tol = 3e-6 if i < 2 else 1e-4
        assert float((a - r).abs().max()) <= tol * float(r.abs().max()), i


def test_premasked_residual_gradient_is_bit_identical():
    """lf_bn_bwd_apply_gated + single-operand residual add (ops_net.PREMASK_RESIDUAL) against the two-operand epilogue
    (add_src = dy, add_mask = y): the same values are added, so every gradient of the block must be bit-identical."""
    from lanedetection_end2end_b200.Networks import ERFNet
    o = ops()
    o.set_conv_mode("tf32x3")
    for C, dil, H, W in ((64, 1, 64, 128), (128, 2, 32, 64)):
        torch.manual_seed(1)
        blk = ERFNet.non_bottleneck_1d(C, 0.3, dil).cuda().train()
        blk.drop_mask_override = (torch.rand(2, C) >= 0.3).float() / 0.7
        x = torch.randn(2, C, H, W, device="cuda")
        gy = torch.randn(2, C, H, W, device="cuda")
        res = {}
        try:
            for pre in (False, True):
                o.PREMASK_RESIDUAL = pre
                xi = x.clone().requires_grad_(True)
                blk.zero_grad()
                blk(xi).backward(gy)
                torch.cuda.synchronize()
                res[pre] = [xi.grad.clone()] + [p.grad.clone() for p in blk.parameters()]
        finally:
            o.PREMASK_RESIDUAL = True
        for a, b in zip(res[True], res[False]):
            assert torch.equal(a, b)
