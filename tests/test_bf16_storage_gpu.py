"""bf16 storage of the non_bottleneck_1d ReLU outputs in bf16 mode (ops_net.nb1d_storage_dtype): t1 = relu(conv3x1_1),
t3 = relu(bn1), t4 = relu(conv3x1_2) are only convolution inputs and ReLU masks, and every kernel that reads them in bf16
mode rounds them to bf16 (nearest even) first.  Storing them rounded therefore changes no result, and every comparison
here is torch.equal, not a tolerance.

The one exception: a positive fp32 ReLU output at most half of bf16's smallest subnormal (2^-134, ~4.6e-41) rounds to
zero in storage and flips its ReLU mask bit.  The block tests assert that no such value occurs in their inputs.
"""
import pytest
import torch

from oracle import inputs

pytestmark = pytest.mark.gpu

TINY = 2.0 ** -134
SAVED_PER_IMAGE = 40_894_464   # config 2: (7 C=64 + 2 C=16 blocks) x 3 MiB + 8 C=128 blocks x 1.5 MiB


def ops():
    from lanedetection_end2end_b200 import ops_net
    return ops_net


@pytest.fixture
def bf16():
    o = ops()
    prev = o.CONV_MODE
    o.set_conv_mode("bf16")
    yield o
    torch.cuda.synchronize()
    o.set_conv_mode(prev)
    o.ACTIVE_PACKS = None


@pytest.fixture(params=[2, 1], ids=["slab", "per_tap"])
def variant(request):
    from lanedetection_end2end_b200 import _capi
    _capi.lib().lf_conv1d_tc_set_variant(request.param)
    yield request.param
    _capi.lib().lf_conv1d_tc_set_variant(2)


def bx(t):
    return t.bfloat16().float()


def no_tiny(*ts):
    for t in ts:
        t = t.float()
        assert not bool(((t > 0) & (t <= TINY)).any())


def _case(C, H, W, vertical, seed, N=2):
    g = torch.Generator().manual_seed(seed)
    kh, kw = (3, 1) if vertical else (1, 3)
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    extra = [torch.randn(N, H, W, C, generator=g).cuda() for _ in range(2)]
    return x, w, b, extra


DILS = [1, 2, 4, 8, 16]


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("vertical", [True, False])
@pytest.mark.parametrize("dil", DILS)
def test_bf16_input_forward_equals_fp32_input(bf16, variant, C, vertical, dil):
    """lf_conv1d_tc_bf16 on a bf16 activation == on its fp32 copy, for every epilogue."""
    o = bf16
    x, w, b, (mask, add) = _case(C, 32, 64, vertical, 10 * C + dil + vertical)
    N, H, W, _ = x.shape
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")

    def run(xin):
        cs = torch.empty(C, device="cuda")
        rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
        out, s = o.conv3_bn_stats(xin, w, vertical, dil, b, gamma, beta, rm, rv, True)
        return (o.conv3(xin, w, vertical, dil, False, bias=b, relu=True),
                o.conv3(xin, w, vertical, dil, False, bias=b, relu=2, add_src=add),
                o.conv3(xin, w, vertical, dil, True, mask_src=mask, colsum=cs), cs,
                out, s.mean, s.invstd, s.scale, s.shift, rm, rv)
    assert o.tc_supported(x, vertical, dil)
    ref, got = run(x), run(x.bfloat16())
    for i, (a, r) in enumerate(zip(got, ref)):
        assert a.dtype == torch.float32 and torch.equal(a, r), i


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("vertical", [True, False])
@pytest.mark.parametrize("dil", [1, 16])
def test_bf16_output_and_bf16_mask(bf16, variant, C, vertical, dil):
    """A bf16 `out` is the fp32 `out` rounded (.to(torch.bfloat16)); a bf16 `mask_src` gates like its fp32 copy."""
    o = bf16
    x, w, b, (dy, m) = _case(C, 32, 64, vertical, 3 * C + dil)
    m16 = m.bfloat16()
    for xin in (x, x.bfloat16()):
        ref = o.conv3(xin, w, vertical, dil, False, bias=b, relu=True)
        got = o.conv3(xin, w, vertical, dil, False, bias=b, relu=True, dtype=torch.bfloat16)
        assert got.dtype == torch.bfloat16 and torch.equal(got, ref.to(torch.bfloat16))
    cs16, cs32 = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
    got = o.conv3(dy, w, vertical, dil, True, mask_src=m16, colsum=cs16)
    ref = o.conv3(dy, w, vertical, dil, True, mask_src=m16.float(), colsum=cs32)
    assert torch.equal(got, ref) and torch.equal(cs16, cs32)


@pytest.mark.parametrize("vertical", [True, False])
def test_bf16_storage_c16_super_pixel_layers(bf16, vertical):
    o = bf16
    x, w, b, (dy, m) = _case(16, 128, 256, vertical, 16 + vertical)
    w = bx(w * 4)
    assert o.super_ok(x, 1)
    m16 = m.bfloat16()
    for xin in (x, x.bfloat16()):
        ref = o.conv3(xin, w, vertical, 1, False, bias=b, relu=True)
        assert torch.equal(o.conv3(x.bfloat16(), w, vertical, 1, False, bias=b, relu=True), ref)
        got = o.conv3(xin, w, vertical, 1, False, bias=b, relu=True, dtype=torch.bfloat16)
        assert torch.equal(got, ref.to(torch.bfloat16))
    cs16, cs32 = torch.empty(16, device="cuda"), torch.empty(16, device="cuda")
    assert torch.equal(o.conv3(dy, w, vertical, 1, True, mask_src=m16, colsum=cs16),
                       o.conv3(dy, w, vertical, 1, True, mask_src=m16.float(), colsum=cs32))
    assert torch.equal(cs16, cs32)
    dw16, db16 = o.wgrad3(x.bfloat16(), dy, w, vertical, 1)
    dw32, db32 = o.wgrad3(x, dy, w, vertical, 1)
    assert torch.equal(dw16, dw32) and torch.equal(db16, db32)


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("vertical", [True, False])
@pytest.mark.parametrize("dil", DILS)
def test_bf16a_weight_gradient_equals_fp32_a(bf16, C, vertical, dil):
    """The 3-tap weight gradient with a bf16 A view (bf16 layer input, fp32 output gradient; traced as lf_wgrad3_tc_bf16a) ==
    the one on the fp32 copy."""
    from lanedetection_end2end_b200 import _capi
    o = bf16
    x, w, _, (dy, _) = _case(C, 32, 64, vertical, 7 * C + dil + vertical)
    _capi.TRACE = []
    try:
        dw16, db16 = o.wgrad3(x.bfloat16(), dy, w, vertical, dil)
        names = [t[0] for t in _capi.TRACE]
    finally:
        _capi.TRACE = None
    assert "lf_wgrad3_tc_bf16a" in names
    dw32, db32 = o.wgrad3(x, dy, w, vertical, dil)
    assert torch.equal(dw16, dw32) and torch.equal(db16, db32)


@pytest.mark.parametrize("C", [16, 64, 128])
def test_bn_apply_bf16_output(bf16, C):
    o = bf16
    g = torch.Generator().manual_seed(C)
    N, H, W = 3, 16, 32
    x = torch.randn(N, H, W, C, generator=g).cuda()
    res = torch.randn(N, H, W, C, generator=g).cuda()
    drop = (torch.rand(N, C, generator=g) > 0.3).float().cuda() / 0.7
    s = o.bn_forward_stats(x, torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda"),
                           torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), True)
    for kw in (dict(relu=True), dict(relu=True, drop=drop, res=res), dict(relu=False)):
        got = o.bn_apply(x, s, dtype=torch.bfloat16, **kw)
        assert got.dtype == torch.bfloat16 and torch.equal(got, o.bn_apply(x, s, **kw).to(torch.bfloat16))


# ---------------------------------------------------------------------------------------------------------------------
# the block, against the same primitives with fp32 intermediates
# ---------------------------------------------------------------------------------------------------------------------
def _reference_block(o, x, m, drop, dy):
    """non_bottleneck_1d forward + backward composed from ops_net primitives with fp32 t1, t3, t4."""
    dil = m.dilated
    P = lambda t: t.detach()
    w1, b1, w2, b2 = P(m.conv3x1_1.weight), P(m.conv3x1_1.bias), P(m.conv1x3_1.weight), P(m.conv1x3_1.bias)
    w3, b3, w4, b4 = P(m.conv3x1_2.weight), P(m.conv3x1_2.bias), P(m.conv1x3_2.weight), P(m.conv1x3_2.bias)
    g1, be1, g2, be2 = P(m.bn1.weight), P(m.bn1.bias), P(m.bn2.weight), P(m.bn2.bias)
    rm1, rv1, rm2, rv2 = (t.clone() for t in (m.bn1.running_mean, m.bn1.running_var, m.bn2.running_mean, m.bn2.running_var))
    t1 = o.conv3(x, w1, True, 1, False, bias=b1, relu=True)
    t2, s1 = o.conv3_bn_stats(t1, w2, False, 1, b2, g1, be1, rm1, rv1, True)
    t3 = o.bn_apply(t2, s1, relu=True)
    t4 = o.conv3(t3, w3, True, dil, False, bias=b3, relu=True)
    t5, s2 = o.conv3_bn_stats(t4, w4, False, dil, b4, g2, be2, rm2, rv2, True)
    y = o.bn_apply(t5, s2, relu=True, drop=drop, res=x)
    no_tiny(t1, t3, t4)
    C = x.shape[-1]
    o._DEFERRED = jobs = []
    try:
        d5, dg2, dbe2, gm = o.bn_backward(dy, y, drop, t5, s2, g2, want_gated=True)
        db1, db3 = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        dw4, _ = o.wgrad3(t4, d5, w4, False, dil, bias_grad="skip")
        d4 = o.conv3(d5, w4, False, dil, True, colsum=db3, mask_src=t4)
        dw3, _ = o.wgrad3(t3, d4, w3, True, dil, bias_grad="skip")
        fused = o.dgrad_relu_bn_fused(d4, w3, True, dil, t2, s1, g1)
        if fused is not None:
            d2, dg1, dbe1 = fused
        else:
            d3 = o.conv3(d4, w3, True, dil, True, mask_src=t3)
            d2, dg1, dbe1 = o.bn_backward(d3, None, None, t2, s1, g1)
        dw2, _ = o.wgrad3(t1, d2, w2, False, 1, bias_grad="skip")
        d1 = o.conv3(d2, w2, False, 1, True, colsum=db1, mask_src=t1)
        dw1, _ = o.wgrad3(x, d1, w1, True, 1, bias_grad="skip")
        dx = o.conv3(d1, w1, True, 1, True, add_src=gm)
        if jobs:
            o.flush_deferred_reductions(jobs)
    finally:
        o._DEFERRED = None
    zero = torch.zeros(C, device="cuda")
    return dict(y=y, dx=dx, w1=dw1, b1=db1, w2=dw2, b2=zero, w3=dw3, b3=db3, w4=dw4, b4=zero, g1=dg1, be1=dbe1, g2=dg2,
                be2=dbe2, rm1=rm1, rv1=rv1, rm2=rm2, rv2=rv2)


def _block(C, dil, H, W, N=2, seed=0):
    from lanedetection_end2end_b200.Networks.ERFNet import non_bottleneck_1d
    torch.manual_seed(seed)
    m = non_bottleneck_1d(C, 0.3, dil).cuda().train()
    with torch.no_grad():
        for bn in (m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.normal_(0, 0.3)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, H, W, C, generator=g).cuda()
    dy = torch.randn(N, H, W, C, generator=g).cuda()
    m.drop_mask_override = ((torch.rand(N, C, generator=g) > 0.3).float() / 0.7).cuda()
    return m, x, dy


def _run_module(m, x, dy):
    xl = x.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    y = m(xl.permute(0, 3, 1, 2))
    y.backward(dy.permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    P = lambda p: p.grad
    return dict(y=y.permute(0, 2, 3, 1), dx=xl.grad, w1=P(m.conv3x1_1.weight), b1=P(m.conv3x1_1.bias),
                w2=P(m.conv1x3_1.weight), b2=P(m.conv1x3_1.bias), w3=P(m.conv3x1_2.weight), b3=P(m.conv3x1_2.bias),
                w4=P(m.conv1x3_2.weight), b4=P(m.conv1x3_2.bias), g1=P(m.bn1.weight), be1=P(m.bn1.bias),
                g2=P(m.bn2.weight), be2=P(m.bn2.bias), rm1=m.bn1.running_mean, rv1=m.bn1.running_var,
                rm2=m.bn2.running_mean, rv2=m.bn2.running_var)


@pytest.mark.parametrize("C,dil,H,W", [(64, 1, 64, 128), (64, 16, 64, 128), (128, 1, 32, 64), (128, 16, 32, 64),
                                       (16, 1, 128, 256)])
def test_block_bf16_storage_matches_fp32_intermediates(bf16, C, dil, H, W):
    o = bf16
    from lanedetection_end2end_b200 import _capi
    m, x, dy = _block(C, dil, H, W, seed=C + dil)
    assert o.nb1d_storage_dtype(x, dil) == torch.bfloat16
    ref = _reference_block(o, x, m, m.drop_mask_override, dy)
    _capi.TRACE = []
    try:
        got = _run_module(m, x, dy)
        names = [t[0] for t in _capi.TRACE]
    finally:
        _capi.TRACE = None
    assert "lf_bn_apply_bf16" in names and "lf_wgrad3_tc_bf16a" in names
    for k in ref:
        assert got[k] is not None and torch.equal(got[k], ref[k]), k


def test_fallback_shape_keeps_fp32_storage(bf16):
    """A block the tensor-core kernels do not take (no 128-pixel patch divides 12 x 12) runs on the FFMA kernels and keeps
    fp32 storage."""
    o = bf16
    m, x, dy = _block(64, 1, 12, 12)
    assert not o.tc_supported(x, True, 1)
    assert o.nb1d_storage_dtype(x, 1) == torch.float32
    got = _run_module(m, x, dy)
    assert all(bool(torch.isfinite(v).all()) for v in got.values())


# ---------------------------------------------------------------------------------------------------------------------
# the whole model
# ---------------------------------------------------------------------------------------------------------------------
def _config2(B):
    from oracle import golden_check
    model, args = golden_check.build_net(2, 2, 0.3, B)
    torch.manual_seed(3)
    model = model.cuda().train()
    for mod in model.modules():
        if hasattr(mod, "dropout"):
            mod.dropout.p = 0
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.momentum = 0.0
    return model, args


def _force_fp32(monkeypatch):
    monkeypatch.setattr(ops(), "nb1d_storage_dtype", lambda x, dil: torch.float32)


def test_model_step_bit_identical_to_fp32_storage(bf16, monkeypatch):
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep, GraphedInference
    B, L = 4, 2
    model, args = _config2(B)
    model.defer_status_check = True
    crit = backprojection_loss(args)
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=21)).cuda()
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=22)
    xgt, valid = torch.from_numpy(xgt_np).cuda(), torch.from_numpy(valid_np).cuda()
    # every training step moves the BatchNorm running statistics (the blocks update them with momentum 0.1): both rounds
    # start from the same state
    state = {k: v.clone() for k, v in model.state_dict().items()}

    def run_all():
        model.load_state_dict(state)
        return eager(), graphed(), infer()

    def eager():
        model.zero_grad(set_to_none=True)
        out = model(x, torch.zeros(B, 4), True)
        loss = sum(crit(out[l], xgt[:, l], valid[:, l])[0] for l in range(L)) / L
        loss.backward()
        torch.cuda.synchronize()
        return loss.detach().clone(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    def graphed():
        step = GraphedTrainStep(model, crit, L, x, xgt, valid, None)
        loss = step().clone()
        torch.cuda.synchronize()
        return loss, {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    def infer():
        model.eval()
        gi = GraphedInference(model, x)
        out = [t.clone() for t in gi.infer(x)[:L]]
        torch.cuda.synchronize()
        model.train()
        return out

    res16 = run_all()
    with monkeypatch.context() as mp:
        _force_fp32(mp)
        res32 = run_all()
    for (l16, g16), (l32, g32) in zip(res16[:2], res32[:2]):
        assert torch.equal(l16, l32)
        assert g16.keys() == g32.keys()
        for n in g32:
            assert torch.equal(g16[n], g32[n]), n
    for a, b in zip(res16[2], res32[2]):
        assert torch.equal(a, b)


def test_forward_memory_drops_by_the_bf16_tensors(bf16, monkeypatch):
    B = 8
    model, _ = _config2(B)
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=5)).cuda()

    def forward_bytes():
        model.zero_grad(set_to_none=True)
        out = model(x, torch.zeros(B, 4), True)
        sum((b ** 2).sum() for b in out[:2]).backward()      # packs and gradients exist before the measurement
        del out
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        out = model(x, torch.zeros(B, 4), True)
        torch.cuda.synchronize()
        used = torch.cuda.memory_allocated() - before
        del out
        return used

    used16 = forward_bytes()
    with monkeypatch.context() as mp:
        _force_fp32(mp)
        used32 = forward_bytes()
    print("forward bytes: fp32 storage %d, bf16 storage %d, saved %d" % (used32, used16, used32 - used16))
    assert used32 - used16 >= 0.99 * B * SAVED_PER_IMAGE
