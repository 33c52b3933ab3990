"""GPU tests of the bf16 convolution mode (ops_net.set_conv_mode("bf16")): the BF16 wgmma paths of conv_tc.cu (3-tap
convolutions, input gradients, C = 16 super-pixel layers), conv_tcg.cu (stride-2 conv / transposed conv, the heads' dense
3x3) and wgrad_tcg.cu (every tensor-core weight gradient), the bf16 weight packing and the whole training step.

  * Exact operands: inputs pre-rounded with t.bfloat16().float(), so every product is exact in fp32 and only the fp32
    summation differs from the fp32 kernels and from torch-CPU fp64.  Gates as tight as the TF32-exact cases of
    test_conv_tc_gpu.py; these catch any fragment, swizzle, descriptor or tap bug.
  * Generic operands: the tolerance is the bf16 rounding scale (see GENERIC_GATE).
  * Full path on the golden inputs: beta and loss error vs fp64, measured on the H100 and committed as
    tests/golden/bf16_accuracy_<case>.json.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import inputs
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

# One bf16 rounding of each operand (relative 2^-9) per product, summed over K = 3C products: the error of a generic-operand
# result is a few times 2^-9 of its scale.  Tolerance = 4 x 2^-9 (the measured errors are printed, run with -s).
GENERIC_GATE = 4 * 2.0 ** -9


def ops():
    from lanedetection_end2end_b200 import ops_net
    return ops_net


def bx(t):
    """Round to bf16 and back: products of such values are exact in fp32."""
    return t.bfloat16().float()


@pytest.fixture(params=[2, 1], ids=["slab", "per_tap"])
def variant(request):
    from lanedetection_end2end_b200 import _capi
    _capi.lib().lf_conv1d_tc_set_variant(request.param)
    yield request.param
    _capi.lib().lf_conv1d_tc_set_variant(2)


def in_mode(mode, fn):
    o = ops()
    prev = o.CONV_MODE
    o.set_conv_mode(mode)
    try:
        r = fn()
        torch.cuda.synchronize()
        return r
    finally:
        o.set_conv_mode(prev)


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


CASES = [
    # N, C, H, W, vertical, dil  (the cases of test_conv_tc_gpu.py)
    (2, 64, 16, 128, True, 1),
    (2, 64, 16, 128, False, 1),
    (3, 128, 32, 64, True, 2),
    (3, 128, 32, 64, False, 4),
    (2, 128, 32, 64, True, 16),
    (2, 128, 32, 64, False, 16),
    (1, 128, 40, 80, True, 8),
    (1, 64, 80, 160, False, 1),
    (5, 64, 64, 128, True, 1),
]


def _fp64_conv(x, w, b, vertical, dil):
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    return F.conv2d(x.double().cpu().permute(0, 3, 1, 2), w.double().cpu(), None if b is None else b.double().cpu(), 1, pad,
                    dl).permute(0, 2, 3, 1)


@pytest.mark.parametrize("N,C,H,W,vertical,dil", CASES)
def test_bf16_forward_exact_operands(N, C, H, W, vertical, dil, variant):
    o = ops()
    g = torch.Generator().manual_seed(N * 1000 + C + dil)
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = bx(torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    ref = in_mode("fp32", lambda: o.conv3(x, w, vertical, dil, False, bias=b))
    got = in_mode("bf16", lambda: (o.tc_supported(x, vertical, dil), o.conv3(x, w, vertical, dil, False, bias=b)))
    assert got[0]
    got = got[1]
    scale = float(ref.abs().max())
    assert float((got - ref).abs().max()) / scale <= 2e-6
    cpu = _fp64_conv(x[:1], w, b, vertical, dil)
    assert float((got[:1].double().cpu() - cpu).abs().max()) / scale <= 2e-6


@pytest.mark.parametrize("C,H,W,dil", [(64, 16, 128, 1), (128, 32, 64, 8)])
def test_bf16_epilogues_and_input_gradient(C, H, W, dil, variant):
    """bias + ReLU, mask, add + add_mask, column sums: the same epilogue as TF32, on exact bf16 products."""
    o = ops()
    g = torch.Generator().manual_seed(7)
    N = 2
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    w = bx(torch.randn(C, C, 1, 3, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    mask, add, addm = (torch.randn(N, H, W, C, generator=g).cuda() for _ in range(3))

    def run():
        cs = torch.empty(C, device="cuda")
        return (o.conv3(x, w, False, dil, False, bias=b, relu=True), o.conv3(x, w, False, dil, True, mask_src=mask),
                o.conv3(x, w, False, dil, True, add_src=add, add_mask=addm), o.conv3(x, w, False, dil, True, colsum=cs, mask_src=mask), cs)
    ref, got = in_mode("fp32", run), in_mode("bf16", run)
    for a, r in zip(got[:4], ref[:4]):
        assert float((a - r).abs().max()) <= 2e-6 * float(r.abs().max())
    want = got[3].double().sum(dim=(0, 1, 2))
    assert float((got[4].double() - want).abs().max()) <= 1e-4 * float(want.abs().max())
    # the input gradient against fp64 autograd
    dy = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    dx = in_mode("bf16", lambda: o.conv3(dy, w, False, dil, True))
    xin = torch.zeros(N, C, H, W, dtype=torch.float64, requires_grad=True)
    F.conv2d(xin, w.double().cpu(), None, 1, (0, dil), (1, dil)).backward(dy.double().cpu().permute(0, 3, 1, 2))
    ref = xin.grad.permute(0, 2, 3, 1)
    assert float((dx.double().cpu() - ref).abs().max()) <= 2e-6 * float(ref.abs().max())


@pytest.mark.parametrize("C,H,W,vertical,dil", [(64, 64, 128, False, 1), (128, 32, 64, False, 4), (128, 32, 64, True, 16)])
def test_bf16_fused_bn_statistics(C, H, W, vertical, dil):
    o = ops()
    g = torch.Generator().manual_seed(3)
    N = 4
    x = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    out, s = in_mode("bf16", lambda: o.conv3_bn_stats(x, w, vertical, dil, b, gamma, beta, rm, rv, True))
    mean = out.double().mean(dim=(0, 1, 2))
    var = out.double().var(dim=(0, 1, 2), unbiased=False)
    assert float((s.mean.double() - mean).abs().max()) <= 1e-5 * float(mean.abs().max() + 1)
    assert float((s.invstd.double() - (var + 1e-3).rsqrt()).abs().max()) <= 1e-5


@pytest.mark.parametrize("C,H,W,dil", [(64, 32, 64, 1), (128, 32, 64, 2), (128, 32, 64, 8)])
def test_bf16_affine_mask_bn_backward_statistics(C, H, W, dil):
    """The input-gradient launch that rebuilds the ReLU mask from the BatchNorm input and accumulates BN backward's sums."""
    o = ops()
    g = torch.Generator().manual_seed(C + dil)
    N = 3
    x = torch.randn(N, H, W, C, generator=g).cuda() * 2 + 0.3
    gamma = (torch.rand(C, generator=g) + 0.5).cuda()
    gamma[1] = -0.7
    gamma[3] = 0.0
    beta = (torch.randn(C, generator=g) * 0.3).cuda()
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    d_out = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    w = bx(torch.randn(C, C, 3, 1, generator=g) / (3 * C) ** 0.5).cuda()

    def run():
        s = o.bn_forward_stats(x, gamma, beta, rm, rv, True)
        y = o.bn_apply(x, s, relu=True)
        fused = o.dgrad_relu_bn_fused(d_out, w, True, dil, x, s, gamma)
        assert fused is not None
        gref = o.conv3(d_out, w, True, dil, True, mask_src=y)
        return fused, o.bn_backward(gref, None, None, x, s, gamma)
    fused, two_pass = in_mode("bf16", run)
    for a_, b_ in zip(fused, two_pass):
        assert rel(a_, b_) < 2e-5


@pytest.mark.parametrize("vertical", [True, False])
def test_bf16_c16_super_pixel_layers(vertical):
    o = ops()
    g = torch.Generator().manual_seed(11)
    N, C, H, W = 2, 16, 128, 256
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    dy = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = bx(torch.randn(C, C, kh, kw, generator=g) / 7).cuda()
    b = torch.randn(C, generator=g).cuda()
    mask = torch.randn(N, H, W, C, generator=g).cuda()

    def run():
        cs = torch.empty(C, device="cuda")
        return (o.conv3(x, w, vertical, 1, False, bias=b, relu=True), o.conv3(dy, w, vertical, 1, True, colsum=cs, mask_src=mask), cs,
                *o.wgrad3(x, dy, w, vertical, 1))
    assert in_mode("bf16", lambda: o.super_ok(x, 1))
    ref, got = in_mode("fp32", run), in_mode("bf16", run)
    for i, (a, r) in enumerate(zip(got, ref)):
        tol = 2e-6 if i < 2 else 2e-5
        assert float((a - r).abs().max()) <= tol * float(r.abs().max()), i


def _wop(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("C,O,tot,H,W,N", [(16, 48, 64, 128, 256, 2), (64, 64, 128, 64, 128, 3), (16, 48, 64, 32, 64, 1)])
def test_bf16_tcg_stride2_conv_and_input_gradient(C, O, tot, H, W, N):
    o = ops()
    g = torch.Generator().manual_seed(C + O)
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    w = bx(torch.randn(O, C, 3, 3, generator=g) / (9 * C) ** 0.5).cuda()
    b = torch.randn(O, generator=g).cuda()
    dcat = bx(torch.randn(N, H // 2, W // 2, tot, generator=g)).cuda()
    kc = ((O + 31) // 32) * 32

    def run():
        assert o.tcg_s2conv_ok(x, C, O) and o.tcg_s2convT_ok(dcat, O, C)
        cat = torch.full((N, H // 2, W // 2, tot), 7.0, device="cuda")
        o.run_tcg_s2conv(x, _wop(o.pack_tcg_s2conv(w)), O, cat, bias=b)
        dx = torch.full((N, H, W, C), 3.0, device="cuda")
        o.run_tcg_s2convT(dcat, O, (_wop(o.pack_tcg_s2convT(w, 0, kc)), _wop(o.pack_tcg_s2convT(w, 1, kc))), C, dx)
        return cat, dx
    cat, dx = in_mode("bf16", run)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    assert rel(cat[..., :O], ref) < 3e-6
    assert bool((cat[..., O:] == 7.0).all())
    ref = F.conv_transpose2d(dcat[..., :O].permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=1,
                             output_padding=1).permute(0, 2, 3, 1)
    assert rel(dx, ref) < 3e-6


@pytest.mark.parametrize("I,O,H,W,N", [(128, 64, 32, 64, 2), (64, 16, 64, 128, 3), (64, 16, 16, 32, 1)])
def test_bf16_tcg_stride2_transposed_conv(I, O, H, W, N):
    o = ops()
    g = torch.Generator().manual_seed(I + O)
    x = bx(torch.randn(N, H, W, I, generator=g)).cuda()
    w = bx(torch.randn(I, O, 3, 3, generator=g) / (9 * I) ** 0.5).cuda()
    b = torch.randn(O, generator=g).cuda()

    def run():
        assert o.tcg_s2convT_ok(x, I, O)
        u = torch.zeros(N, 2 * H, 2 * W, O, device="cuda")
        o.run_tcg_s2convT(x, I, (_wop(o.pack_tcg_s2convT(w, 0, I)), _wop(o.pack_tcg_s2convT(w, 1, I))), O, u, bias2=b.repeat(2))
        return u
    u = in_mode("bf16", run)
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1,
                             output_padding=1).permute(0, 2, 3, 1)
    assert rel(u, ref) < 3e-6


@pytest.mark.parametrize("Ci,Co,k", [(128, 128, 1), (128, 64, 3), (64, 64, 3)])
def test_bf16_heads_dense_convolutions(Ci, Co, k):
    """The Classification heads' dense convolutions (lf_conv_tcg with 1 or 9 taps) and their gradients."""
    from lanedetection_end2end_b200 import ops_heads as hd
    g = torch.Generator().manual_seed(Ci + Co + k)
    N, H, W = 2, 8, 32
    x = bx(torch.randn(N, H, W, Ci, generator=g)).cuda()
    w = bx(torch.randn(Co, Ci, k, k, generator=g) * 0.1).cuda()
    b = torch.randn(Co, generator=g).cuda()
    dy = bx(torch.randn(N, H, W, Co, generator=g)).cuda()
    y, dx, dw = in_mode("bf16", lambda: (hd.conv_fwd(x, w, b), hd.conv_dgrad(dy, w), hd.conv_wgrad(x, dy, w)))
    xin = x.permute(0, 3, 1, 2).double().cpu().requires_grad_(True)
    wd = w.double().cpu().requires_grad_(True)
    ref = F.conv2d(xin, wd, b.double().cpu(), padding=(k - 1) // 2)
    ref.backward(dy.permute(0, 3, 1, 2).double().cpu())
    assert rel(y.cpu(), ref.detach().permute(0, 2, 3, 1)) < 3e-6
    assert rel(dx.cpu(), xin.grad.permute(0, 2, 3, 1)) < 3e-6
    assert rel(dw.cpu(), wd.grad) < 2e-5


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("vertical", [True, False])
@pytest.mark.parametrize("dil", [1, 2, 4, 8, 16])
def test_bf16_wgrad3_tcg_exact_operands(C, vertical, dil):
    """The bf16 3-tap weight gradient (lf_wgrad_tcg precision 2, traced as lf_wgrad3_tc_bf16) vs torch-CPU fp64 autograd."""
    o = ops()
    g = torch.Generator().manual_seed(C + dil + 100 * vertical)
    N, H, W = 2, 32, 64
    x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    dy = bx(torch.randn(N, H, W, C, generator=g)).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = torch.zeros(C, C, kh, kw, device="cuda")
    assert in_mode("bf16", lambda: o.wgrad3_tcg_ok(N, H, W, C))
    dw, db = in_mode("bf16", lambda: o.wgrad3(x, dy, w, vertical, dil))
    wd = torch.zeros(C, C, kh, kw, dtype=torch.float64, requires_grad=True)
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    F.conv2d(x.double().cpu().permute(0, 3, 1, 2), wd, None, 1, pad, dl).backward(dy.double().cpu().permute(0, 3, 1, 2))
    assert rel(dw.cpu(), wd.grad) < 2e-5
    assert rel(db.cpu(), dy.double().cpu().sum(dim=(0, 1, 2))) < 1e-5


@pytest.mark.parametrize("kind,C,O,tot,H,W,N", [("conv", 16, 48, 64, 128, 256, 2), ("conv", 64, 64, 128, 64, 128, 3),
                                                ("convT", 64, 128, 0, 32, 64, 2), ("convT", 16, 64, 0, 64, 128, 2),
                                                ("convT", 64, 96, 0, 32, 64, 2), ("conv", 16, 32, 32, 64, 128, 2)])
def test_bf16_tcg_weight_gradients(kind, C, O, tot, H, W, N):
    """lf_wgrad_tcg precision 2 over Nn in {32, 64, 96, 128} vs fp64 autograd."""
    o = ops()
    g = torch.Generator().manual_seed(C * 7 + O)
    if kind == "conv":
        x = bx(torch.randn(N, H, W, C, generator=g)).cuda()
        dcat = bx(torch.randn(N, H // 2, W // 2, tot, generator=g)).cuda()
        dw = in_mode("bf16", lambda: (o.wgrad_tcg_ok(x, C, dcat, ((O + 31) // 32) * 32), o.wgrad_tcg_conv(x, C, dcat, O)))
        w = torch.zeros(O, C, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv2d(x.permute(0, 3, 1, 2).double().cpu(), w, stride=2, padding=1).backward(dcat[..., :O].permute(0, 3, 1, 2).double().cpu())
    else:
        x = bx(torch.randn(N, H, W, O, generator=g)).cuda()
        du = bx(torch.randn(N, 2 * H, 2 * W, C, generator=g)).cuda()
        dw = in_mode("bf16", lambda: (o.wgrad_tcg_ok(du, C, x, O), o.wgrad_tcg_convT(x, O, du, C)))
        w = torch.zeros(O, C, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv_transpose2d(x.permute(0, 3, 1, 2).double().cpu(), w, stride=2, padding=1, output_padding=1).backward(
            du.permute(0, 3, 1, 2).double().cpu())
    assert dw[0]
    assert rel(dw[1].cpu(), w.grad) < 2e-5


@pytest.mark.parametrize("N,C,H,W,vertical,dil", CASES[:6])
def test_bf16_generic_operands(N, C, H, W, vertical, dil):
    """Generic fp32 operands: within the bf16 rounding scale of fp64 (forward, input gradient, weight gradient)."""
    o = ops()
    g = torch.Generator().manual_seed(N * 1000 + C + dil)
    x = torch.randn(N, H, W, C, generator=g).cuda()
    dy = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    y, dx, (dw, _) = in_mode("bf16", lambda: (o.conv3(x, w, vertical, dil, False), o.conv3(dy, w, vertical, dil, True),
                                              o.wgrad3(x, dy, w, vertical, dil)))
    xin = x.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
    wd = w.double().cpu().requires_grad_(True)
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    ref = F.conv2d(xin, wd, None, 1, pad, dl)
    ref.backward(dy.double().cpu().permute(0, 3, 1, 2))
    errs = (rel(y.cpu(), ref.detach().permute(0, 2, 3, 1)), rel(dx.cpu(), xin.grad.permute(0, 2, 3, 1)), rel(dw.cpu(), wd.grad))
    print("bf16 generic err (fwd, dgrad, wgrad):", errs)
    assert max(errs) < GENERIC_GATE, errs
    assert max(errs) > 2.0 ** -14, errs       # it IS bf16 arithmetic, not an fp32 path


def _net(B, L=2):
    from oracle import golden_check
    model, args = golden_check.build_net(L, 2, 0.3, B)
    torch.manual_seed(3)
    model = model.cuda().train()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0
        if isinstance(m, torch.nn.BatchNorm2d):
            m.momentum = 0.0
    return model, args


def test_bf16_weight_pack_cache_serves_bf16_operands():
    """In bf16 mode WeightPackCache serves operands bit-identical to fn(w).to(torch.bfloat16), picks up in-place updates,
    and a mode switch never serves an operand of another form."""
    from lanedetection_end2end_b200 import ops_net as o, _capi
    prev = o.CONV_MODE
    o.set_conv_mode("bf16")
    try:
        B = 2
        model, _ = _net(B)
        x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=11)).cuda()

        def step():
            model.zero_grad(set_to_none=True)
            out = model(x, torch.zeros(B, 4), True)
            betas = [b for b in out[:4] if b is not None]
            sum((b ** 2).sum() for b in betas).backward()
            torch.cuda.synchronize()
            return torch.cat([b.flatten() for b in betas]).clone(), {n: p.grad.clone() for n, p in model.named_parameters()
                                                                    if p.grad is not None}

        b1, g1 = step()
        packs = model.net.__dict__["_weight_packs"]
        assert len(packs.entries) > 100 and packs.dirty
        _capi.TRACE = []
        b2, g2 = step()
        names = [t[0] for t in _capi.TRACE]
        _capi.TRACE = None
        assert names.count("lf_pack_gather") == 1
        assert "lf_conv1d_tc_bf16" in names and "lf_wgrad3_tc_bf16" in names and "lf_conv_tcg" in names
        assert "lf_conv1d_tc" not in names and "lf_conv1d_tc_x3" not in names
        assert torch.equal(b1, b2)
        for n in g1:
            assert torch.equal(g1[n], g2[n]), n
        tc_entries = [(k, e) for k, e in packs.entries.items() if k[1].startswith("tc") or k[1].startswith("tcg")]
        assert tc_entries and all(k[2] == "bf16" and e[2].dtype == torch.bfloat16 for k, e in tc_entries)
        with torch.no_grad():
            for p in model.parameters():
                p.mul_(1.01)
        w = model.net.encoder.layers[1].conv3x1_1.weight
        e = packs.entries[(w.data_ptr(), "tc_fwd", "bf16")]
        assert packs.get(w, "tc_fwd", o.pack_tc_fwd, "bf16") is None       # stale: not served
        b3, _ = step()
        assert torch.equal(e[2], o.pack_tc_fwd(w).to(torch.bfloat16))
        assert not torch.equal(b3, b2)
        # every registered bf16 operand is bit-identical to its packer's output rounded by torch
        for (ptr_, kind, split), e in packs.entries.items():
            if split == "bf16":
                assert e[3] == e[0]._version
        # mode switch: the 3xTF32 operand of the same weight is a different entry, never the bf16 one
        o.set_conv_mode("tf32x3")
        step()
        step()
        t = o.packed(w, "tc_fwd", o.pack_tc_fwd, split=o.pack_split())
        assert t.dtype == torch.float32 and t.dim() == 3
        o.set_conv_mode("bf16")
        t = o.packed(w, "tc_fwd", o.pack_tc_fwd, split=o.pack_split())
        assert t.dtype == torch.bfloat16 and torch.equal(t, o.pack_tc_fwd(w).to(torch.bfloat16))
    finally:
        o.set_conv_mode(prev)
        o.ACTIVE_PACKS = None


@pytest.mark.parametrize("name", ["net_l2_d2", "net_l4_d3"])
def test_full_path_bf16_mode_accuracy(name):
    """bf16 mode on the golden inputs: beta norm-wise error and loss error vs fp64 (a labelled fast mode, outside the 1e-4
    gate; gated at about 2x the H100 numbers in tests/golden/bf16_accuracy_<case>.json)."""
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from oracle import golden_check
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(g["meta"]))
    L, order, B = meta["L"], meta["order"], meta["B"]
    model, args = golden_check.build_net(L, order, meta["mask_pct"], B)
    sd = model.state_dict()
    for k, v in inputs.make_erfnet_params(3, L, seed=meta["param_seed"]).items():
        sd[k] = torch.from_numpy(v)
    model.load_state_dict(sd)
    model = model.cuda().train()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=meta["image_seed"])).cuda()
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=meta["target_seed"])
    xgt, valid = torch.from_numpy(xgt_np).cuda(), torch.from_numpy(valid_np).cuda()
    ops_net.set_conv_mode("bf16")
    try:
        out = model(x, torch.zeros(B, 4), True)
        crit = backprojection_loss(args)
        loss = sum(crit(out[l], xgt[:, l], valid[:, l])[0] for l in range(L)) / L
        loss.backward()
        torch.cuda.synchronize()
    finally:
        ops_net.set_conv_mode("tf32x3")
    ours = torch.stack([out[l].squeeze(-1) for l in range(L)], 1).detach().cpu().numpy()
    nw = lambda a, b: float((np.abs(a - b).max(-1) / np.abs(b).max(-1)).max())
    rec = {"case": name, "beta_normwise_err_bf16": nw(ours, g["beta_f64"]), "beta_normwise_err_ref_fp32": nw(g["beta_f32"], g["beta_f64"]),
           "loss_rel_err_bf16": abs(float(loss.detach()) - float(g["loss_f64"])) / abs(float(g["loss_f64"])),
           "gpu": torch.cuda.get_device_name()}
    outdir = os.environ.get("LANEFIT_ACCURACY_OUT")   # optional: where to write the measured record (re-measuring the golden)
    if outdir and os.path.isdir(outdir):
        with open(os.path.join(outdir, "bf16_accuracy_%s.json" % name), "w") as f:
            json.dump(rec, f)
    print(rec)
    committed = os.path.join(GOLDEN, "bf16_accuracy_%s.json" % name)
    if os.path.exists(committed):
        h100 = json.load(open(committed))
        gate_beta = 2 * h100["beta_normwise_err_bf16"]
        gate_loss = max(2 * h100["loss_rel_err_bf16"], 1e-3)
    else:
        gate_beta, gate_loss = 2e-2, 5e-2
    assert rec["beta_normwise_err_bf16"] < gate_beta and rec["loss_rel_err_bf16"] < gate_loss, rec


def test_bf16_training_lowers_the_loss():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import train_synthetic
    from lanedetection_end2end_b200 import ops_net
    ops_net.set_conv_mode("bf16")
    try:
        rep = train_synthetic.run(steps=40, batch=4)
    finally:
        ops_net.set_conv_mode("tf32x3")
    assert rep["skipped"] == 0
    assert rep["loss_last"] < 0.5 * rep["loss_first"], rep
    assert all(v == v and v < 1e12 for v in rep["losses"]), rep


def test_bf16_graph_replay_matches_eager_step_and_eval_runs():
    from lanedetection_end2end_b200 import ops_net, _capi
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    ops_net.set_conv_mode("bf16")
    try:
        B, L = 2, 2
        model, args = _net(B, L)
        model.defer_status_check = True
        crit = backprojection_loss(args)
        x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=5)).cuda()
        xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=6)
        xgt, valid = torch.from_numpy(xgt_np).cuda(), torch.from_numpy(valid_np).cuda()

        def eager():
            model.zero_grad(set_to_none=True)
            out = model(x, torch.zeros(B, 4), True)
            loss = sum(crit(out[l], xgt[:, l], valid[:, l])[0] for l in range(L)) / L
            loss.backward()
            torch.cuda.synchronize()
            return float(loss), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
        eager()
        l_e, g_e = eager()
        step = GraphedTrainStep(model, crit, L, x, xgt, valid, None)
        l_g = float(step())
        torch.cuda.synchronize()
        assert abs(l_g - l_e) <= 1e-6 * abs(l_e), (l_g, l_e)
        for n, p in model.named_parameters():
            if n in g_e:       # (a conv bias followed by BatchNorm has an exactly zero gradient)
                assert float((p.grad - g_e[n]).abs().max()) <= 1e-5 * float(g_e[n].abs().max()), n
        del step
        # eval mode (ops_eval, BatchNorm folded into bf16 operands)
        model.eval()
        _capi.TRACE = []
        with torch.no_grad():
            out = model(x, torch.zeros(B, 4), True)
        torch.cuda.synchronize()
        names = [t[0] for t in _capi.TRACE]
        _capi.TRACE = None
        assert "lf_conv1d_tc_bf16" in names and "lf_conv_tcg" in names
        assert all(bool(torch.isfinite(o_).all()) for o_ in out[:L])
    finally:
        _capi.TRACE = None
        ops_net.set_conv_mode("tf32x3")
        ops_net.ACTIVE_PACKS = None
