"""Eval-mode fused inference of the ERFNet blocks (SURVEY.md 8f-4; the reference's validate() / test_model() run
model.eval(): BP/main.py:419-526, BP/test.py:23-129).

With running statistics a BatchNorm2d is a per-channel affine known before the launch, so it is folded into the
convolution that feeds it (w' = w * scale[co], b' = b * scale + shift) and every block becomes convolution launches only:

  non_bottleneck_1d   4 launches: conv3x1_1 (+bias, ReLU), conv1x3_1' (bn1 folded, ReLU), conv3x1_2 (+bias, ReLU),
                      conv1x3_2' (bn2 folded) + residual + ReLU in the epilogue (LfConvTcArgs.relu bit 1); Dropout2d is
                      the identity in eval mode.  Was 4 convs + 2 lf_bn_eval_prepare + 2 lf_bn_apply.
  DownsamplerBlock    2 launches: stride-2 conv' (folded, ReLU in the epilogue) + max-pool with the affine and ReLU of its
                      channel slice (lf_maxpool2_affine_relu).
  UpsamplerBlock      2 launches (one per output-row parity): transposed conv' (folded, ReLU).

The folded, GEMM-layout (and TF32 hi/lo split) operands are built once per set of parameter / running-statistics versions
and cached on the module -- parameter-sized torch ops, nothing per step.  Only taken for inference (no autograd graph) on
shapes the tensor-core kernels serve; everything else keeps the unfused eval path of ops_net (same results to fp32 rounding,
tests/test_net_gpu.py::test_eval_fused_matches_unfused)."""
import torch

from . import _capi
from . import ops_net as o

ptr = _capi.ptr


def bn_affine(bn):
    """(scale, shift) of an eval-mode BatchNorm2d: y = x * scale + shift."""
    scale = bn.weight.detach() * torch.rsqrt(bn.running_var + bn.eps)
    return scale, bn.bias.detach() - bn.running_mean * scale


def _cached(mod, tensors, build):
    key = tuple((t.data_ptr(), t._version) for t in tensors) + (o.CONV_MODE,)
    ent = mod.__dict__.get("_eval_fold")
    if ent is None or ent[0] != key:
        with torch.no_grad():
            ent = mod.__dict__["_eval_fold"] = (key, build())
    return ent[1]


def _bn_tensors(bn):
    return [bn.weight, bn.bias, bn.running_mean, bn.running_var]


def inference_only(*tensors):
    return not (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors))


def nb1d(x, mod):
    """relu(bn2(conv1x3_2(relu(conv3x1_2(relu(bn1(conv1x3_1(relu(conv3x1_1(x)))))))) + x) with both BatchNorms folded, or
    None when a tensor-core kernel does not take the shape."""
    N, H, W, C = x.shape
    dil = mod.dilated
    sup = o.super_ok(x, 1) and dil == 1
    if not sup and not all(o.tc_supported(x, v, d) for v in (True, False) for d in (1, dil)):
        return None
    c1, c2, c3, c4 = mod.conv3x1_1, mod.conv1x3_1, mod.conv3x1_2, mod.conv1x3_2

    def build():
        res = []
        for conv, bn in ((c2, mod.bn1), (c4, mod.bn2)):
            scale, shift = bn_affine(bn)
            w = conv.weight.detach() * scale.view(-1, 1, 1, 1)
            b = conv.bias.detach() * scale + shift
            wp = o.pack_tc_super(w, False, False) if sup else o.pack_tc_fwd(w)
            res.append((o.tc_operand(wp).contiguous(), b.contiguous()))
        return res

    (wp2, b2), (wp4, b4) = _cached(mod, [c2.weight, c2.bias, c4.weight, c4.bias] + _bn_tensors(mod.bn1) + _bn_tensors(mod.bn2), build)
    sd = o.nb1d_storage_dtype(x, dil)     # the three intermediates are convolution inputs only
    t = o.conv3(x, c1.weight, True, 1, False, bias=c1.bias, relu=True, dtype=sd)
    t = o.conv3(t, None, False, 1, False, wp=wp2, bias=b2, relu=True, dtype=sd)
    t = o.conv3(t, c3.weight, True, dil, False, bias=c3.bias, relu=True, dtype=sd)
    return o.conv3(t, None, False, dil, False, wp=wp4, bias=b4, relu=2, add_src=x)


def down(x, mod):
    """relu(bn(cat[conv3x3/s2(x), maxpool2(x)])) with the BatchNorm folded; None if the gather-GEMM does not take the layer."""
    N, H, W, cx = x.shape
    cin, w = mod.ninput, mod.conv.weight
    cc = w.shape[0]
    if not (cx == cin and cc % 16 == 0 and o.tcg_s2conv_ok(x, cin, cc)):
        return None

    def build():
        scale, shift = bn_affine(mod.bn)
        wf = w.detach() * scale[:cc].view(-1, 1, 1, 1)
        b = mod.conv.bias.detach() * scale[:cc] + shift[:cc]
        wg = o.pack_tcg_s2conv(wf)
        return o.tc_operand(wg).contiguous(), b.contiguous(), scale.contiguous(), shift.contiguous()

    wg, b, scale, shift = _cached(mod, [w, mod.conv.bias] + _bn_tensors(mod.bn), build)
    cat = torch.empty(N, H // 2, W // 2, cc + cin, dtype=torch.float32, device=x.device)
    o.run_tcg_s2conv(x, wg, cc, cat, bias=b, relu=True)
    _capi.call("lf_maxpool2_affine_relu", ptr(x), N, H, W, cin, cx, ptr(scale), ptr(shift), ptr(cat), cc + cin, cc, o._stream())
    return cat


def up(x, mod):
    """relu(bn(convT3x3/s2(x))) with the BatchNorm folded."""
    N, H, W, ci = x.shape
    w = mod.conv.weight                       # [ci, co, 3, 3]
    co = w.shape[1]
    if not o.tcg_s2convT_ok(x, ci, co):
        return None

    def build():
        scale, shift = bn_affine(mod.bn)
        wf = w.detach() * scale.view(1, -1, 1, 1)
        b = (mod.conv.bias.detach() * scale + shift).repeat(2)
        wgs = tuple(o.pack_tcg_s2convT(wf, par, ci) for par in (0, 1))
        return tuple(o.tc_operand(g).contiguous() for g in wgs), b.contiguous()

    wgs, b2 = _cached(mod, [w, mod.conv.bias] + _bn_tensors(mod.bn), build)
    out = torch.empty(N, 2 * H, 2 * W, co, dtype=torch.float32, device=x.device)
    return o.run_tcg_s2convT(x, ci, wgs, co, out, bias2=b2, relu=True)
