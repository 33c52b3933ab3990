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

In the inference-only fp8 mode the four convolutions of a non_bottleneck_1d run on lf_conv1d_tc_fp8: e4m3 weights
quantised per output channel (quantize_fp8_weight, cached like the folded operands) and activations quantised per image
inside the kernel from a per-image max |x| that the producing convolution's epilogue reduces (out_amax), or, for a
block input that a Downsampler / Upsampler produced, one lf_amax_per_image launch.  down / up run as in bf16 mode.

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


def quantize_fp8_weight(w):
    """fp8 operand of a convolution weight w [Co, ...] (fp32): a_w[co] = max |w[co]|, q = e4m3(w * (448 / a_w[co]))
    (both fp32 operations rounded to nearest; the product is within +-448, so torch's float8_e4m3fn conversion is the
    round-to-nearest-even, saturating one of the kernel) and the dequantisation factor s_w[co] = a_w[co] / 448.  A channel
    with a_w = 0 gets q = 0 and s_w = 0.  -> (q float8_e4m3fn, s_w fp32 [Co])."""
    a = w.abs().amax(dim=tuple(range(1, w.dim())))
    e = torch.full_like(a, 448.0)   # tensor / tensor: IEEE division (torch may multiply by a scalar divisor's reciprocal)
    inv = torch.where(a > 0, e / torch.where(a > 0, a, e), torch.zeros_like(a))
    q = (w * inv.view((-1,) + (1,) * (w.dim() - 1))).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q, a / e


def _fp8_operand(w, vertical, sup):
    """(packed e4m3 operand as uint8 [Co][3*Ci], w_scale [Co]) of lf_conv1d_tc_fp8; super-pixel layers: the [64][192]
    operand of the quantised 16 -> 16 weight and its scales per super-channel."""
    q, s = quantize_fp8_weight(w)
    qf = q.float()                            # e4m3 values are exact in fp32: packing moves them unchanged
    wp = o.pack_tc_super(qf, vertical, False) if sup else o.pack_tc_fwd(qf)
    return wp.to(torch.float8_e4m3fn).view(torch.uint8).contiguous(), (s.repeat(o.SUPER) if sup else s).contiguous()


def nb1d_operands(mod, sup):
    """The cached operands of a non_bottleneck_1d in the active mode: [(wp2, b2), (wp4, b4)] (conv1x3_1 / conv1x3_2 with
    bn1 / bn2 folded; conv3x1_1 / conv3x1_2 go through the weight packer), or in fp8 mode [(wq, w_scale, bias)] for all
    four convolutions.  The cache key includes the mode: a mode switch rebuilds them."""
    c1, c2, c3, c4 = mod.conv3x1_1, mod.conv1x3_1, mod.conv3x1_2, mod.conv1x3_2
    fp8 = o.fp8_mode()

    def folded(conv, bn):
        scale, shift = bn_affine(bn)
        return conv.weight.detach() * scale.view(-1, 1, 1, 1), conv.bias.detach() * scale + shift

    def build():
        if fp8:
            ws = [(c1.weight.detach(), c1.bias.detach()), folded(c2, mod.bn1), (c3.weight.detach(), c3.bias.detach()),
                  folded(c4, mod.bn2)]
            return [_fp8_operand(w, k % 2 == 0, sup) + (b.contiguous(),) for k, (w, b) in enumerate(ws)]
        res = []
        for conv, bn in ((c2, mod.bn1), (c4, mod.bn2)):
            w, b = folded(conv, bn)
            wp = o.pack_tc_super(w, False, False) if sup else o.pack_tc_fwd(w)
            res.append((o.tc_operand(wp).contiguous(), b.contiguous()))
        return res

    tensors = [c2.weight, c2.bias, c4.weight, c4.bias] + _bn_tensors(mod.bn1) + _bn_tensors(mod.bn2)
    if fp8:
        tensors += [c1.weight, c1.bias, c3.weight, c3.bias]
    return _cached(mod, tensors, build)


def nb1d(x, mod):
    """relu(bn2(conv1x3_2(relu(conv3x1_2(relu(bn1(conv1x3_1(relu(conv3x1_1(x)))))))) + x) with both BatchNorms folded, or
    None when a tensor-core kernel does not take the shape."""
    N, H, W, C = x.shape
    dil = mod.dilated
    sup = o.super_ok(x, 1) and dil == 1
    if not sup and not all(o.tc_supported(x, v, d) for v in (True, False) for d in (1, dil)):
        return None
    if o.fp8_mode():
        return _nb1d_fp8(x, mod, sup)
    c1, c3 = mod.conv3x1_1, mod.conv3x1_2
    (wp2, b2), (wp4, b4) = nb1d_operands(mod, sup)
    sd = o.nb1d_storage_dtype(x, dil)     # the three intermediates are convolution inputs only
    t = o.conv3(x, c1.weight, True, 1, False, bias=c1.bias, relu=True, dtype=sd)
    t = o.conv3(t, None, False, 1, False, wp=wp2, bias=b2, relu=True, dtype=sd)
    t = o.conv3(t, c3.weight, True, dil, False, bias=c3.bias, relu=True, dtype=sd)
    return o.conv3(t, None, False, dil, False, wp=wp4, bias=b4, relu=2, add_src=x)


_FP8_LAST = None   # (output, its per-image max |.| [N]) of the last fp8 block: the next block's input scale


def block_input_amax(x):
    """Per-image max |x| of an fp8 block input: the previous block's out_amax when x is that block's output (same
    memory, shape, strides and version), else one lf_amax_per_image launch."""
    last = _FP8_LAST
    if (last is not None and last[0].data_ptr() == x.data_ptr() and last[0].shape == x.shape and last[0].stride() == x.stride()
            and last[0].dtype == x.dtype and last[0]._version == x._version):
        return last[1]
    N = x.shape[0]
    am = torch.zeros(N, dtype=torch.float32, device=x.device)
    _capi.call("lf_amax_per_image", ptr(x), _capi.dtype_id(x), x.numel() // N, N, ptr(am), o._stream())
    return am


def _nb1d_fp8(x, mod, sup):
    """The fp8 block: four lf_conv1d_tc_fp8 launches; each epilogue reduces the per-image max of what it stores (t1..t3
    as in bf16 mode, y fp32), which is the next convolution's activation scale."""
    global _FP8_LAST
    dil = mod.dilated
    (w1, s1, b1), (w2, s2, b2), (w3, s3, b3), (w4, s4, b4) = nb1d_operands(mod, sup)
    am = torch.zeros(4, x.shape[0], dtype=torch.float32, device=x.device)   # max |t1|, |t2|, |t3|, |y| per image
    ax = block_input_amax(x)
    sd = o.nb1d_storage_dtype(x, dil)
    t = o.conv3(x, None, True, 1, False, wp=w1, bias=b1, relu=True, dtype=sd, fp8=(ax, s1, am[0]))
    t = o.conv3(t, None, False, 1, False, wp=w2, bias=b2, relu=True, dtype=sd, fp8=(am[0], s2, am[1]))
    t = o.conv3(t, None, True, dil, False, wp=w3, bias=b3, relu=True, dtype=sd, fp8=(am[1], s3, am[2]))
    y = o.conv3(t, None, False, dil, False, wp=w4, bias=b4, relu=2, add_src=x, fp8=(am[2], s4, am[3]))
    _FP8_LAST = (y, am[3])
    return y


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
