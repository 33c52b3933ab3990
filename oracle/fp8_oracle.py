"""CPU restatement of the inference-only fp8 convolution mode (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Semantics (ops_net.set_conv_mode("fp8"), ops_eval.py, csrc/conv_tc.cu lf_conv1d_tc_fp8), restated here independently of
the product code:
  * weights (BatchNorm folded: w' = w * scale[co]): a_w[co] = max |w'[co]|, q_w = e4m3(w' * (448 / a_w[co])),
    s_w[co] = a_w[co] / 448; a_w = 0 -> q_w = 0, s_w = 0;
  * activations, per image n of each 3-tap convolution's STORED input (bf16 for t1..t3, fp32 for the block input):
    a_x[n] = max |v|, q = e4m3(v * (448 / a_x[n])) (fp32 multiply, then round to nearest even with saturation);
    a_x[n] = 0 -> q = 0;
  * output, each step one fp32 operation rounded to nearest: y = acc * ((a_x[n] / 448) * s_w[co]) + b', then ReLU
    (or + x and ReLU for a block's last convolution); t1..t3 are stored as bf16.
acc is the exact sum of the quantised products, rounded to fp32 once (the kernel sums each tap's 32-channel chunk on the
tensor core and the chunks with fp32 adds: within fp32 accumulation of it).
The stride-2 layers run with bf16 operands (BatchNorm folded), the stem and the output ConvTranspose2d in fp32.

eval_forward(x, P, mode) runs erfnet_oracle.erfnet_forward(training=False) with the blocks replaced by these
restatements: mode "fp8" (the fp8 mode), "bf16" (every convolution but the stem / output one on bf16 operands: the bf16
mode's eval path), or "exact" (erfnet_oracle's own blocks, in the parameters' dtype).
"""
import contextlib
import json
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import erfnet_oracle as eo
from . import inputs
from . import lsq_oracle as lo
from .golden_check import GOLDEN

E4M3_MAX = 448.0


def e4m3(v):
    """Round fp32 values within +-448 (saturated first) to e4m3 (nearest even) and back to fp32."""
    return v.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).float()


def inverse_scale(a):
    """448 / a, IEEE fp32 division (as tensor / tensor), 0 where a = 0."""
    e = torch.full_like(a, E4M3_MAX)
    return torch.where(a > 0, e / torch.where(a > 0, a, e), torch.zeros_like(a))


def scale(a):
    """a / 448, IEEE fp32 division."""
    return a / torch.full_like(a, E4M3_MAX)


def quantize_weight(w):
    """w [Co, ...] fp32 -> (q_w fp32 holding e4m3 values, s_w [Co])."""
    a = w.abs().amax(dim=tuple(range(1, w.dim())))
    return e4m3(w * inverse_scale(a).view((-1,) + (1,) * (w.dim() - 1))), scale(a)


def image_amax(v):
    """[N, ...] -> [N] fp32: max |v| per image."""
    return v.float().abs().flatten(1).amax(1)


def quantize_act(v, amax):
    """Stored activations v [N, ...] and their per-image max [N] -> fp32 tensor holding the e4m3 operand."""
    return e4m3(v.float() * inverse_scale(amax).view((-1,) + (1,) * (v.dim() - 1)))


def conv3_fp64(qx, qw, vertical, dil):
    """fp64 evaluation of one 3-tap convolution (NCHW) from the quantised operands: the exact sum of the products."""
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    return F.conv2d(qx.double(), qw.double(), None, 1, pad, dl)


def dequantize(acc, amax_x, s_w, b):
    """y = acc * ((a_x[n] / 448) * s_w[co]) + b, fp32, each operation rounded to nearest (acc [N, Co, H, W] fp32)."""
    return acc * (scale(amax_x).view(-1, 1, 1, 1) * s_w.view(1, -1, 1, 1)) + b.view(1, -1, 1, 1)


def conv3_fp8(x, w, b, vertical, dil, relu=True, add=None, store_bf16=False):
    """One fp8 3-tap convolution of a stored NCHW input x: -> (stored output fp32 tensor, its per-image max)."""
    ax = image_amax(x)
    qw, sw = quantize_weight(w.float())
    y = dequantize(conv3_fp64(quantize_act(x, ax), qw, vertical, dil).float(), ax, sw, b.float())
    if relu:
        y = F.relu(y)
    if add is not None:
        y = F.relu(y + add)
    if store_bf16:
        y = y.bfloat16().float()
    return y, image_amax(y)


def bn_affine(P, bn):
    """(scale, shift) of an eval-mode BatchNorm (eps 1e-3): y = x * scale + shift."""
    scale = P[bn + ".weight"] * torch.rsqrt(P[bn + ".running_var"] + eo.BN_EPS)
    return scale, P[bn + ".bias"] - P[bn + ".running_mean"] * scale


def fold(P, conv, bn, out_dim=0):
    """(w', b') of a convolution followed by an eval-mode BatchNorm, output channels along `out_dim` of w."""
    scale, shift = bn_affine(P, bn)
    w = P[conv + ".weight"]
    shape = [1] * w.dim()
    shape[out_dim] = -1
    return w * scale.view(shape), P[conv + ".bias"] * scale + shift


def _bf16(t):
    return t.bfloat16().float()


def nb1d_fp8(x, P, prefix, dil, training=False, drop_mask=None, taps=None, stats_out=None):
    w2, b2 = fold(P, prefix + ".conv1x3_1", prefix + ".bn1")
    w4, b4 = fold(P, prefix + ".conv1x3_2", prefix + ".bn2")
    t, _ = conv3_fp8(x, P[prefix + ".conv3x1_1.weight"], P[prefix + ".conv3x1_1.bias"], True, 1, store_bf16=True)
    t, _ = conv3_fp8(t, w2, b2, False, 1, store_bf16=True)
    t, _ = conv3_fp8(t, P[prefix + ".conv3x1_2.weight"], P[prefix + ".conv3x1_2.bias"], True, dil, store_bf16=True)
    return conv3_fp8(t, w4, b4, False, dil, relu=False, add=x)[0]


def nb1d_bf16(x, P, prefix, dil, training=False, drop_mask=None, taps=None, stats_out=None):
    w2, b2 = fold(P, prefix + ".conv1x3_1", prefix + ".bn1")
    w4, b4 = fold(P, prefix + ".conv1x3_2", prefix + ".bn2")
    w1, b1 = P[prefix + ".conv3x1_1.weight"], P[prefix + ".conv3x1_1.bias"]
    w3, b3 = P[prefix + ".conv3x1_2.weight"], P[prefix + ".conv3x1_2.bias"]
    t = _bf16(F.relu(F.conv2d(_bf16(x), _bf16(w1), b1, padding=(1, 0))))
    t = _bf16(F.relu(F.conv2d(t, _bf16(w2), b2, padding=(0, 1))))
    t = _bf16(F.relu(F.conv2d(t, _bf16(w3), b3, padding=(dil, 0), dilation=(dil, 1))))
    return F.relu(F.conv2d(t, _bf16(w4), b4, padding=(0, dil), dilation=(1, dil)) + x)


def downsampler_bf16(x, P, prefix, training=False, taps=None, stats_out=None):
    """Eval DownsamplerBlock with bf16 conv operands; the 3-channel stem stays fp32 (erfnet_oracle's block)."""
    if prefix == "encoder.initial_block":
        return _EXACT["downsampler"](x, P, prefix, False, taps, stats_out)
    cc = P[prefix + ".conv.weight"].shape[0]
    scale, shift = bn_affine(P, prefix + ".bn")
    w = P[prefix + ".conv.weight"] * scale[:cc].view(-1, 1, 1, 1)
    b = P[prefix + ".conv.bias"] * scale[:cc] + shift[:cc]
    c = F.conv2d(_bf16(x), _bf16(w), b, stride=2, padding=1)
    p = F.max_pool2d(x, 2, stride=2) * scale[cc:].view(1, -1, 1, 1) + shift[cc:].view(1, -1, 1, 1)
    return F.relu(torch.cat([c, p], 1))


def upsampler_bf16(x, P, prefix, training=False, taps=None, stats_out=None):
    w, b = fold(P, prefix + ".conv", prefix + ".bn", out_dim=1)
    return F.relu(F.conv_transpose2d(_bf16(x), _bf16(w), b, stride=2, padding=1, output_padding=1))


_EXACT = {"downsampler": eo.downsampler, "non_bottleneck_1d": eo.non_bottleneck_1d, "upsampler": eo.upsampler}
_MODES = {"fp8": {"downsampler": downsampler_bf16, "non_bottleneck_1d": nb1d_fp8, "upsampler": upsampler_bf16},
          "bf16": {"downsampler": downsampler_bf16, "non_bottleneck_1d": nb1d_bf16, "upsampler": upsampler_bf16},
          "exact": _EXACT}


@contextlib.contextmanager
def _blocks(mode):
    saved = {k: getattr(eo, k) for k in _EXACT}
    try:
        for k, fn in _MODES[mode].items():
            setattr(eo, k, fn)
        yield
    finally:
        for k, fn in saved.items():
            setattr(eo, k, fn)


def eval_forward(x, P, mode):
    """erfnet_oracle's eval-mode forward (running statistics from P) with the blocks of `mode` -> (enc, dec)."""
    with torch.no_grad(), _blocks(mode):
        return eo.erfnet_forward(x, P, training=False)


def with_training_statistics(x, P):
    """P (fp32) with every BatchNorm's running mean / (unbiased) variance set to the batch statistics of one fp64
    training-mode forward of x, so an eval forward sees activations at training scale -> (P32, P64)."""
    P64 = {k: v.double() for k, v in P.items()}
    stats = {}
    with torch.no_grad():
        eo.erfnet_forward(x.double(), P64, training=True, stats_out=stats)
    for bn, (m, v) in stats.items():
        P64[bn + ".running_mean"], P64[bn + ".running_var"] = m, v
    return {k: v.float() for k, v in P64.items()}, P64


def eval_beta(dec, grid, order, zero_rows):
    """Curve coefficients of an eval forward's decoder output: square activation, row mask, weighted least squares
    (BP/main.py:452 -> LSQ_layer) -> beta [B, L, d+1] float64."""
    masked = lo.activate_and_mask(dec, "square", zero_rows)
    beta, _ = lo.wls_forward(masked, grid.to(dec.dtype), order, 255.0, 0.0)
    return beta.double()


def normwise(a, b):
    """max over (image, lane) of max |a - b| / max |b| along the coefficients."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float((np.abs(a - b).max(-1) / np.abs(b).max(-1)).max())


def emulate_golden_case(name):
    """Golden case `name` (net_l2_d2 / net_l4_d3) in eval mode with running statistics from one training-mode forward
    of its input -> (record of beta's norm-wise error from the fp64 eval forward for the fp8, bf16 and fp32
    arithmetic, P32 with those statistics, beta64 [B, L, d+1])."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(g["meta"]))
    L, order, B = meta["L"], meta["order"], meta["B"]
    P = {k[4:]: torch.from_numpy(v).float() for k, v in inputs.make_erfnet_params(3, L, seed=meta["param_seed"]).items()}
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=meta["image_seed"])).float()
    grid = torch.from_numpy(np.load(os.path.join(GOLDEN, "lsq_bp_l2_d2.npz"))["grid0"])
    zero_rows = lo.mask_rows(256, meta["mask_pct"])
    P32, P64 = with_training_statistics(x, P)
    beta64 = eval_beta(eval_forward(x.double(), P64, "exact")[1], grid.double(), order, zero_rows).numpy()
    rec = {"case": name}
    for mode in ("fp8", "bf16", "exact"):
        beta = eval_beta(eval_forward(x, P32, mode)[1], grid, order, zero_rows).numpy()
        rec["beta_normwise_err_%s" % ("fp32" if mode == "exact" else mode)] = normwise(beta, beta64)
    return rec, P32, beta64
