"""Host side of the Classification heads (`--clas 1`; BP/Networks/LSQ_layer.py:157-207, wired at :250-257,296-298)
on the library's kernels: each head is four conv -> BatchNorm2d(eps 1e-5) -> ReLU stages on the shared encoder output
([B,128,32,64]), a pooling step and one or two fully connected layers.

  conv 1x1 / 3x3 (stride 1)   lf_conv_tcg, the run-time-tap gather-GEMM on tensor cores (1 or 9 taps over one NHWC view; 3xTF32 in
                              the default mode), input gradient = the same kernel with mirrored taps and transposed weights,
                              weight gradient = lf_wgrad_tcg over the same taps; in fp32 mode (or for shapes the tensor-core
                              kernels do not tile) the CUDA-core implicit GEMM lf_conv_f32 / lf_wgrad_f32.
  BatchNorm + ReLU            the ERFNet kernels (lf_bn_stats / _finalize / _apply, lf_bn_bwd_*), eps passed per layer.
  MaxPool2d(2) + flatten      lf_maxpool2_fwd/bwd on NHWC, then lf_nhwc_to_nchw (the reference flattens NCHW).
  AvgPool2d((1,64)) + flatten lf_rowmean_fwd/bwd (writes the NCHW-flattened order directly).
  Linear (+ReLU)              lf_linear_fwd / _bwd_data / _bwd_weight (csrc/linear.cu; HBM-bound on the weights).
No torch operator touches a feature map; parameters stay in the reference's layouts / names (state_dict compatible).
"""
import ctypes

import torch

from . import _capi
from . import net_plans as plans
from . import ops_net as o

HEAD_BN_EPS = 1e-5           # nn.BatchNorm2d default (the heads do not pass eps; ERFNet's blocks use 1e-3)
ptr = _capi.ptr


def _taps(kh, kw, mirror=False):
    s = -1 if mirror else 1
    return [(s * (ky - (kh - 1) // 2), s * (kx - (kw - 1) // 2)) for ky in range(kh) for kx in range(kw)]


def dense_tcg_ok(x, Ng):
    N, H, W, C = x.shape
    return (o.tc_mode() and C % 32 == 0 and C <= 256 and Ng % 16 == 0 and Ng <= 128 and x.is_contiguous()
            and int(_capi.lib().lf_conv_tcg_supported(N, H, W, C, Ng)) > 0)


def run_tcg_dense(x, wg, taps, Ng, out, bias=None):
    """out[n,y,x,:Ng] = bias + sum_t x[n, y+dy_t, x+dx_t, :] . wg[:, t*C:(t+1)*C]  (stride-1 conv, zero padding = TMA OOB fill)."""
    N, H, W, C = x.shape
    cot = out.shape[-1]
    a = _capi.LfConvTcgArgs()
    a.a[0] = o._tcg_view(x, H, W, H * W * C, W * C, C)
    a.wg, a.bias, a.out = wg.data_ptr(), (bias.data_ptr() if bias is not None else None), out.data_ptr()
    a.osn, a.osy, a.osx, a.oy_mul, a.oy0 = H * W * cot, W * cot, cot, 1, 0
    a.N, a.Hs, a.Ws, a.Kc, a.Ng, a.ntaps = N, H, W, C, Ng, len(taps)
    a.precision = o.tcg_precision(wg)
    for t, (dy, dx) in enumerate(taps):
        a.map[t], a.dy[t], a.dx[t] = 0, dy, dx
    _capi.call("lf_conv_tcg", ctypes.byref(a), o._stream(), flops=2 * N * H * W * len(taps) * C * Ng,
               nbytes=4 * N * H * W * (C + Ng))
    return out


def conv_fwd(x, w, b):
    """Conv2d(stride 1, 'same' padding) of an NHWC tensor -> NHWC [N,H,W,Co]."""
    N, H, W, Ci = x.shape
    Co, _, kh, kw = w.shape
    out = torch.empty(N, H, W, Co, dtype=torch.float32, device=x.device)
    if dense_tcg_ok(x, Co):
        return run_tcg_dense(x, o.packed(w, "tc_fwd", o.pack_tc_fwd, split=o.pack_split()), _taps(kh, kw), Co, out, bias=b)
    phases, _ = plans.conv_fwd_plan(H, W, kh, kw, 1, (kh - 1) // 2, (kw - 1) // 2, 1, 1)
    return o.run_conv(phases, x, o.packed(w, "conv_fwd", o.pack_conv_fwd), Ci, out, Co, bias=b)


def conv_dgrad(dy, w):
    N, H, W, Co = dy.shape
    _, Ci, kh, kw = w.shape
    dx = torch.empty(N, H, W, Ci, dtype=torch.float32, device=dy.device)
    if dense_tcg_ok(dy, Ci):
        return run_tcg_dense(dy, o.packed(w, "tc_dgrad", o.pack_tc_dgrad, split=o.pack_split()), _taps(kh, kw, mirror=True), Ci, dx)
    phases, _ = plans.conv_dgrad_plan_s1(H, W, kh, kw, (kh - 1) // 2, (kw - 1) // 2, 1, 1)
    return o.run_conv(phases, dy, o.packed(w, "conv_dgrad", o.pack_conv_dgrad), Co, dx, Ci)


def _wgrad_tcg_dense(x, dy, taps):
    """-> [ntaps*Ci][Co]: row t*Ci + ci = sum over pixels of x[pixel + tap t][ci] * dy[pixel][:], or None if unsupported."""
    N, H, W, Ci = x.shape
    Co = dy.shape[-1]
    if not (o.tc_mode() and Ci % 32 == 0 and Co % 32 == 0 and Co <= 128 and x.is_contiguous() and dy.is_contiguous()):
        return None
    return o.wgrad_tcg_rows([o._tcg_view(x, H, W, H * W * Ci, W * Ci, Ci)], o._tcg_view(dy, H, W, H * W * Co, W * Co, Co),
                            [(0, ty, tx) for ty, tx in taps], N, H, W, Ci, Co, range(len(taps), 0, -1), x.device)


def conv_wgrad(x, dy, w):
    """dW [Co,Ci,kh,kw] of the stride-1 conv."""
    N, H, W, Ci = x.shape
    Co, _, kh, kw = w.shape
    res = _wgrad_tcg_dense(x, dy, _taps(kh, kw))
    if res is not None:
        return res.view(kh, kw, Ci, Co).permute(3, 2, 0, 1).contiguous()
    dw = torch.empty_like(w)
    o.run_wgrad(plans.conv_wgrad_plan(H, W, kh, kw, 1, (kh - 1) // 2, (kw - 1) // 2, 1, 1), x, Ci, dy, Co, 0, N, dw,
                (1, kh * kw, Ci * kh * kw))
    return dw


class ConvBnReluFunction(torch.autograd.Function):
    """relu(bn(conv(x) + b)) on NHWC fp32 (one stage of Classification.forward, reference :194-197)."""

    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, rm, rv, training, eps, sync=None):
        """sync: ops_net.BNSync (SyncBatchNorm container) or None."""
        _capi.require_cuda(x)
        u = conv_fwd(x, w, b)
        s = o.bn_forward_stats(u, gamma, beta, rm, rv, training, eps, sync=sync)
        y = o.bn_apply(u, s, relu=True)
        ctx.save_for_backward(x, w, u, y, gamma, s.mean, s.invstd, s.count)
        ctx.training, ctx.sync = training, sync
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, u, y, gamma, mean, invstd, count = ctx.saved_tensors
        o._require_training_for_backward(ctx.training)
        s = o.BNState()
        s.mean, s.invstd, s.count = mean, invstd, count
        du, dgamma, dbeta = o.bn_backward(dy.contiguous(), y, None, u, s, gamma, sync=ctx.sync)
        dw = conv_wgrad(x, du, w)
        # the conv feeds a training-mode BatchNorm: sum over pixels of du vanishes identically (DESIGN.md, deviations)
        db = torch.zeros(w.shape[0], dtype=torch.float32, device=x.device)
        dx = conv_dgrad(du, w) if ctx.needs_input_grad[0] else None
        return dx, dw, db, dgamma, dbeta, None, None, None, None, None


class MaxPool2FlatFunction(torch.autograd.Function):
    """MaxPool2d(2, 2) on NHWC, returned flattened in the reference's NCHW order: [B, C*(H/2)*(W/2)] (reference :199,202)."""

    @staticmethod
    def forward(ctx, x):
        N, H, W, C = x.shape
        st = o._stream()
        p = torch.empty(N, H // 2, W // 2, C, dtype=torch.float32, device=x.device)
        _capi.call("lf_maxpool2_fwd", ptr(x), N, H, W, C, C, ptr(p), C, 0, st)
        flat = torch.empty(N, C * (H // 2) * (W // 2), dtype=torch.float32, device=x.device)
        _capi.call("lf_nhwc_to_nchw", ptr(p), N, H // 2, W // 2, C, ptr(flat), st)
        ctx.save_for_backward(x)
        return flat

    @staticmethod
    def backward(ctx, dflat):
        x, = ctx.saved_tensors
        N, H, W, C = x.shape
        st = o._stream()
        dp = torch.empty(N, H // 2, W // 2, C, dtype=torch.float32, device=x.device)
        _capi.call("lf_nchw_to_nhwc", ptr(dflat.contiguous()), N, C, H // 2, W // 2, ptr(dp), st)
        dx = torch.empty_like(x)
        _capi.call("lf_maxpool2_bwd", ptr(x), N, H, W, C, C, ptr(dp), C, 0, ptr(dx), C, 0, st)
        return dx


class MaxPool2Function(torch.autograd.Function):
    """MaxPool2d(2, 2) on NHWC, NHWC out: [B, H/2, W/2, C] (the spatial-transformer branch pools between two convs)."""

    @staticmethod
    def forward(ctx, x):
        N, H, W, C = x.shape
        p = torch.empty(N, H // 2, W // 2, C, dtype=torch.float32, device=x.device)
        _capi.call("lf_maxpool2_fwd", ptr(x), N, H, W, C, C, ptr(p), C, 0, o._stream())
        ctx.save_for_backward(x)
        return p

    @staticmethod
    def backward(ctx, dp):
        x, = ctx.saved_tensors
        N, H, W, C = x.shape
        dx = torch.empty_like(x)
        _capi.call("lf_maxpool2_bwd", ptr(x), N, H, W, C, C, ptr(dp.contiguous()), C, 0, ptr(dx), C, 0, o._stream())
        return dx


class NchwFlatFunction(torch.autograd.Function):
    """NHWC [B, H, W, C] flattened in the reference's NCHW order, x.view(B, -1) on NCHW: [B, C*H*W]."""

    @staticmethod
    def forward(ctx, x):
        N, H, W, C = x.shape
        flat = torch.empty(N, C * H * W, dtype=torch.float32, device=x.device)
        _capi.call("lf_nhwc_to_nchw", ptr(x.contiguous()), N, H, W, C, ptr(flat), o._stream())
        ctx.shape = (N, H, W, C)
        return flat

    @staticmethod
    def backward(ctx, dflat):
        N, H, W, C = ctx.shape
        dx = torch.empty(N, H, W, C, dtype=torch.float32, device=dflat.device)
        _capi.call("lf_nchw_to_nhwc", ptr(dflat.contiguous()), N, C, H, W, ptr(dx), o._stream())
        return dx


class RowMeanFlatFunction(torch.autograd.Function):
    """AvgPool2d((1, W)) on NHWC, flattened in NCHW order: [B, C*H] (reference :184,201-202)."""

    @staticmethod
    def forward(ctx, x):
        N, H, W, C = x.shape
        out = torch.empty(N, C * H, dtype=torch.float32, device=x.device)
        _capi.call("lf_rowmean_fwd", ptr(x), N, H, W, C, ptr(out), o._stream())
        ctx.shape = (N, H, W, C)
        return out

    @staticmethod
    def backward(ctx, dout):
        N, H, W, C = ctx.shape
        dx = torch.empty(N, H, W, C, dtype=torch.float32, device=dout.device)
        _capi.call("lf_rowmean_bwd", ptr(dout.contiguous()), N, H, W, C, ptr(dx), o._stream())
        return dx


class LinearFunction(torch.autograd.Function):
    """y = x W^T + b (optionally ReLU) with W in nn.Linear's [O][K] layout."""

    @staticmethod
    def forward(ctx, x, W, b, relu):
        _capi.require_cuda(x)
        x = x.contiguous()
        B, K = x.shape
        O = W.shape[0]
        h = _capi.lib()
        partial = torch.empty(int(h.lf_linear_chunks(K)) * B * O, dtype=torch.float32, device=x.device)
        y = torch.empty(B, O, dtype=torch.float32, device=x.device)
        _capi.call("lf_linear_fwd", ptr(x), ptr(W.contiguous()), ptr(b), B, K, O, int(relu), ptr(partial), ptr(y), o._stream(),
                   flops=2 * B * K * O, nbytes=4 * (K * O + B * K + B * O))
        ctx.save_for_backward(x, W, y if relu else None)
        ctx.relu = relu
        return y

    @staticmethod
    def backward(ctx, dy):
        x, W, y = ctx.saved_tensors
        dy = dy.contiguous()
        B, K = x.shape
        O = W.shape[0]
        st = o._stream()
        dW = torch.empty_like(W)
        db = torch.empty(O, dtype=torch.float32, device=x.device)
        _capi.call("lf_linear_bwd_weight", ptr(dy), ptr(y), ptr(x), B, K, O, ptr(dW), ptr(db), st,
                   flops=2 * B * K * O, nbytes=4 * (K * O + B * K + B * O))
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _capi.call("lf_linear_bwd_data", ptr(dy), ptr(y), ptr(W.contiguous()), B, K, O, ptr(dx), st,
                       flops=2 * B * K * O, nbytes=4 * (K * O + B * K + B * O))
        return dx, dW, db, None


def conv_bn_relu(x, conv, bn, training, track):
    y = ConvBnReluFunction.apply(x, conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var, training,
                                 bn.eps, o.bn_sync(bn, training))
    track(bn, training)
    return y
