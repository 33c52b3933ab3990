"""Host side of the ERFNet blocks: one ``torch.autograd.Function`` per reference block
(DownsamplerBlock, non_bottleneck_1d, UpsamplerBlock, output ConvTranspose2d -- see
BP/Networks/ERFNet.py), each a fixed sequence of C-ABI launches (include/lanefit_b200.h)
on NHWC fp32 tensors.  Torch provides device memory, the stream and the autograd graph;
no torch operator touches a feature map on this path.

Training-mode memory plan per non_bottleneck_1d (what backward needs):
  x (block input), t1 = relu(conv3x1_1), t2 = conv1x3_1 (pre-BN), t3 = relu(bn1),
  t4 = relu(conv3x1_2), t5 = conv1x3_2 (pre-BN), y = block output, the two (mean, invstd)
  pairs and the dropout mask.  t1, t3 and t4 are only convolution inputs and ReLU masks: in bf16 mode
  they are stored as bf16 (nb1d_storage_dtype).
"""
import ctypes
import os

import torch

from . import _capi
from . import net_plans as plans

BN_EPS = 1e-3
BN_MOMENTUM = 0.1
LfConvArgs, LfWgradArgs, LfConvTcArgs = _capi.LfConvArgs, _capi.LfWgradArgs, _capi.LfConvTcArgs

# Convolution arithmetic for the dense 3-tap convolutions of non_bottleneck_1d (C in {64,128}):
#   "fp32": CUDA-core FFMA implicit GEMM (parity mode, fp32-exact)
#   "tf32x3": tensor cores, every product formed from TF32 hi/lo splits of both operands
#           (a_hi*w_hi + a_hi*w_lo + a_lo*w_hi, fp32 accumulate): fp32-grade results at tensor-core speed -- the
#           default, and the mode bench.py times (csrc/conv_tc.cu);
#   "tf32": tensor cores, single-pass TF32 multiply / fp32 accumulate (what cuDNN does for the reference's
#           fp32 convs on Ampere+ GPUs; 1e-3 from fp32 on the curve coefficients -- a labelled extra);
#   "bf16": tensor cores, both operands rounded to bf16 (nearest even) inside the kernels, exact products, fp32
#           accumulate (a labelled fast mode, ~5e-3 from fp64 on the curve coefficients); the non_bottleneck_1d
#           tensors that only feed convolutions and ReLU masks are stored as bf16 (same results, see
#           nb1d_storage_dtype), everything else stays fp32;
#   "fp8": INFERENCE ONLY (an eval-mode forward without autograd, ops_eval.py): the four 3-tap convolutions of every
#           non_bottleneck_1d run on FP8 e4m3 operands (weights scaled per output channel, activations per image,
#           lf_conv1d_tc_fp8); every other layer runs exactly as in bf16 mode (bf16_mode() is true in fp8 mode).  A
#           training forward or one that builds an autograd graph raises (require_inference_mode);
#   shapes a tensor-core kernel does not take stay on the fp32 kernel in every mode.
CONV_MODES = ("fp32", "tf32", "tf32x3", "bf16", "fp8")
CONV_MODE = os.environ.get("LANEFIT_CONV_MODE", "tf32x3")


def set_conv_mode(mode):
    global CONV_MODE
    if mode not in CONV_MODES:
        raise ValueError(mode)
    CONV_MODE = mode


def tc_mode():
    """True when the dense convolutions run on tensor cores (TF32, 3xTF32, BF16 or FP8)."""
    return CONV_MODE in ("tf32", "tf32x3", "bf16", "fp8")


def x3_mode():
    return CONV_MODE == "tf32x3"


def bf16_mode():
    """True when the layers run with bf16 operands: the bf16 mode, and every layer of the fp8 mode except the
    non_bottleneck_1d 3-tap convolutions of ops_eval."""
    return CONV_MODE in ("bf16", "fp8")


def fp8_mode():
    return CONV_MODE == "fp8"


def require_inference_mode(training, *tensors):
    """The fp8 mode serves eval-mode forwards without autograd only: raise for a training forward or one that would
    build an autograd graph (any of `tensors` requiring grad with grad mode on), instead of running another mode."""
    if fp8_mode() and (training or (torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors))):
        raise RuntimeError("conv mode 'fp8' is inference-only: run the model in eval mode under torch.no_grad() "
                           "(or torch.inference_mode()), or set another conv mode for training")


def pack_split():
    """The operand form the active mode's tensor-core kernels read, as the ``split`` argument of packed():
    True = the TF32 hi/lo pair (tf32x3), "bf16" = bf16 operand, False = the fp32 operand."""
    return "bf16" if bf16_mode() else x3_mode()


def tc_operand(t):
    """A packed fp32 tensor-core operand in the active mode's form (what packed() serves for ``pack_split()``)."""
    return split_tf32(t) if x3_mode() else t.to(torch.bfloat16) if bf16_mode() else t


def tcg_precision(wg):
    """LfConvTcgArgs.precision of a packed operand: 2 = bf16, 1 = [2, Ng, K] TF32 hi / lo pair, 0 = TF32."""
    return 2 if wg.dtype == torch.bfloat16 else int(wg.dim() == 3)


# Experiment switch (labelled extra in bench.py, never a default): in tf32x3 mode, run ONLY the weight-gradient kernels as
# single-pass TF32.  Activations, beta, the loss and every input gradient stay fp32-grade; the parameter gradients pick up
# TF32 rounding noise (~5e-4, a sum of ~65 k independently rounded products), which is below the reference's own fp32-vs-fp64
# gradient noise on this ill-conditioned path (2.6e-3 .. 3.8e-2, SURVEY.md 7.2 #1) -- but above the 1e-4 the north star
# names, hence not the default.
WGRAD_SINGLE_PASS = os.environ.get("LANEFIT_WGRAD_TF32", "0") == "1"


def wgrad_x3():
    return x3_mode() and not WGRAD_SINGLE_PASS


def wgrad_precision():
    """LfWgradTcgArgs.precision of the active mode (0 = TF32, 1 = 3xTF32, 2 = BF16)."""
    return 2 if bf16_mode() else int(wgrad_x3())


def split_tf32(t):
    """fp32 tensor -> stacked [2, ...] (hi, lo): hi = t rounded to TF32 (nearest, ties away; low 13 mantissa bits
    cleared), lo = TF32 rounding of t - hi.  Bit-for-bit what lf_pack_gather writes for LF_PACK_TF32_HI / _LO."""
    def rna(v):
        return ((v.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)
    t = t.float()
    hi = rna(t)
    return torch.stack([hi, rna(t - hi)])

ptr = _capi.ptr


def _lib():
    return _capi.lib()


def _stream():
    return _capi.stream_ptr()


def _empty(shape, like, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device=like.device)


# --------------------------------------------------------------------------------------
# weight packing (parameter-sized tensors; reference layouts -> GEMM layouts)
# --------------------------------------------------------------------------------------

def pack_conv_fwd(w, ci_pad=None):
    """Conv2d weight [Co,Ci,kh,kw] -> [kh*kw, CiPad, CoPad] (zero padded)."""
    Co, Ci, kh, kw = w.shape
    ci_pad = ci_pad or Ci
    out = w.new_zeros(kh * kw, ci_pad, plans.cout_pad(Co))
    out[:, :Ci, :Co] = w.permute(2, 3, 1, 0).reshape(kh * kw, Ci, Co)
    return out


def pack_conv_dgrad(w):
    """Conv2d weight [Co,Ci,kh,kw] -> [kh*kw, Co, CiPad]: the transposed GEMM operand."""
    Co, Ci, kh, kw = w.shape
    out = w.new_zeros(kh * kw, Co, plans.cout_pad(Ci))
    out[:, :, :Ci] = w.permute(2, 3, 0, 1).reshape(kh * kw, Co, Ci)
    return out


def pack_convT_fwd(w):
    """ConvTranspose2d weight [Ci,Co,kh,kw] -> [kh*kw, Ci, CoPad]."""
    Ci, Co, kh, kw = w.shape
    out = w.new_zeros(kh * kw, Ci, plans.cout_pad(Co))
    out[:, :, :Co] = w.permute(2, 3, 0, 1).reshape(kh * kw, Ci, Co)
    return out


def pack_convT_dgrad(w):
    """ConvTranspose2d weight [Ci,Co,kh,kw] -> [kh*kw, Co, CiPad]."""
    Ci, Co, kh, kw = w.shape
    out = w.new_zeros(kh * kw, Co, plans.cout_pad(Ci))
    out[:, :, :Ci] = w.permute(2, 3, 1, 0).reshape(kh * kw, Co, Ci)
    return out


# --------------------------------------------------------------------------------------
# Resolution-changing layers on the tensor cores (csrc/conv_tcg.cu, tf32 mode).
# Two horizontally adjacent pixels of an NHWC tensor form a "pair pixel" with 2C channels (a free view);
# even / odd rows are two strided views.  In these coordinates
#   * a 3x3 stride-2 convolution (Down forward; input gradient of the stride-2 transposed conv) is a 6-tap
#     unit-stride gather: kernel row ky reads the odd-row view at i-1 (ky=0), the even-row view at i (ky=1),
#     the odd-row view at i (ky=2); kernel column kx=0 is the second half of pair j-1, kx=1 / kx=2 the two
#     halves of pair j;
#   * a 3x3 stride-2 transposed convolution (Up forward; input gradient of the stride-2 conv) produces, per
#     output-row parity a, the pair pixel (2j, 2j+1) of row 2i+a from inputs (i[+1], j[+1]).
# --------------------------------------------------------------------------------------
TCG_S2CONV_TAPS = [(1, -1, -1), (1, -1, 0), (0, 0, -1), (0, 0, 0), (1, 0, -1), (1, 0, 0)]   # (row view, dy, dx), t = 2*ky + dxi


def pack_tcg_s2conv(w):
    """[O, C, 3, 3] (Conv2d weight, or ConvTranspose2d weight read as [out=Cin_T][in=Cout_T]) ->
    Wg [pad16(O)][6 * 2C], column = t*2C + b*C + c with t = 2*ky + dxi (TCG_S2CONV_TAPS)."""
    O, C = w.shape[0], w.shape[1]
    Og = plans.pad_to(O, 16)
    g = w.new_zeros(Og, 3, 2, 2, C)                 # [o][ky][dxi][b][c]
    g[:O, :, 0, 1] = w[:, :, :, 0].permute(0, 2, 1)  # pair j-1, second half  <- kx = 0
    g[:O, :, 1, 0] = w[:, :, :, 1].permute(0, 2, 1)  # pair j,   first half   <- kx = 1
    g[:O, :, 1, 1] = w[:, :, :, 2].permute(0, 2, 1)  # pair j,   second half  <- kx = 2
    return g.reshape(Og, 6 * 2 * C)


def tcg_s2convT_taps(a):
    """(dy, dx, ky) of the taps feeding output rows of parity a."""
    rows = [(0, 1)] if a == 0 else [(0, 2), (1, 0)]
    return [(dy, dx, ky) for dy, ky in rows for dx in (0, 1)]


def pack_tcg_s2convT(w, a, kc):
    """[I, O, 3, 3] (ConvTranspose2d weight, or Conv2d weight read as [in=Cout][out=Cin]) -> Wg [2*O][ntaps*kc]
    for output-row parity a: row = b*O + o, column = t*kc + i (zero for i >= I)."""
    I, O = w.shape[0], w.shape[1]
    taps = tcg_s2convT_taps(a)
    g = w.new_zeros(2, O, len(taps), kc)            # [b][o][t][i]
    for t, (dy, dx, ky) in enumerate(taps):
        if dx == 0:
            g[0, :, t, :I] = w[:, :, ky, 1].t()     # column 2j   <- kx = 1 from input column j
            g[1, :, t, :I] = w[:, :, ky, 2].t()     # column 2j+1 <- kx = 2 from input column j
        else:
            g[1, :, t, :I] = w[:, :, ky, 0].t()     # column 2j+1 <- kx = 0 from input column j+1
    return g.reshape(2 * O, len(taps) * kc)


def _tcg_view(t, H, W, sn, sy, sx, offset=0):
    v = _capi.LfTcgView()
    v.ptr, v.H, v.W, v.sn, v.sy, v.sx = t.data_ptr() + 4 * offset, H, W, sn, sy, sx
    return v


def tcg_s2conv_ok(x, C, O):
    """stride-2 conv of x[..., :C] (dense [N,H,W,C]) to O channels on lf_conv_tcg?"""
    N, H, W, cx = x.shape
    return (tc_mode() and cx == C and (2 * C) % 32 == 0 and H % 2 == 0 and W % 2 == 0 and x.is_contiguous()
            and int(_lib().lf_conv_tcg_supported(N, H // 2, W // 2, 2 * C, plans.pad_to(O, 16))) > 0)


def run_tcg_s2conv(x, wg, O, out, bias=None, relu=False):
    """out[n,i,j,:O] = bias + conv3x3/s2/p1(x) with wg = pack_tcg_s2conv(w); x dense [N,H,W,C]; out [N,H/2,W/2,Co_total]
    (the first pad16(O) channels are written: the caller overwrites / ignores any padding columns)."""
    N, H, W, C = x.shape
    _, Ho, Wo, cot = out.shape
    a = _capi.LfConvTcgArgs()
    a.a[0] = _tcg_view(x, H // 2, W // 2, H * W * C, 2 * W * C, 2 * C)             # even rows, pair pixels
    a.a[1] = _tcg_view(x, H // 2, W // 2, H * W * C, 2 * W * C, 2 * C, W * C)      # odd rows
    a.wg, a.bias, a.out = wg.data_ptr(), (bias.data_ptr() if bias is not None else None), out.data_ptr()
    a.osn, a.osy, a.osx, a.oy_mul, a.oy0 = Ho * Wo * cot, Wo * cot, cot, 1, 0
    a.N, a.Hs, a.Ws, a.Kc, a.Ng, a.ntaps = N, Ho, Wo, 2 * C, wg.shape[-2], 6
    a.precision = tcg_precision(wg)
    a.relu = int(relu)
    for t, (m, dy, dx) in enumerate(TCG_S2CONV_TAPS):
        a.map[t], a.dy[t], a.dx[t] = m, dy, dx
    _capi.call("lf_conv_tcg", ctypes.byref(a), _stream(), flops=2 * N * Ho * Wo * 9 * C * O, nbytes=4 * N * (H * W * C + Ho * Wo * O))
    return out


def tcg_s2convT_ok(x, I, O):
    """stride-2 transposed conv of x[..., :I] ([N,H,W,cx], cx >= pad32(I)) to O channels on lf_conv_tcg?"""
    N, H, W, cx = x.shape
    kc = plans.pad_to(I, 32)
    return (tc_mode() and cx >= kc and cx % 4 == 0 and (2 * O) % 16 == 0 and 2 * O <= 128 and x.is_contiguous()
            and int(_lib().lf_conv_tcg_supported(N, H, W, kc, 2 * O)) > 0)


def run_tcg_s2convT(x, I, wgs, O, out, bias2=None, relu=False):
    """out [N,2H,2W,O] = bias + convT3x3/s2/p1/op1(x[..., :I]); wgs = (pack_tcg_s2convT(w,0,kc), pack_tcg_s2convT(w,1,kc));
    bias2 = bias tiled twice (pair pixel)."""
    N, H, W, cx = x.shape
    kc = plans.pad_to(I, 32)
    for par in (0, 1):
        taps = tcg_s2convT_taps(par)
        a = _capi.LfConvTcgArgs()
        a.a[0] = _tcg_view(x, H, W, H * W * cx, W * cx, cx)
        a.wg, a.bias, a.out = wgs[par].data_ptr(), (bias2.data_ptr() if bias2 is not None else None), out.data_ptr()
        a.osn, a.osy, a.osx, a.oy_mul, a.oy0 = 4 * H * W * O, 2 * W * O, 2 * O, 2, par
        a.N, a.Hs, a.Ws, a.Kc, a.Ng, a.ntaps = N, H, W, kc, 2 * O, len(taps)
        a.precision = tcg_precision(wgs[par])
        a.relu = int(relu)
        for t, (dy, dx, _ky) in enumerate(taps):
            a.map[t], a.dy[t], a.dx[t] = 0, dy, dx
        _capi.call("lf_conv_tcg", ctypes.byref(a), _stream(), flops=2 * N * H * W * len(taps) * I * 2 * O,
                   nbytes=4 * N * H * W * (I + 2 * O))
    return out


# weight gradients of the same layers (csrc/wgrad_tcg.cu): D[(t, k)][n] over the pair-pixel taps, then one gather
_TCG_WGRAD_IDX = {}


def _tcg_wgrad_index(kind, C, O, Nn, device):
    """Gather indices from the reduced [6*2C][Nn] tap-major result into the reference weight layout.
    kind "conv":  A = layer input (pair view, C channels), B = output gradient -> dW[O][C][3][3]   (row = t*2C + b*C + c, col = o)
    kind "convT": A = output gradient (pair view, C = Cout_T channels), B = layer input -> dW[O=Cin_T][C][3][3] (col = o)"""
    key = (kind, C, O, Nn, str(device))
    if key not in _TCG_WGRAD_IDX:
        idx = torch.empty(O, C, 3, 3, dtype=torch.long)
        o = torch.arange(O).view(O, 1)
        c = torch.arange(C).view(1, C)
        for ky in range(3):
            for kx, (dxi, b) in enumerate(((0, 1), (1, 0), (1, 1))):
                idx[:, :, ky, kx] = ((2 * ky + dxi) * 2 * C + b * C + c) * Nn + o
        _TCG_WGRAD_IDX[key] = idx.reshape(-1).to(device)
    return _TCG_WGRAD_IDX[key]


WGRAD_TCG = os.environ.get("LANEFIT_WGRAD_TCG", "1") != "0"


def wgrad_tcg_ok(a_t, C, b_t, Nn):
    """A = dense [N,2Hs,2Ws,C] tensor (pair view 2C channels), B = [N,Hs,Ws,>=Nn] tensor."""
    N, H2, W2, ca = a_t.shape
    if not (WGRAD_TCG and tc_mode() and ca == C and (2 * C) % 32 == 0 and H2 % 2 == 0 and W2 % 2 == 0 and Nn % 32 == 0 and Nn <= 128
            and b_t.shape[-1] >= Nn and b_t.shape[1] == H2 // 2 and b_t.shape[2] == W2 // 2
            and a_t.is_contiguous() and b_t.is_contiguous()):
        return False
    per_tap = (2 * C) // 32
    taps_per_launch = _wgrad_tcg_taps_per_launch(N, H2 // 2, W2 // 2, C, Nn)
    return taps_per_launch > 0


def _wgrad_tcg_ctas(*args):
    return int((_lib().lf_wgrad_tcg_ctas_bf16 if bf16_mode() else _lib().lf_wgrad_tcg_ctas_x3 if wgrad_x3()
                else _lib().lf_wgrad_tcg_ctas)(*args))


def _wgrad_tcg_taps_per_launch(N, Hs, Ws, C, Nn):
    """6, 3 or 2 taps per launch (block table and shared-memory stages permitting), 0 = unsupported."""
    per_tap = (2 * C) // 32
    for tpl in (6, 3, 2):
        nb = tpl * per_tap
        if ((nb + 3) // 4) * Nn <= 512 and nb <= _capi.WGRAD_TCG_MAX_BLOCKS and _wgrad_tcg_ctas(N, Hs, Ws, 2 * C, Nn, nb) > 0:
            return tpl
    return 0


def run_wgrad_tcg(a_t, C, b_t, Nn):
    """-> reduced [6*2C][Nn] tensor: row (t*2C + k) = sum over pixels of A_t(pixel + tap t)[k] * B(pixel)[:Nn]
    with the six pair-pixel taps of TCG_S2CONV_TAPS."""
    N, H2, W2, _ = a_t.shape
    Hs, Ws = H2 // 2, W2 // 2
    Ka = 2 * C
    per_tap = Ka // 32
    cb_tot = b_t.shape[-1]
    taps_per_launch = _wgrad_tcg_taps_per_launch(N, Hs, Ws, C, Nn)
    res = torch.empty(6 * Ka, Nn, dtype=torch.float32, device=a_t.device)
    st = _stream()
    for t0 in range(0, 6, taps_per_launch):
        nblocks = taps_per_launch * per_tap
        nctas = _wgrad_tcg_ctas(N, Hs, Ws, Ka, Nn, nblocks)
        partial = torch.empty(nctas * nblocks * 32 * Nn, dtype=torch.float32, device=a_t.device)
        a = _capi.LfWgradTcgArgs()
        a.a[0] = _tcg_view(a_t, Hs, Ws, H2 * W2 * C, 2 * W2 * C, 2 * C)
        a.a[1] = _tcg_view(a_t, Hs, Ws, H2 * W2 * C, 2 * W2 * C, 2 * C, W2 * C)
        a.b = _tcg_view(b_t, Hs, Ws, Hs * Ws * cb_tot, Ws * cb_tot, cb_tot)
        a.partial, a.N, a.Hs, a.Ws, a.Ka, a.Nn, a.nblocks, a.nctas = partial.data_ptr(), N, Hs, Ws, Ka, Nn, nblocks, nctas
        a.precision = wgrad_precision()
        for i in range(nblocks):
            m, dy, dx = TCG_S2CONV_TAPS[t0 + i // per_tap]
            a.map[i], a.dy[i], a.dx[i], a.cblk[i] = m, dy, dx, i % per_tap
        _capi.call("lf_wgrad_tcg", ctypes.byref(a), st, flops=2 * N * Hs * Ws * nblocks * 32 * Nn,
                   nbytes=4 * N * Hs * Ws * (nblocks * 32 + Nn))
        _capi.call("lf_wgrad_reduce", ptr(partial), nctas, 1, nblocks * 32, Nn, nblocks * 32, Nn,
                   res.data_ptr() + 4 * t0 * Ka * Nn, 0, Nn, 1, st)
    return res


def wgrad_tcg_conv(x, cin, dcat, cc):
    """dW [cc, cin, 3, 3] of the stride-2 Conv2d (DownsamplerBlock): A = x, B = dcat[..., :pad32(cc)]."""
    Nn = plans.pad_to(cc, 32)
    res = run_wgrad_tcg(x, cin, dcat, Nn)
    return res.reshape(-1)[_tcg_wgrad_index("conv", cin, cc, Nn, x.device)].view(cc, cin, 3, 3)


def wgrad_tcg_convT(x, ci, du, co):
    """dW [ci, co, 3, 3] of the stride-2 ConvTranspose2d (UpsamplerBlock): A = du (output gradient), B = x."""
    res = run_wgrad_tcg(du, co, x, ci)
    return res.reshape(-1)[_tcg_wgrad_index("convT", co, ci, ci, x.device)].view(ci, co, 3, 3)


# --------------------------------------------------------------------------------------
# one-launch weight packing
# --------------------------------------------------------------------------------------
def pack_gather_table(fn, shape):
    """int32 gather indices t with fn(w).flatten()[k] == (w.flatten()[t[k]] if t[k] >= 0 else 0), shaped like
    fn(w): obtained by running the packer on 1-based element numbers (0 = structural zero)."""
    n = 1
    for d in shape:
        n *= int(d)
    numbered = torch.arange(1, n + 1, dtype=torch.float64).view(tuple(shape))
    return (fn(numbered).to(torch.int64) - 1).to(torch.int32).contiguous()


class WeightPackCache:
    """All GEMM-layout weight operands of a model, refreshed by ONE kernel per step (lf_pack_gather).

    Every packer above is pure data movement, so its gather table is obtained by running the packer on an
    index tensor once.  ``refresh()`` (called at the top of ERFNet.forward) re-packs every registered
    operand from the current parameter values; ``get()`` hands the packed tensor to conv3()/wgrad3()/... if it
    is current (same parameter object still at that address, same in-place version as at the last refresh),
    else returns None and the caller packs directly (first use, eval of a foreign tensor, ...).
    Operands are registered lazily on their first miss and served from the next refresh on."""

    BLOCKS_PER_JOB = 12

    def __init__(self, module):
        self.module = module
        self.by_ptr = {}
        self.entries = {}        # (data_ptr, kind) -> [param, idx(int32 dev), out(dev), version_at_refresh]
        self.jobs = None
        self.dirty = False

    def _scan(self):
        # `_pack_extra`: further modules whose conv weights are served by this cache (the Classification heads, which
        # hang off LSQ_layer.Net next to the ERFNet module that owns the cache)
        mods = [self.module] + list(self.module.__dict__.get("_pack_extra", ()))
        self.by_ptr = {p.data_ptr(): p for m in mods for p in m.parameters() if p.is_cuda}

    def get(self, w, kind, fn, split=False):
        """split: False (fp32 operand), True (TF32 hi/lo pair) or "bf16" -- part of the key, so a mode switch never
        serves an operand of another form."""
        if not w.is_cuda:
            return None
        p = self.by_ptr.get(w.data_ptr())
        if p is None or p.shape != w.shape:
            return None
        key = (w.data_ptr(), kind, split)
        e = self.entries.get(key)
        if e is None:
            if torch.cuda.is_current_stream_capturing():
                return None
            idx = pack_gather_table(fn, p.shape)
            if split is True:       # [2, ...]: TF32 hi parts, then lo parts (structural zeros stay negative)
                assert p.numel() <= _capi.PACK_INDEX_MASK
                idx = torch.stack([torch.where(idx >= 0, idx | _capi.PACK_TF32_HI, idx),
                                   torch.where(idx >= 0, idx | _capi.PACK_TF32_LO, idx)])
            dtype = torch.bfloat16 if split == "bf16" else torch.float32
            self.entries[key] = [p, idx.to(w.device), torch.empty(idx.shape, dtype=dtype, device=w.device), -1]
            self.dirty = True
            return None
        if e[3] != p._version or e[0] is not p:
            return None
        return e[2]

    def refresh(self):
        self._scan()
        dead = [k for k, e in self.entries.items() if self.by_ptr.get(k[0]) is not e[0]]
        for k in dead:
            del self.entries[k]
            self.dirty = True
        if not self.entries:
            return
        if self.dirty:
            if torch.cuda.is_current_stream_capturing():
                return                      # keep serving the operands that are already in the table
            # LfPackJob rows: src, dst, idx, n, dst_dtype (the int64 holds the dtype and the zero pad field)
            rows = [[e[0].data_ptr(), e[2].data_ptr(), e[1].data_ptr(), e[1].numel(), _capi.dtype_id(e[2])]
                    for e in self.entries.values()]
            dev = next(iter(self.entries.values()))[2].device
            self.jobs = torch.tensor(rows, dtype=torch.int64).to(dev)
            self.job_entries = list(self.entries.values())
            self.dirty = False
        _capi.call("lf_pack_gather", ptr(self.jobs), len(self.job_entries), self.BLOCKS_PER_JOB, _stream())
        for e in self.job_entries:
            e[3] = e[0]._version


ACTIVE_PACKS = None


def packed(w, kind, fn, split=False):
    """The packed operand ``fn(w)`` (``split``: True = its TF32 hi/lo pair, see split_tf32; "bf16" = rounded to bf16):
    from the active WeightPackCache when current, else computed now."""
    c = ACTIVE_PACKS
    if c is not None:
        t = c.get(w, kind, fn, split)
        if t is not None:
            return t
    if split == "bf16":
        return fn(w).to(torch.bfloat16)
    return split_tf32(fn(w)) if split else fn(w)


# --------------------------------------------------------------------------------------
# launch helpers
# --------------------------------------------------------------------------------------

def run_conv(phases, x, wmat, cin, out, cout, out_coff=0, bias=None, relu=False, mask_src=None, add_src=None,
             add_mask=None):
    """x: [N,Hin,Win,Cx] NHWC (Cx = channel stride), out: [N,Hout,Wout,Co_total]."""
    h = _lib()
    N, Hin, Win, cx = x.shape
    _, Hout, Wout, cot = out.shape
    a = LfConvArgs()
    a.inp, a.wmat, a.bias, a.out = x.data_ptr(), wmat.data_ptr(), (bias.data_ptr() if bias is not None else None), \
        out.data_ptr()
    a.mask_src = mask_src.data_ptr() if mask_src is not None else None
    a.add_src = add_src.data_ptr() if add_src is not None else None
    a.add_mask = add_mask.data_ptr() if add_mask is not None else None
    a.N, a.Hin, a.Win, a.Cin, a.in_cstride = N, Hin, Win, cin, cx
    a.Hout, a.Wout, a.out_cstride, a.out_coff, a.Cout, a.CoutPad = Hout, Wout, cot, out_coff, cout, wmat.shape[2]
    a.relu = int(relu)
    assert wmat.shape[1] == cin, (wmat.shape, cin)
    st = _stream()
    for ph in phases:
        a.Hs, a.Ws, a.osy, a.osx, a.oy0, a.ox0, a.isy, a.isx = (ph["Hs"], ph["Ws"], ph["osy"], ph["osx"], ph["oy0"],
                                                               ph["ox0"], ph["isy"], ph["isx"])
        taps = ph["taps"]
        a.ntaps = len(taps)
        for t, (dy, dx, slot) in enumerate(taps):
            a.dy[t], a.dx[t], a.wtap[t] = dy, dx, slot
        _capi.call("lf_conv_f32", ctypes.byref(a), st,
                   flops=2 * N * ph["Hs"] * ph["Ws"] * len(taps) * cin * cout,
                   nbytes=4 * N * ph["Hs"] * ph["Ws"] * (cin + cout))
    return out


def pack_tc_fwd(w):
    """Conv2d weight [Co,Ci,kh,kw] (3 taps) -> [Co][3*Ci], K = (tap, ci) contiguous."""
    Co, Ci, kh, kw = w.shape
    return w.permute(0, 2, 3, 1).reshape(Co, kh * kw * Ci).contiguous()


def pack_tc_dgrad(w):
    """-> [Ci][3*Co]: the GEMM operand of the input gradient (taps negated by the caller)."""
    Co, Ci, kh, kw = w.shape
    return w.permute(1, 2, 3, 0).reshape(Ci, kh * kw * Co).contiguous()


# ----------------------------------------------------------------------------------------
# C = 16 layers on the tensor-core kernels: "super-pixel" packing.
# A [N,H,W,16] tensor IS a [N,H,W/4,64] tensor in memory (4 neighbouring x positions x 16 channels = 64
# super-channels).  A 3-tap convolution of the original is a 3-tap convolution of the super-pixel grid
# with 64x64 weight blocks built from the 16x16 ones: block-diagonal for the vertical (3x1) conv, banded
# for the horizontal (1x3) conv whose x-1 / x+1 taps cross into the neighbouring super-pixel.  3/4 of the
# MMA work multiplies zeros, but the tensor-core kernels are faster than the CUDA-core kernels on these
# bandwidth-bound layers and nothing new runs on the device.
# ----------------------------------------------------------------------------------------
SUPER = 4


def _super_map(vertical, transposed):
    """[(T, s_in, s_out, t)] : super tap T / sub-positions for every original tap t and output sub-position."""
    out = []
    for s in range(SUPER):
        for t in range(3):
            off = (t - 1) * (-1 if transposed else 1)      # input offset of weight slot t along the conv axis
            if vertical:
                out.append((t, s, s, t))                   # rows are not packed: same tap, same sub-position
            else:
                xs = s + off
                T_in = xs // SUPER                          # -1, 0, +1 super-pixel offset
                out.append((((-T_in if transposed else T_in) + 1), xs % SUPER, s, t))
    return out


_SUPER_IDX = {}


def _super_indices(c, vertical, transposed, device):
    """Cached gather indices (one device op per packing instead of 12 slice updates)."""
    key = (c, vertical, transposed, str(device))
    if key not in _SUPER_IDX:
        nsrc = c * c * 3                                     # blk[out][in][t] flattened; slot nsrc = 0.0
        pack = torch.full((SUPER * c, 3 * SUPER * c), nsrc, dtype=torch.long)
        unpack = torch.full((c, c, 3, SUPER), SUPER * c * SUPER * c * 3, dtype=torch.long)
        o = torch.arange(c).view(c, 1)
        i = torch.arange(c).view(1, c)
        for T, s_in, s_out, t in _super_map(vertical, transposed):
            pack[s_out * c:(s_out + 1) * c, T * SUPER * c + s_in * c:T * SUPER * c + (s_in + 1) * c] = (o * c + i) * 3 + t
        for T, s_in, s_out, t in _super_map(vertical, False):
            # dws[co_s][ci_s][T] flattened, co_s = s_out*c + co, ci_s = s_in*c + ci
            unpack[:, :, t, s_out] = ((s_out * c + o) * (SUPER * c) + (s_in * c + i)) * 3 + T
        # unpack without a zero slot: clamp the missing sources to element 0 and weight them with 0
        missing = unpack == SUPER * c * SUPER * c * 3
        unpack_w = (~missing).to(torch.float32)
        unpack_c = torch.where(missing, torch.zeros_like(unpack), unpack)
        _SUPER_IDX[key] = (pack.to(device), unpack.to(device), unpack_c.to(device), unpack_w.to(device))
    return _SUPER_IDX[key]


def pack_tc_super(w, vertical, transposed):
    """3-tap 16->16 weight [16,16,kh,kw] -> packed [64][3*64] operand of lf_conv1d_tc on the super-pixel
    grid (layout of pack_tc_fwd / pack_tc_dgrad: row = output super-channel, column = T*64 + input
    super-channel).  Weight slot T of the packed operand reads the super-pixel at (T-1) (forward) or
    -(T-1) (transposed), matching the tap lists conv3() builds."""
    c = w.shape[0]
    w3 = w.reshape(c, c, 3)                                  # [co][ci][t]
    blk = w3.permute(1, 0, 2) if transposed else w3          # [out][in][t] of the convolution actually run
    pack = _super_indices(c, vertical, transposed, w.device)[0]
    src = torch.cat([blk.reshape(-1), blk.new_zeros(1)])
    return src[pack]


def unpack_wgrad_super(dw_super, vertical):
    """dw_super [64(co_s),64(ci_s),3] (weight-gradient of the super-pixel conv in Conv2d layout) ->
    dw [16,16,3]: sum of the (up to 4) blocks each original weight occupies in the packed operand."""
    c = dw_super.shape[0] // SUPER
    _, _, idx, wgt = _super_indices(c, vertical, False, dw_super.device)
    return (dw_super.reshape(-1)[idx] * wgt).sum(-1)         # 3 launches (was 5 with a concatenated zero slot)


def super_ok(x, dil):
    N, H, W, C = x.shape
    if not (tc_mode() and C == 16 and dil == 1 and W % SUPER == 0 and x.is_contiguous()):
        return False
    if x3_mode():
        return min(int(_lib().lf_conv1d_tc_x3_rows(N, H, W // SUPER, SUPER * C, v, 1)) for v in (0, 1)) > 0
    return int(_lib().lf_conv1d_tc_supported(N, H, W // SUPER, SUPER * C)) > 0


def tc_rows(x, vertical=None, dil=1, stats=False):
    """0 if the active tensor-core kernel does not take this call, else the row count of its colsum / stats partials.
    tf32: any 3-tap pattern on a supported shape (the per-tap variant is the in-library fallback; `stats` needs the
    slab kernel); tf32x3: per (axis, dilation) -- vertical=None asks for d=1 along both axes."""
    N, H, W, C = x.shape
    if C not in (64, 128) or not tc_mode():
        return 0
    if x3_mode():
        if vertical is None:
            return min(int(_lib().lf_conv1d_tc_x3_rows(N, H, W, C, v, dil)) for v in (0, 1))
        return int(_lib().lf_conv1d_tc_x3_rows(N, H, W, C, int(vertical), dil))
    rows = int(_lib().lf_conv1d_tc_supported(N, H, W, C))
    if rows and stats and not _lib().lf_conv1d_tc_slab_ok(N, H, W, C, int(bool(vertical)), dil):
        return 0
    return rows


def tc_supported(x, vertical=None, dil=1):
    return tc_rows(x, vertical, dil) > 0


def _taps_axis(taps):
    """(vertical, dilation) of a 3-tap list [(dy, dx)] * 3."""
    vertical = taps[0][0] != 0 or taps[2][0] != 0
    d = abs(taps[0][0] if vertical else taps[0][1])
    return vertical, d


def run_conv_tc(taps, x, wpack, out, bias=None, relu=False, mask_src=None, add_src=None, add_mask=None, colsum=None,
                mask_affine=None, stats_partial=None, fp8=None):
    """3-tap convolution on tensor cores.  taps: [(dy, dx)] * 3 in weight-slot order.  colsum: optional [C]
    tensor receiving the column sums of `out` (bias gradient), accumulated in the kernel's epilogue.
    fp8: (x_amax [N], w_scale [C], out_amax [N]) with an e4m3 `wpack` (uint8 storage): lf_conv1d_tc_fp8, the fp8 mode's
    only 3-tap route; out_amax receives max |out| per image and must be zeroed by the caller."""
    N, H, W, C = x.shape
    a = LfConvTcArgs()
    a.inp, a.wpack, a.out = x.data_ptr(), wpack.data_ptr(), out.data_ptr()
    a.bias = bias.data_ptr() if bias is not None else None
    a.mask_src = mask_src.data_ptr() if mask_src is not None else None
    a.add_src = add_src.data_ptr() if add_src is not None else None
    a.add_mask = add_mask.data_ptr() if add_mask is not None else None
    part = None
    if colsum is not None:
        rows = tc_rows(x, *_taps_axis(taps))
        part = torch.empty(rows * C, dtype=torch.float32, device=x.device)
        a.colsum_partial = part.data_ptr()
    if stats_partial is not None:
        a.stats_partial = stats_partial.data_ptr()
    if mask_affine is not None:        # (scale, shift): mask_src is a BatchNorm INPUT, the mask bit is fma(x, scale, shift) > 0
        a.mask_scale, a.mask_shift = mask_affine[0].data_ptr(), mask_affine[1].data_ptr()
    a.N, a.H, a.W, a.C = N, H, W, C
    for t, (dy, dx) in enumerate(taps):
        a.dy[t], a.dx[t] = dy, dx
    a.relu = int(relu)
    a.in_dtype, a.out_dtype = _capi.dtype_id(x), _capi.dtype_id(out)
    a.mask_dtype = _capi.dtype_id(mask_src) if mask_src is not None else _capi.LF_F32
    width = sum(t.element_size() for t in (x, out, mask_src, add_src, add_mask) if t is not None)
    if fp8 is not None:
        f = _capi.LfConvTcFp8Args()
        f.conv = a
        f.x_amax, f.w_scale, f.out_amax = (t.data_ptr() for t in fp8)
        entry, arg = "lf_conv1d_tc_fp8", f
    elif fp8_mode():
        raise _capi.LanefitError("run_conv_tc: the fp8 mode runs 3-tap convolutions only with fp8 operands (ops_eval)")
    else:
        entry, arg = "lf_conv1d_tc_x3" if x3_mode() else "lf_conv1d_tc_bf16" if bf16_mode() else "lf_conv1d_tc", a
    _capi.call(entry, ctypes.byref(arg), _stream(), flops=2 * N * H * W * 3 * C * C, nbytes=width * N * H * W * C)
    if part is not None:
        if _DEFERRED is not None:
            _reduce(part, rows, 1, 1, C, 1, C, colsum, 0, 0, 1)
        else:
            _capi.call("lf_vec_reduce", ptr(part), rows, C, C, ptr(colsum), _stream())
    return out


# Deferred split reductions: inside Nb1dFunction.backward the weight / bias gradient reductions of the block are
# collected here and run by ONE lf_reduce_multi launch at the end (instead of six ~12 us launches).
_DEFERRED = None


def _reduce(partial, nsplit, ntaps, cp, cq, cp_pad, cq_pad, dst, st, sp, sq):
    if _DEFERRED is not None:
        _DEFERRED.append((partial, nsplit, ntaps, cp, cq, cp_pad, cq_pad, dst, st, sp, sq))
        return
    _capi.call("lf_wgrad_reduce", ptr(partial), nsplit, ntaps, cp, cq, cp_pad, cq_pad, ptr(dst), st, sp, sq, _stream())


def flush_deferred_reductions(jobs):
    for k in range(0, len(jobs), _capi.REDUCE_MAX_JOBS):
        chunk = jobs[k:k + _capi.REDUCE_MAX_JOBS]
        arr = (_capi.LfReduceJob * len(chunk))()
        for j, (partial, nsplit, ntaps, cp, cq, cp_pad, cq_pad, dst, st, sp, sq) in zip(arr, chunk):
            j.partial, j.dst = partial.data_ptr(), dst.data_ptr()
            j.nsplit, j.ntaps, j.Cp, j.Cq, j.CpPad, j.CqPad, j.st, j.sp, j.sq = nsplit, ntaps, cp, cq, cp_pad, cq_pad, st, sp, sq
        _capi.call("lf_reduce_multi", arr, len(chunk), _stream())


def _super_conv_launch(taps, xs, w, vertical, transposed, out, N, H, W, C, cs, epi_s, wp=None):
    if wp is None:
        wp = packed(w, "tc_super_%d%d" % (vertical, transposed), lambda t: pack_tc_super(t, vertical, transposed), split=pack_split())
    run_conv_tc(taps, xs, wp, out.view(N, H, W // SUPER, SUPER * C), colsum=cs, **epi_s)


def conv3(x, w, vertical, dil, transposed, colsum=None, wp=None, dtype=torch.float32, **epi):
    """One factorised 3-tap convolution of non_bottleneck_1d (or its input gradient when
    ``transposed``): dispatches to the tensor-core kernel in tf32 mode, else to the fp32 kernel.
    ``colsum`` ([C] tensor): also produce the per-channel sums of the result.
    ``wp``: the already packed tensor-core operand (ops_eval's BatchNorm-folded weights) -- tensor-core routes only.
    ``dtype``: of the result; bf16 (like a bf16 ``x`` or ``mask_src``) only on the bf16 tensor-core routes."""
    N, H, W, C = x.shape
    out = torch.empty(x.shape, dtype=dtype, device=x.device)
    if super_ok(x, dil):
        xs = x.view(N, H, W // SUPER, SUPER * C)
        sgn = -1 if transposed else 1
        taps = [((sgn * (k - 1), 0) if vertical else (0, sgn * (k - 1))) for k in range(3)]
        epi_s = {k: (v.view(N, H, W // SUPER, SUPER * C) if (torch.is_tensor(v) and v.dim() == 4) else v) for k, v in epi.items()}
        if epi_s.get("bias") is not None:
            epi_s["bias"] = epi_s["bias"].repeat(SUPER)
        cs = torch.empty(SUPER * C, dtype=torch.float32, device=x.device) if colsum is not None else None
        global _DEFERRED
        saved, _DEFERRED = _DEFERRED, None     # the column sums are post-processed right below: reduce them now
        try:
            _super_conv_launch(taps, xs, w, vertical, transposed, out, N, H, W, C, cs, epi_s, wp=wp)
        finally:
            _DEFERRED = saved
        if colsum is not None:
            colsum.copy_(cs.view(SUPER, C).sum(0))
        return out
    if tc_supported(x, vertical, dil):
        sgn = -1 if transposed else 1
        taps = [((sgn * (k - 1) * dil, 0) if vertical else (0, sgn * (k - 1) * dil)) for k in range(3)]
        if wp is None:
            wp = (packed(w, "tc_dgrad", pack_tc_dgrad, split=pack_split()) if transposed
                  else packed(w, "tc_fwd", pack_tc_fwd, split=pack_split()))
        return run_conv_tc(taps, x, wp, out, colsum=colsum, **epi)
    if wp is not None:
        raise _capi.LanefitError("conv3: a pre-packed operand needs a tensor-core route")
    if any(t.dtype != torch.float32 for t in [x, out] + [v for v in epi.values() if torch.is_tensor(v)]):
        raise _capi.LanefitError("conv3: bf16 operands need a bf16 tensor-core route")
    kh, kw = (3, 1) if vertical else (1, 3)
    ph, pw = (dil, 0) if vertical else (0, dil)
    dh, dw = (dil, 1) if vertical else (1, dil)
    if transposed:
        phases, _ = plans.conv_dgrad_plan_s1(H, W, kh, kw, ph, pw, dh, dw)
        run_conv(phases, x, packed(w, "conv_dgrad", pack_conv_dgrad), C, out, C, **epi)
    else:
        phases, _ = plans.conv_fwd_plan(H, W, kh, kw, 1, ph, pw, dh, dw)
        run_conv(phases, x, packed(w, "conv_fwd", pack_conv_fwd), C, out, C, **epi)
    if colsum is not None:
        run_colsum(out, C, 0, colsum)
    return out


def wgrad3(x_in, d_out, w, vertical, dil, bias_grad="compute"):
    """Weight + bias gradient of one factorised 3-tap convolution -> (dw [Co,Ci,kh,kw], db [Co] or None).
    bias_grad: "compute" (column sums of d_out), or "skip" (the caller gets it elsewhere)."""
    N, H, W, C = x_in.shape
    sfx = "_x3" if wgrad_x3() else "_bf16" if bf16_mode() else ""   # which tensor-core weight-gradient kernel
    xbf = x_in.dtype == torch.bfloat16                               # a bf16 layer input: the bf16-A kernel
    if xbf and not bf16_mode():
        raise _capi.LanefitError("wgrad3: a bf16 layer input needs the bf16 mode")
    entry = "lf_wgrad3_tc" + sfx + ("a" if xbf else "")
    nbytes = (x_in.element_size() + 4) * N * H * W * C
    if super_ok(x_in, dil) and d_out.is_contiguous():
        Cs, Ws = SUPER * C, W // SUPER
        nctas = getattr(_lib(), "lf_wgrad3_tc%s_ctas" % sfx)(N, H, Ws, Cs)
        if nctas > 0:
            tdy = (ctypes.c_int * 3)(*[((k - 1) if vertical else 0) for k in range(3)])
            tdx = (ctypes.c_int * 3)(*[(0 if vertical else (k - 1)) for k in range(3)])
            partial = torch.empty(nctas * 3 * Cs * Cs, dtype=torch.float32, device=x_in.device)
            dws = torch.empty(Cs, Cs, 3, dtype=torch.float32, device=x_in.device)
            st = _stream()
            _capi.call(entry, ptr(x_in), ptr(d_out), N, H, Ws, Cs, tdy, tdx, ptr(partial), nctas, st,
                       flops=2 * N * H * W * 3 * C * C, nbytes=nbytes)
            _capi.call("lf_wgrad_reduce", ptr(partial), nctas, 3, Cs, Cs, Cs, Cs, ptr(dws), 1, 3, Cs * 3, st)
            dw = unpack_wgrad_super(dws, vertical).reshape(w.shape)
            db = None
            if bias_grad == "compute":
                db = torch.empty(C, dtype=torch.float32, device=x_in.device)
                run_colsum(d_out, C, 0, db)
            return dw, db
    dw = torch.empty_like(w)
    db = torch.empty(C, dtype=torch.float32, device=x_in.device) if bias_grad == "compute" else None
    lay = (1, 3, C * 3)                                   # (tap, ci, co) strides of [Co,Ci,3] weights
    nctas = getattr(_lib(), "lf_wgrad3_tc%s_ctas" % sfx)(N, H, W, C) if (tc_mode() and C in (64, 128)) else 0
    if nctas > 0:
        tdy = (ctypes.c_int * 3)(*[((k - 1) * dil if vertical else 0) for k in range(3)])
        tdx = (ctypes.c_int * 3)(*[(0 if vertical else (k - 1) * dil) for k in range(3)])
        partial = torch.empty(nctas * 3 * C * C, dtype=torch.float32, device=x_in.device)
        st = _stream()
        _capi.call(entry, ptr(x_in), ptr(d_out), N, H, W, C, tdy, tdx, ptr(partial), nctas, st,
                   flops=2 * N * H * W * 3 * C * C, nbytes=nbytes)
        _reduce(partial, nctas, 3, C, C, C, C, dw, lay[0], lay[1], lay[2])
        if db is not None:
            run_colsum(d_out, C, 0, db)
        return dw, db
    if xbf:
        raise _capi.LanefitError("wgrad3: a bf16 layer input needs a tensor-core route")
    kh, kw = (3, 1) if vertical else (1, 3)
    ph, pw = (dil, 0) if vertical else (0, dil)
    dh, dw_ = (dil, 1) if vertical else (1, dil)
    run_wgrad(plans.conv_wgrad_plan(H, W, kh, kw, 1, ph, pw, dh, dw_), x_in, C, d_out, C, 0, N, dw, lay, db)
    return dw, db


def _sm_count():
    import torch
    if not torch.cuda.is_available():
        return 132      # host-side planning without a device (nothing is launched)
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _nsplit_for(tiles, M):
    target = _sm_count() * 6
    ns = max(1, min((target + tiles - 1) // tiles, max(1, M // 256)))
    return int(ns)


def run_wgrad(plan, P, cp, Q, cq, q_coff, N, dst_w, layout, dst_b=None, cp_true=None, cq_true=None):
    """Weight (and optionally bias) gradient.  layout: (st, sp, sq) strides of dst_w for
    (tap, cp, cq).  cp/cq: channel counts handed to the GEMM (multiples of 4); *_true: the
    counts actually written (<= cp/cq)."""
    h = _lib()
    _, Hp, Wp, cps = P.shape
    _, Hq, Wq, cqs = Q.shape
    ntaps = len(plan["ptaps"])
    a = LfWgradArgs()
    a.P, a.Q = P.data_ptr(), Q.data_ptr()
    a.N, a.Hs, a.Ws = N, plan["Hs"], plan["Ws"]
    a.Hp, a.Wp, a.Cp, a.p_cstride, a.p_coff, a.psy, a.psx = Hp, Wp, cp, cps, 0, plan["psy"], plan["psx"]
    a.Hq, a.Wq, a.Cq, a.q_cstride, a.q_coff, a.qsy, a.qsx = Hq, Wq, cq, cqs, q_coff, plan["qsy"], plan["qsx"]
    a.ntaps = ntaps
    for t in range(ntaps):
        a.pdy[t], a.pdx[t] = plan["ptaps"][t]
        a.qdy[t], a.qdx[t] = plan["qtaps"][t]
    a.CpPad, a.CqPad = plans.pad_to(cp, 64), plans.pad_to(cq, 64)
    tiles = (a.CpPad // 64) * (a.CqPad // 64) * ntaps
    M = N * plan["Hs"] * plan["Ws"]
    a.nsplit = _nsplit_for(tiles, M)
    a.qsum_partial = 1 if dst_b is not None else None      # the query only looks at whether it is requested
    pref = int(h.lf_wgrad_f32_nsplit(ctypes.byref(a)))
    if pref > 0:
        a.nsplit = pref
    a.qsum_partial = None
    partial = torch.empty(a.nsplit * ntaps * a.CpPad * a.CqPad, dtype=torch.float32, device=P.device)
    a.partial = partial.data_ptr()
    qpart = None
    if dst_b is not None:
        qpart = torch.empty(a.nsplit * a.CqPad, dtype=torch.float32, device=P.device)
        a.qsum_partial = qpart.data_ptr()
    st = _stream()
    _capi.call("lf_wgrad_f32", ctypes.byref(a), st, flops=2 * M * ntaps * cp * cq, nbytes=4 * M * (cp + cq))
    s_t, s_p, s_q = layout
    _capi.call("lf_wgrad_reduce", ptr(partial), a.nsplit, ntaps, cp_true or cp, cq_true or cq, a.CpPad, a.CqPad,
                                  ptr(dst_w), s_t, s_p, s_q, st)
    if dst_b is not None:
        _capi.call("lf_vec_reduce", ptr(qpart), a.nsplit, cq_true or cq, a.CqPad, ptr(dst_b), st)


def run_colsum(src, C, coff, dst):
    """dst[c] = sum over all pixels of src[..., coff + c]   (src NHWC)."""
    h = _lib()
    npix = src.numel() // src.shape[-1]
    nblk = h.lf_colsum_blocks(npix)
    cpad = plans.pad_to(C, 4)
    part = torch.empty(nblk * cpad, dtype=torch.float32, device=src.device)
    st = _stream()
    _capi.call("lf_colsum", ptr(src), npix, C, src.shape[-1], coff, ptr(part), cpad, st)
    _capi.call("lf_vec_reduce", ptr(part), nblk, C, cpad, ptr(dst), st)


class BNState:
    """Per-call BatchNorm2d state: batch (mean, invstd) for backward, (scale, shift) for apply; with a BNSync also
    ``count``, the global pixel count (fp64 [1] on the device) the backward divides by."""
    __slots__ = ("mean", "invstd", "scale", "shift", "count")


class BNSync:
    """Training-mode BatchNorm synchronised over the ranks of ``group`` (an ``nn.SyncBatchNorm``'s ``process_group``; None =
    the default group): every rank's partial sums are collapsed into a totals buffer (lf_bn_collapse), SUM all-reduced
    (ddp.allreduce_totals) and finalized from the totals (lf_bn_*finalize*_tot).  Without a process group or with one rank
    the same launches run without the collective and give the bits of the plain path."""
    __slots__ = ("group",)

    def __init__(self, group=None):
        self.group = group

    def allreduce(self, totals):
        from .ddp import allreduce_totals
        allreduce_totals(totals, self.group)


def bn_sync(bn, training):
    """The synchronisation of a BatchNorm container: BNSync(bn.process_group) for an nn.SyncBatchNorm in training mode
    (what torch.nn.SyncBatchNorm.convert_sync_batchnorm makes), else None (per-process statistics)."""
    return BNSync(bn.process_group) if training and isinstance(bn, torch.nn.SyncBatchNorm) else None


def _bn_state(C, device):
    s = BNState()
    buf = torch.empty(4, C, dtype=torch.float32, device=device)
    s.mean, s.invstd, s.scale, s.shift = buf[0], buf[1], buf[2], buf[3]
    s.count = None
    return s


def _bn_collapse(part, nblk, npix, C, sync, keep_local=False):
    """SyncBatchNorm: partials [nblk][2][C] -> all-reduced totals [2C+1] (sums, count); keep_local: also this rank's totals
    (returned second, before the all-reduce).  The backward reduces only the 2C sums: its count is the forward's."""
    tot = torch.empty(2 if keep_local else 1, 2 * C + 1, dtype=torch.float64, device=part.device)
    _capi.call("lf_bn_collapse", ptr(part), nblk, C, 1, npix, ptr(tot[0]), ptr(tot[1]) if keep_local else None, _stream())
    sync.allreduce(tot[0, :2 * C] if keep_local else tot[0])
    return (tot[0], tot[1]) if keep_local else tot[0]


def bn_finalize(part, nblk, npix, C, gamma, beta, running_mean, running_var, eps=BN_EPS, sync=None):
    """part: float64 [nblk][2][C] partial sums / sums of squares -> BNState (+ running-stat update); sync: a BNSync for the
    statistics of every rank, else this process's."""
    s = _bn_state(C, part.device)
    if sync is not None:
        tot = _bn_collapse(part, nblk, npix, C, sync)
        _capi.call("lf_bn_finalize_tot", ptr(tot), C, ptr(gamma), ptr(beta), eps, BN_MOMENTUM, ptr(running_mean),
                   ptr(running_var), ptr(s.mean), ptr(s.invstd), ptr(s.scale), ptr(s.shift), _stream())
        s.count = tot[2 * C:]
        return s
    _capi.call("lf_bn_finalize", ptr(part), nblk, npix, C, ptr(gamma), ptr(beta), eps, BN_MOMENTUM,
               ptr(running_mean), ptr(running_var), ptr(s.mean), ptr(s.invstd), ptr(s.scale), ptr(s.shift), _stream())
    return s


def bn_forward_stats(x, gamma, beta, running_mean, running_var, training, eps=BN_EPS, sync=None):
    """x: dense NHWC.  Returns BNState; updates running stats in training mode
    (nn.BatchNorm2d(eps=1e-3, momentum=0.1), ERFNet.py:17,33,39,102).  sync: BNSync (training mode only)."""
    h = _lib()
    C = x.shape[-1]
    npix = x.numel() // C
    if training:
        nblk = h.lf_bn_blocks(npix, C)
        part = torch.empty(nblk * 2 * C, dtype=torch.float64, device=x.device)
        _capi.call("lf_bn_stats", ptr(x), npix, C, ptr(part), _stream(), nbytes=4 * npix * C)
        return bn_finalize(part, nblk, npix, C, gamma, beta, running_mean, running_var, eps, sync)
    s = _bn_state(C, x.device)
    _capi.call("lf_bn_eval_prepare", C, ptr(gamma), ptr(beta), eps, ptr(running_mean), ptr(running_var),
               ptr(s.scale), ptr(s.shift), _stream())
    return s


def conv3_bn_stats(x, w, vertical, dil, bias, gamma, beta, running_mean, running_var, training, sync=None):
    """conv (forward) followed by the BatchNorm statistics of its output -> (out, BNState).  On the tensor-core slab
    kernel the per-channel sums are accumulated in the conv epilogue, saving a full pass over `out`."""
    N, H, W, C = x.shape
    rows = tc_rows(x, vertical, dil, stats=True) if training else 0
    if rows > 0:
        part = torch.empty(rows * 2 * C, dtype=torch.float64, device=x.device)
        taps = [(((k - 1) * dil, 0) if vertical else (0, (k - 1) * dil)) for k in range(3)]
        out = run_conv_tc(taps, x, packed(w, "tc_fwd", pack_tc_fwd, split=pack_split()),
                          torch.empty(x.shape, dtype=torch.float32, device=x.device), bias=bias, stats_partial=part)
        return out, bn_finalize(part, rows, N * H * W, C, gamma, beta, running_mean, running_var, sync=sync)
    out = conv3(x, w, vertical, dil, False, bias=bias)
    return out, bn_forward_stats(out, gamma, beta, running_mean, running_var, training, sync=sync)


def bn_apply(x, s, relu, drop=None, res=None, dtype=torch.float32):
    """y = relu?((x*scale+shift) * drop? + res?), stored as ``dtype`` (fp32, or bf16 rounded to nearest even)."""
    C = x.shape[-1]
    npix = x.numel() // C
    y = torch.empty(x.shape, dtype=dtype, device=x.device)
    ppi = x.shape[1] * x.shape[2]
    entry = "lf_bn_apply_bf16" if dtype == torch.bfloat16 else "lf_bn_apply"
    _capi.call(entry, ptr(x), npix, C, ppi, ptr(s.scale), ptr(s.shift), ptr(drop), ptr(res), int(relu), ptr(y),
               _stream(), nbytes=npix * C * (4 * (1 + (res is not None)) + y.element_size()))
    return y


PREMASK_RESIDUAL = os.environ.get("LANEFIT_PREMASK_RES", "1") != "0"


def bn_backward(dy, ymask, drop, x, s, gamma, want_gated=False, sync=None):
    """-> (dx, dgamma, dbeta[, gated]).  g = dy*(ymask>0)*drop is recomputed on the fly; want_gated: also return
    dy*(ymask>0), stored by the apply pass (lf_bn_bwd_apply_gated).  sync: the forward's BNSync (s.count set)."""
    h = _lib()
    C = x.shape[-1]
    npix = x.numel() // C
    ppi = x.shape[1] * x.shape[2]
    st = _stream()
    nblk = h.lf_bn_blocks(npix, C)
    part = torch.empty(nblk * 2 * C, dtype=torch.float64, device=x.device)
    _capi.call("lf_bn_bwd_reduce", ptr(dy), ptr(ymask), ptr(drop), ptr(x), npix, C, ppi, ptr(s.mean), ptr(s.invstd),
                                   ptr(part), st, nbytes=4 * npix * C * (2 + (ymask is not None)))
    buf = torch.empty(4, C, dtype=torch.float32, device=x.device)
    dgamma, dbeta, c1, c2 = buf[0], buf[1], buf[2], buf[3]
    if sync is not None:
        glob, loc = _bn_collapse(part, nblk, npix, C, sync, keep_local=True)
        _capi.call("lf_bn_bwd_finalize_tot", ptr(loc), ptr(glob), ptr(s.count), C, ptr(dgamma), ptr(dbeta), ptr(c1), ptr(c2), st)
    else:
        _capi.call("lf_bn_bwd_finalize", ptr(part), nblk, npix, C, ptr(dgamma), ptr(dbeta), ptr(c1), ptr(c2), st)
    dx = torch.empty_like(x)
    if want_gated:
        gated = torch.empty_like(x)
        _capi.call("lf_bn_bwd_apply_gated", ptr(dy), ptr(ymask), ptr(drop), ptr(x), npix, C, ppi, ptr(s.mean), ptr(s.invstd),
                   ptr(gamma), ptr(c1), ptr(c2), ptr(dx), ptr(gated), st, nbytes=4 * npix * C * (4 + (ymask is not None)))
        return dx, dgamma, dbeta, gated
    _capi.call("lf_bn_bwd_apply", ptr(dy), ptr(ymask), ptr(drop), ptr(x), npix, C, ppi, ptr(s.mean), ptr(s.invstd),
                                  ptr(gamma), ptr(c1), ptr(c2), ptr(dx), st, nbytes=4 * npix * C * (3 + (ymask is not None)))
    return dx, dgamma, dbeta


# Fused BatchNorm backward for relu(bn(x)) feeding a 3-tap conv (BN1 of non_bottleneck_1d): the conv's input-gradient
# launch takes the BatchNorm INPUT x as its mask operand, rebuilds the ReLU mask bit with the forward's own
# fma(x, scale, shift) > 0, and accumulates sum g and sum g*x in its epilogue, from which sum g*xhat = invstd*(sum g*x -
# mean*sum g) -- so the separate reduction pass over (g, x) disappears, relu(bn(x)) is not read, and no division by the
# BatchNorm weight is involved (round 1 recovered xhat from (y - beta)/gamma, undefined at gamma = 0: ADVICE r1).
FUSE_BN_BWD = os.environ.get("LANEFIT_FUSE_BN_BWD", "1") != "0"


def dgrad_relu_bn_fused(d_out, w, vertical, dil, x, s, gamma, sync=None):
    """(dgrad of the 3-tap conv) * (relu(bn(x)) > 0) -> g, then BatchNorm backward -> (dx, dgamma, dbeta); s carries the
    forward's (mean, invstd, scale, shift[, count]).  Returns None when the shapes are not served by the slab kernel (caller
    takes the two-pass route).  sync: the forward's BNSync."""
    N, H, W, C = d_out.shape
    rows = tc_rows(d_out, vertical, dil, stats=True) if FUSE_BN_BWD else 0
    if rows <= 0:
        return None
    part = torch.empty(rows * 2 * C, dtype=torch.float64, device=d_out.device)
    taps = [((-(k - 1) * dil, 0) if vertical else (0, -(k - 1) * dil)) for k in range(3)]
    g = run_conv_tc(taps, d_out, packed(w, "tc_dgrad", pack_tc_dgrad, split=pack_split()), torch.empty_like(d_out), mask_src=x,
                    stats_partial=part, mask_affine=(s.scale, s.shift))
    npix = N * H * W
    buf = torch.empty(4, C, dtype=torch.float32, device=d_out.device)
    dgamma, dbeta, c1, c2 = buf[0], buf[1], buf[2], buf[3]
    st = _stream()
    if sync is not None:
        glob, loc = _bn_collapse(part, rows, npix, C, sync, keep_local=True)
        _capi.call("lf_bn_bwd_finalize_sx_tot", ptr(loc), ptr(glob), ptr(s.count), C, ptr(s.mean), ptr(s.invstd), ptr(dgamma),
                   ptr(dbeta), ptr(c1), ptr(c2), st)
    else:
        _capi.call("lf_bn_bwd_finalize_sx", ptr(part), rows, npix, C, 1, ptr(s.mean), ptr(s.invstd), ptr(dgamma), ptr(dbeta),
                   ptr(c1), ptr(c2), st)
    dx = torch.empty_like(x)
    _capi.call("lf_bn_bwd_apply", ptr(g), None, None, ptr(x), npix, C, H * W, ptr(s.mean), ptr(s.invstd), ptr(gamma), ptr(c1),
               ptr(c2), ptr(dx), st, nbytes=4 * npix * C * 3)
    return dx, dgamma, dbeta


def _require_training_for_backward(training):
    if not training:
        raise RuntimeError("backward through eval-mode BatchNorm is not implemented on the H100 path "
                           "(the reference only back-propagates in train mode, BP/main.py:232,338)")


# --------------------------------------------------------------------------------------
# DownsamplerBlock  (ERFNet.py:11-22):  relu(bn(cat[conv3x3 s2 p1 (x), maxpool2(x)]))
# --------------------------------------------------------------------------------------
class DownFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cin, w, b, gamma, beta, rm, rv, training, need_dx, sync=None):
        """x: [N,H,W,Cx] NHWC with Cx >= cin (stem: 3 channels padded to 4).  sync: BNSync (SyncBatchNorm) or None."""
        _capi.require_cuda(x)
        require_inference_mode(training)
        h = _lib()
        N, H, W, cx = x.shape
        cc = w.shape[0]                      # conv output channels = noutput - ninput
        cout = cc + cin
        cin_gemm = plans.pad_to(cin, 4)
        phases, (Ho, Wo) = plans.conv_fwd_plan(H, W, 3, 3, 2, 1, 1, 1, 1)
        cat = _empty((N, Ho, Wo, cout), x)
        if cc % 16 == 0 and tcg_s2conv_ok(x, cin, cc):
            run_tcg_s2conv(x, packed(w, "tcg_s2conv", pack_tcg_s2conv, split=pack_split()), cc, cat, bias=b)
        else:
            wmat = packed(w, "conv_fwd_%d" % cin_gemm, lambda t: pack_conv_fwd(t, cin_gemm))
            run_conv(phases, x, wmat, cin_gemm, cat, cc, 0, bias=b)
        _capi.call("lf_maxpool2_fwd", ptr(x), N, H, W, cin, cx, ptr(cat), cout, cc, _stream())
        s = bn_forward_stats(cat, gamma, beta, rm, rv, training, sync=sync)
        y = bn_apply(cat, s, relu=True)
        ctx.save_for_backward(x, w, cat, y, gamma, s.mean, s.invstd, s.count)
        ctx.cfg = (cin, training, need_dx, sync)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, cat, y, gamma, mean, invstd, count = ctx.saved_tensors
        cin, training, need_dx, sync = ctx.cfg
        _require_training_for_backward(training)
        h = _lib()
        dy = dy.contiguous()
        N, H, W, cx = x.shape
        cc = w.shape[0]
        cout = cc + cin
        s = BNState()
        s.mean, s.invstd, s.count = mean, invstd, count
        dcat, dgamma, dbeta = bn_backward(dy, y, None, cat, s, gamma, sync=sync)
        # weight / bias gradient of the conv part (channels [0,cc) of dcat)
        dw = torch.empty_like(w)
        db = _empty((cc,), x)
        wplan = plans.conv_wgrad_plan(H, W, 3, 3, 2, 1, 1, 1, 1)
        cin_gemm = plans.pad_to(cin, 4)
        cq_gemm = plans.pad_to(cc, 4)
        if cx == cin and wgrad_tcg_ok(x, cin, dcat, plans.pad_to(cc, 32)):
            dw = wgrad_tcg_conv(x, cin, dcat, cc)
            run_colsum(dcat, cc, 0, db)
        else:
            run_wgrad(wplan, x, cin_gemm, dcat, cq_gemm, 0, N, dw, (1, 9, cin * 9), db, cp_true=cin, cq_true=cc)
        dx = None
        if need_dx:
            dx = _empty((N, H, W, cx), x)
            if cx == cin and tcg_s2convT_ok(dcat, cc, cin):
                kc = plans.pad_to(cc, 32)
                wgs = tuple(packed(w, "tcg_s2convT%d_%d" % (par, kc), lambda t, par=par: pack_tcg_s2convT(t, par, kc), split=pack_split())
                            for par in (0, 1))
                run_tcg_s2convT(dcat, cc, wgs, cin, dx)
            else:
                wd = packed(w, "conv_dgrad", pack_conv_dgrad)   # [9, cc, cinPad]
                phases, _ = plans.transposed_gather_plan(dcat.shape[1], dcat.shape[2], H, W, 3, 1)
                run_conv(phases, dcat, wd, cc, dx, cin, 0)
            _capi.call("lf_maxpool2_bwd", ptr(x), N, H, W, cin, cx, ptr(dcat), cout, cc, ptr(dx), cx, 1, _stream())
        return dx, None, dw, db, dgamma, dbeta, None, None, None, None, None


# --------------------------------------------------------------------------------------
# non_bottleneck_1d  (ERFNet.py:25-60)
# --------------------------------------------------------------------------------------
def nb1d_storage_dtype(x, dil):
    """Element type of the non_bottleneck_1d tensors that are only convolution inputs and ReLU masks: t1, t3, t4 of
    Nb1dFunction and the three intermediates of ops_eval.nb1d (also in fp8 mode, whose kernels take either and
    quantise them per image).  bf16 in bf16 mode when every launch of the block,
    forward and backward, runs on the bf16 tensor-core kernels: they round these operands to bf16 (nearest even)
    anyway, so storing them rounded changes no result (a positive value at most half of bf16's smallest subnormal,
    2^-134, would round to zero and flip its ReLU mask bit).  fp32 otherwise."""
    if not bf16_mode():
        return torch.float32
    N, H, W, C = x.shape
    if super_ok(x, dil):
        ok = _lib().lf_wgrad3_tc_bf16_ctas(N, H, W // SUPER, SUPER * C) > 0
    else:
        ok = (all(tc_supported(x, v, d) for v in (True, False) for d in (1, dil))
              and _lib().lf_wgrad3_tc_bf16_ctas(N, H, W, C) > 0)
    return torch.bfloat16 if ok else torch.float32


class Nb1dFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, g1, be1, w3, b3, w4, b4, g2, be2, rm1, rv1, rm2, rv2, dil, drop, training, sync1=None,
                sync2=None):
        """sync1 / sync2: BNSync of bn1 / bn2 (SyncBatchNorm containers) or None."""
        _capi.require_cuda(x)
        if fp8_mode():
            raise RuntimeError("conv mode 'fp8' is inference-only: non_bottleneck_1d runs it on the folded eval path "
                               "(ops_eval.nb1d) only")
        N, H, W, C = x.shape
        sd = nb1d_storage_dtype(x, dil)
        t1 = conv3(x, w1, True, 1, False, bias=b1, relu=True, dtype=sd)
        t2, s1 = conv3_bn_stats(t1, w2, False, 1, b2, g1, be1, rm1, rv1, training, sync=sync1)
        t3 = bn_apply(t2, s1, relu=True, dtype=sd)
        t4 = conv3(t3, w3, True, dil, False, bias=b3, relu=True, dtype=sd)
        t5, s2 = conv3_bn_stats(t4, w4, False, dil, b4, g2, be2, rm2, rv2, training, sync=sync2)
        y = bn_apply(t5, s2, relu=True, drop=drop, res=x)
        ctx.save_for_backward(x, t1, t2, t3, t4, t5, y, w1, w2, w3, w4, g1, g2, s1.mean, s1.invstd, s2.mean, s2.invstd,
                              drop if drop is not None else x.new_empty(0), s1.scale, s1.shift, s1.count, s2.count)
        ctx.cfg = (dil, training, drop is not None, sync1, sync2)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x, t1, t2, t3, t4, t5, y, w1, w2, w3, w4, g1, g2, m1, is1, m2, is2, drop, sc1, sh1, n1, n2) = ctx.saved_tensors
        dil, training, has_drop, sync1, sync2 = ctx.cfg
        _require_training_for_backward(training)
        drop = drop if has_drop else None
        dy = dy.contiguous()
        N, H, W, C = x.shape
        s1, s2 = BNState(), BNState()
        s1.mean, s1.invstd, s2.mean, s2.invstd = m1, is1, m2, is2
        s1.scale, s1.shift = sc1, sh1
        s1.count, s2.count = n1, n2

        global _DEFERRED
        _DEFERRED = jobs = []
        try:
            return Nb1dFunction._backward_body(x, t1, t2, t3, t4, t5, y, w1, w2, w3, w4, g1, g2, s1, s2, drop, dil, dy, jobs,
                                               sync1, sync2)
        finally:
            _DEFERRED = None

    @staticmethod
    def _backward_body(x, t1, t2, t3, t4, t5, y, w1, w2, w3, w4, g1, g2, s1, s2, drop, dil, dy, jobs, sync1=None, sync2=None):
        N, H, W, C = x.shape
        # y = relu(bn2(t5)*drop + x).  The apply pass also emits gm = dy*(y>0), the gradient of the skip connection, so the
        # block's last conv adds one pre-masked operand instead of reading dy and y again in its epilogue.
        gm = None
        if PREMASK_RESIDUAL and tc_mode():
            d5, dg2, dbe2, gm = bn_backward(dy, y, drop, t5, s2, g2, want_gated=True, sync=sync2)
        else:
            d5, dg2, dbe2 = bn_backward(dy, y, drop, t5, s2, g2, sync=sync2)
        # Bias gradients.  conv1x3_1 / conv1x3_2 feed a BatchNorm: sum_pixels(BN backward output) == 0
        # identically (the reference's autograd returns pure round-off there), so db2 = db4 = 0.
        # conv3x1_1 / conv3x1_2 feed a ReLU: db = column sums of the masked input gradient, which the
        # dgrad launch below accumulates in its epilogue (colsum=...).
        zero2 = torch.zeros(2, C, device=x.device)           # one fill launch for both
        db2, db4 = zero2[0], zero2[1]
        db1, db3 = _empty((C,), x), _empty((C,), x)
        # conv1x3_2 (dilated)
        dw4, _ = wgrad3(t4, d5, w4, False, dil, bias_grad="skip")
        d4 = conv3(d5, w4, False, dil, True, colsum=db3, mask_src=t4)
        # conv3x1_2 (dilated)
        dw3, _ = wgrad3(t3, d4, w3, True, dil, bias_grad="skip")
        fused = dgrad_relu_bn_fused(d4, w3, True, dil, t2, s1, g1, sync=sync1)
        if fused is not None:
            d2, dg1, dbe1 = fused          # dgrad + relu mask + BatchNorm reductions in one launch, then apply
        else:
            d3 = conv3(d4, w3, True, dil, True, mask_src=t3)
            # bn1 (+relu already applied through mask_src=t3)
            d2, dg1, dbe1 = bn_backward(d3, None, None, t2, s1, g1, sync=sync1)
        # conv1x3_1
        dw2, _ = wgrad3(t1, d2, w2, False, 1, bias_grad="skip")
        d1 = conv3(d2, w2, False, 1, True, colsum=db1, mask_src=t1)
        # conv3x1_1, plus the residual branch: dx = dgrad + dy*(y>0)
        dw1, _ = wgrad3(x, d1, w1, True, 1, bias_grad="skip")
        dx = conv3(d1, w1, True, 1, True, add_src=gm) if gm is not None else conv3(d1, w1, True, 1, True, add_src=dy, add_mask=y)
        if jobs:
            flush_deferred_reductions(jobs)
        return (dx, dw1, db1, dw2, db2, dg1, dbe1, dw3, db3, dw4, db4, dg2, dbe2, None, None, None, None, None, None,
                None, None, None)


# --------------------------------------------------------------------------------------
# UpsamplerBlock  (ERFNet.py:98-107):  relu(bn(convT3x3 s2 p1 op1 (x)))
# --------------------------------------------------------------------------------------
class UpFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, rm, rv, training, sync=None):
        """sync: BNSync (SyncBatchNorm) or None."""
        _capi.require_cuda(x)
        require_inference_mode(training)
        N, H, W, ci = x.shape
        co = w.shape[1]
        phases, (Ho, Wo) = plans.transposed_gather_plan(H, W, 2 * H, 2 * W, 3, 1)
        if tcg_s2convT_ok(x, ci, co):
            wgs = tuple(packed(w, "tcg_s2convT%d_%d" % (par, ci), lambda t, par=par: pack_tcg_s2convT(t, par, ci), split=pack_split())
                        for par in (0, 1))
            u = run_tcg_s2convT(x, ci, wgs, co, _empty((N, Ho, Wo, co), x), bias2=packed(b, "tile2", lambda t: t.repeat(2)))
        else:
            u = run_conv(phases, x, packed(w, "convT_fwd", pack_convT_fwd), ci, _empty((N, Ho, Wo, co), x), co, bias=b)
        s = bn_forward_stats(u, gamma, beta, rm, rv, training, sync=sync)
        y = bn_apply(u, s, relu=True)
        ctx.save_for_backward(x, w, u, y, gamma, s.mean, s.invstd, s.count)
        ctx.training, ctx.sync = training, sync
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, u, y, gamma, mean, invstd, count = ctx.saved_tensors
        _require_training_for_backward(ctx.training)
        dy = dy.contiguous()
        N, H, W, ci = x.shape
        co = w.shape[1]
        s = BNState()
        s.mean, s.invstd, s.count = mean, invstd, count
        du, dgamma, dbeta = bn_backward(dy, y, None, u, s, gamma, sync=ctx.sync)
        dw, db = torch.empty_like(w), _empty((co,), x)
        if wgrad_tcg_ok(du, co, x, ci):
            dw = wgrad_tcg_convT(x, ci, du, co)
        else:
            run_wgrad(plans.convT_wgrad_plan(H, W, 3, 1), x, ci, du, co, 0, N, dw, (1, co * 9, 9))
        run_colsum(du, co, 0, db)
        if ci % 16 == 0 and tcg_s2conv_ok(du, co, ci):
            dx = run_tcg_s2conv(du, packed(w, "tcg_s2conv", pack_tcg_s2conv, split=pack_split()), ci, torch.empty_like(x))
        else:
            pd, _ = plans.convT_dgrad_plan(2 * H, 2 * W, H, W, 3, 1)
            dx = run_conv(pd, du, packed(w, "convT_dgrad", pack_convT_dgrad), co, torch.empty_like(x), ci)
        return dx, dw, db, dgamma, dbeta, None, None, None, None


# --------------------------------------------------------------------------------------
# Decoder.output_conv (ERFNet.py:124,152): ConvTranspose2d(16 -> L, 2, stride 2)
# NHWC in -> planar NCHW out (what the LSQ layer consumes and Net.forward returns)
# --------------------------------------------------------------------------------------
class OutConvFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        _capi.require_cuda(x)
        h = _lib()
        N, H, W, ci = x.shape
        L = w.shape[1]
        out = _empty((N, L, 2 * H, 2 * W), x)
        _capi.call("lf_outconv_fwd", ptr(x), ptr(w.contiguous()), ptr(b), N, H, W, ci, L, ptr(out), _stream())
        ctx.save_for_backward(x, w)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w = ctx.saved_tensors
        h = _lib()
        dout = dout.contiguous()
        N, H, W, ci = x.shape
        L = w.shape[1]
        st = _stream()
        dx = torch.empty_like(x)
        _capi.call("lf_outconv_bwd_data", ptr(dout), ptr(w.contiguous()), N, H, W, ci, L, ptr(dx), st)
        nblk = h.lf_outconv_wgrad_blocks(N * H * W)
        width = ci * L * 4 + L
        part = torch.empty(nblk * width, dtype=torch.float32, device=x.device)
        _capi.call("lf_outconv_bwd_weight", ptr(x), ptr(dout), N, H, W, ci, L, ptr(part), st)
        red = _empty((width,), x)
        _capi.call("lf_vec_reduce", ptr(part), nblk, width, width, ptr(red), st)
        dw = red[:ci * L * 4].view(ci, L, 2, 2)
        db = red[ci * L * 4:]
        return dx, dw, db


# --------------------------------------------------------------------------------------
# layout changes at the module boundary
# --------------------------------------------------------------------------------------
def image_to_nhwc_pad(x, cpad):
    """[N,C,H,W] fp32 -> [N,H,W,cpad] (zero padded); no gradient (input images)."""
    _capi.require_cuda(x)
    x = x.contiguous().float()
    N, C, H, W = x.shape
    out = _empty((N, H, W, cpad), x)
    _capi.call("lf_nchw_to_nhwc_pad", ptr(x), N, C, H, W, cpad, ptr(out), _stream())
    return out


class ToNHWC(torch.autograd.Function):
    """NCHW-contiguous -> NHWC-contiguous [N,H,W,C]."""

    @staticmethod
    def forward(ctx, x):
        _capi.require_cuda(x)
        x = x.contiguous()
        N, C, H, W = x.shape
        out = _empty((N, H, W, C), x)
        _capi.call("lf_nchw_to_nhwc", ptr(x), N, C, H, W, ptr(out), _stream())
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        N, H, W, C = g.shape
        out = _empty((N, C, H, W), g)
        _capi.call("lf_nhwc_to_nchw", ptr(g), N, H, W, C, ptr(out), _stream())
        return out


def as_nhwc(x):
    """Accept what a reference caller passes (NCHW-shaped) and return a dense [N,H,W,C] tensor.
    channels_last inputs (what our own blocks emit, viewed as NCHW) are re-viewed for free."""
    if x.dim() != 4:
        raise ValueError("expected a 4-D feature map")
    xp = x.permute(0, 2, 3, 1)
    if xp.is_contiguous():
        return xp
    return ToNHWC.apply(x)


def as_nchw_view(y):
    """[N,H,W,C] dense -> NCHW-shaped view (channels_last strides), zero copy."""
    return y.permute(0, 3, 1, 2)
