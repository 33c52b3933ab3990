"""fp64 restatements of the heads' kernel contracts (include/lanefit_b200.h; csrc/linear.cu, csrc/seg.cu): the fully
connected layer (lf_linear_fwd / _bwd_data / _bwd_weight), the row mean (lf_rowmean_fwd / _bwd), the weighted 2-D cross
entropy (lf_ce2d_fwd / _bwd) and the lane maps (lf_seg_lane_maps / _line) -- the per-entry gates the GPU tests hold the
kernels to, fp32 emulations of each kernel in its own operation order, and seeded mutations of those emulations.

The restatements are torch float64 on whatever device the operands live on.  u = 2^-24; a chain of k fp32 roundings
(adds or FMAs) is within k u S of the exact sum, S = sum |term|; gate(k, S) = (k + 8) u S, the +8 covering the second
order part (f32_contract.gate).
  lf_linear_fwd         each lane runs an FMA chain of <= 8 over its chunk's columns lane + 32 j, then 5 xor-shuffle
                        adds, then the finish kernel adds bias + the lf_linear_chunks(K) partials in chunk order:
                        k = 8 + 5 + nchunks + 1, S = |bias| + sum_k |x W|.  ReLU comes after the sum and
                        |relu(a) - relu(b)| <= |a - b|, so the same gate holds on y.
  lf_linear_bwd_data    one FMA chain over o: k = O, S = sum_o |g W|.  The gate g = dy * (relu_out > 0) is exact and is
                        checked exactly (+0.0, -0.0 and the smallest subnormal are not > 0, resp. are, as IEEE says).
  lf_linear_bwd_weight  dW and db are chains over the batch rows, BT rows per pass, the padded rows exact zeros, each pass
                        after the first continuing from the stored value: k = B.
  lf_rowmean_fwd        lpc = max(1, 256 // C) lanes per channel; lane p sums the ceil(W / lpc) columns w = p (mod lpc),
                        the lpc partials are summed in order, then one IEEE division by W: k = ceil(W/lpc) + lpc + 1,
                        S = sum_w |x| / W.
  lf_rowmean_bwd        dx = dout * fl32(1 / W): one fp32 multiply, bit-exact.
  lf_ce2d_fwd           per pixel, in fp32: m = max_c v_c (exact); e_c = expf(v_c - m) (the subtraction rounds by
                        u |d_c|, expf adds <= 2 ulp <= 4u); s = sum_c e_c in C - 1 adds of positive terms.  So
                        |s^/s - 1| <= sum_c p_c (|d_c| + 4) u + (C - 1) u <= (2C + 3) u, since p_c |d_c| = e^d |d| / s
                        <= 1/e.  logf adds <= 1 ulp <= 2u log C; m + log s, - x_t and w * b each round once.  Per pixel
                        |b^_i - b_i| <= u (3 |m| + 2 |x_t| + 5 log C + 2C + 3) w_i; the cross-pixel sums are fp64 (N 2^-53
                        relative).  Gate on the loss: sum_i w_i u (3|m_i| + 2|x_t,i| + 5 log C + 2C + 3 + 8) / sum_i w_i
                        plus the fp64 terms.
  lf_ce2d_bwd           dx = fl(fl(gscale w) (p_c - [c = t])), gscale = fl32(gout / sum w), p_c = fl(e_c fl(1/s)):
                        |p^_c / p_c - 1| <= u (|d_c| + 2C + 9); the subtraction rounds by u |p_c - [c = t]| whether or not
                        nvcc contracts e * inv - 1 into an FMA (the fused form rounds once, the unfused twice, both
                        inside this); gscale, gscale w and the last product add 3u.  Gate per entry:
                        |G w| u (p_c (|d_c| + 2C + 9) + 4 |p_c - [c = t]| + 8 (p_c + [c = t])) + |G w| 2^-126 + 2^-148,
                        the two absolute terms for expf / the products underflowing into subnormals.  The u |d_c| term
                        is reached in full by correct arithmetic when |d_c| lies just above a power of two, so widely
                        spread logits sit near |d_c| / (|d_c| + 2C + 29) of this gate.  A pixel whose target is outside
                        [0, C) writes +0.0 exactly.
  lf_seg_lane_maps      exact: the first maximum wins, rows < mask_rows are zero; with gt_line, a flagged lane gets image
                        0's (argmax == 1) map.
"""
import math

import torch
import torch.nn.functional as F

from f32_contract import F64, U, excess, gate  # noqa: F401  (re-exported for the tests)

LIN_KC = 256                   # K columns per forward / backward CTA (csrc/linear.cu)
LIN_BWD_SMEM = 96 * 1024       # the backward kernels' shared-memory cap: O * BT * 4 bytes


# ---------------------------------------------------------------------------------------------------------------------
# lf_linear_*
# ---------------------------------------------------------------------------------------------------------------------
def lin_chunks(K):
    return -(-K // LIN_KC)


def lin_bt(n):
    return 8 if n <= 8 else 16 if n <= 16 else 32 if n <= 32 else 64


def lin_passes(B):
    """(b0, BT) of every 64-row pass the host makes."""
    return [(b0, lin_bt(B - b0)) for b0 in range(0, B, 64)]


def lin_bwd_accepts(B, O):
    """The backward entry points refuse a pass whose dy tile O * BT * 4 bytes exceeds the cap; the first pass is the
    widest, so a refusal comes before any launch."""
    return O * lin_bt(B) * 4 <= LIN_BWD_SMEM


def linear_fwd_k(K):
    return 8 + 5 + lin_chunks(K) + 1


def relu_gate(dy, relu_out, ge=False):
    """g = dy where relu_out > 0 (NaN, +-0 and negatives gate), else +0.0.  ge: the mutation that gates with >= 0."""
    if relu_out is None:
        return dy
    keep = (relu_out >= 0) if ge else (relu_out > 0)
    return torch.where(keep, dy, torch.zeros_like(dy))


def linear_fwd(x, W, bias=None, relu=False):
    """x [B, K], W [O, K] -> (y [B, O], S)."""
    x, W = x.to(F64), W.to(F64)
    y, S = x @ W.T, x.abs() @ W.abs().T
    if bias is not None:
        y, S = y + bias.to(F64), S + bias.to(F64).abs()
    return (y.clamp_min(0) if relu else y), S


def linear_bwd_data(dy, relu_out, W):
    """-> (dx [B, K], S); k = O."""
    g, W = relu_gate(dy, relu_out).to(F64), W.to(F64)
    return g @ W, g.abs() @ W.abs()


def linear_bwd_weight(dy, relu_out, x):
    """-> (dW [O, K], S, db [O], S of db); k = B."""
    g, x = relu_gate(dy, relu_out).to(F64), x.to(F64)
    return g.T @ x, g.abs().T @ x.abs(), g.sum(0), g.abs().sum(0)


def _fma(a, b, c):
    """fl32(a b + c) for fp32 operands: the product is exact in fp64; the sum is rounded to fp64, then to fp32 (a double
    rounding the exact FMA does not have -- off by one fp32 ulp at most, far inside every gate)."""
    return (a.double() * b.double() + c.double()).float()


def emulate_linear_fwd(x, W, bias=None, relu=False, mutate=None):
    """fp32 in linear_fwd_kernel's order.  mutate: "drop_last_chunk" (the finish kernel leaves the last K chunk out)."""
    B, K = x.shape
    O, nch = W.shape[0], lin_chunks(K)
    Kp = nch * LIN_KC
    xs = F.pad(x.float(), (0, Kp - K)).view(B, 1, nch, 8, 32)        # column c*256 + 32 j + lane
    ws = F.pad(W.float(), (0, Kp - K)).view(1, O, nch, 8, 32)
    s = torch.zeros(B, O, nch, 32, dtype=torch.float32)
    for j in range(8):
        s = _fma(ws[..., j, :], xs[..., j, :], s)
    lane = torch.arange(32)
    for off in (16, 8, 4, 2, 1):                                      # warp_sum: xor butterfly, lane 0's value
        s = s + s[..., lane ^ off]
    part = s[..., 0]
    y = bias.float().expand(B, O).clone() if bias is not None else torch.zeros(B, O, dtype=torch.float32)
    for c in range(nch - 1 if mutate == "drop_last_chunk" else nch):
        y = y + part[..., c]
    return y.clamp_min(0) if relu else y


def emulate_linear_bwd_data(dy, relu_out, W, mutate=None):
    """fp32 in linear_bwd_data_kernel's order.  mutate: "relu_ge" (relu_out >= 0 lets the gradient through)."""
    g = relu_gate(dy.float(), relu_out, ge=(mutate == "relu_ge"))
    W = W.float()
    acc = torch.zeros(g.shape[0], W.shape[1], dtype=torch.float32)
    for o in range(W.shape[0]):
        acc = _fma(g[:, o:o + 1], W[o][None, :], acc)
    return acc


def emulate_linear_bwd_weight(dy, relu_out, x, mutate=None):
    """fp32 in linear_bwd_weight_kernel's order -> (dW, db).  mutate: "pad_leak" (the padded rows of a BT tile repeat the
    tile's first row instead of holding zeros), "no_accumulate" (each 64-row pass overwrites dW / db)."""
    g, x = relu_gate(dy.float(), relu_out), x.float()
    B, O, K = g.shape[0], g.shape[1], x.shape[1]
    dW, db = torch.zeros(O, K, dtype=torch.float32), torch.zeros(O, dtype=torch.float32)
    for b0, bt in lin_passes(B):
        if b0 > 0 and mutate == "no_accumulate":
            dW, db = torch.zeros_like(dW), torch.zeros_like(db)
        for b in range(bt):
            r = b0 + b
            if r >= B:
                if mutate != "pad_leak":
                    continue                  # exact zeros: fma(0, 0, s) = s, s + 0 = s
                r = b0
            dW = _fma(g[r][:, None], x[r][None, :], dW)
            db = db + g[r]
    return dW, db


# ---------------------------------------------------------------------------------------------------------------------
# lf_rowmean_*: x NHWC [B, H, W, C] -> out [B, C*H], out[b][c*H + h] = mean_w x[b][h][w][c]
# ---------------------------------------------------------------------------------------------------------------------
def rowmean_lpc(C):
    return max(1, 256 // C)


def rowmean_k(W, C):
    lpc = rowmean_lpc(C)
    return -(-W // lpc) + lpc + 1


def _nchw_flat(t):
    """[B, H, C] -> [B, C*H] in the reference's NCHW view order."""
    return t.permute(0, 2, 1).reshape(t.shape[0], -1)


def rowmean_fwd(x):
    """-> (out [B, C*H], S)."""
    x = x.to(F64)
    W = x.shape[2]
    return _nchw_flat(x.mean(2)), _nchw_flat(x.abs().sum(2) / W)


def rowmean_bwd(dout, B, H, W, C):
    """The exact fp32 result: dx[b][h][w][c] = dout[b][c*H + h] * fl32(1/W) (on dout's device)."""
    inv = torch.ones((), dtype=torch.float32, device=dout.device) / torch.full((), float(W), dtype=torch.float32,
                                                                               device=dout.device)
    g = dout.float().view(B, C, H).permute(0, 2, 1)[:, :, None, :] * inv
    return g.expand(B, H, W, C).contiguous()


def emulate_rowmean_fwd(x, mutate=None):
    """fp32 in rowmean_fwd_kernel's order.  mutate: "div_w_minus_1", "drop_last_lane" (the lpc partials stop one short)."""
    x = x.float()
    B, H, W, C = x.shape
    lpc = rowmean_lpc(C)
    steps = -(-W // lpc)
    xw = F.pad(x, (0, 0, 0, steps * lpc - W)).view(B, H, steps, lpc, C)    # column w = step * lpc + lane
    s = torch.zeros(B, H, lpc, C, dtype=torch.float32)
    for st in range(steps):
        s = s + xw[:, :, st]
    t = torch.zeros(B, H, C, dtype=torch.float32)
    for p in range(lpc - 1 if mutate == "drop_last_lane" else lpc):
        t = t + s[:, :, p]
    div = float(W - 1 if mutate == "div_w_minus_1" else W)
    return _nchw_flat(t / torch.full((), div, dtype=torch.float32))


# ---------------------------------------------------------------------------------------------------------------------
# lf_ce2d_*: x [B, C, H, W] planar logits, target [B, H, W] int64, weight [C] or None
# ---------------------------------------------------------------------------------------------------------------------
def ce_weights(target, weight, C, dtype=F64):
    """(counted, t clamped to a valid class, w_i): w_i = weight[t_i] (1 without a weight vector), 0 when uncounted."""
    counted = (target >= 0) & (target < C)
    t = torch.where(counted, target, torch.zeros_like(target))
    w = weight.to(dtype)[t] if weight is not None else torch.ones(t.shape, dtype=dtype, device=t.device)
    return counted, t, torch.where(counted, w, torch.zeros_like(w))


def _ce_pixels(x, target, weight):
    x = x.to(F64)
    C = x.shape[1]
    counted, t, w = ce_weights(target, weight, C)
    m = x.max(1).values
    d = x - m[:, None]
    e = torch.exp(d)
    s = e.sum(1)
    xt = x.gather(1, t[:, None]).squeeze(1)
    return counted, t, w, m, d, e / s[:, None], m + torch.log(s) - xt, xt


def ce2d_fwd(x, target, weight):
    """-> (loss, gate, den = sum_i w_i) in fp64.  den = 0 gives NaN, as torch's cross_entropy does."""
    C, N = x.shape[1], target.numel()
    _, _, w, m, _, _, b, xt = _ce_pixels(x, target, weight)
    num, den = (w * b).sum(), w.sum()
    loss = num / den
    per = w * U * (3 * m.abs() + 2 * xt.abs() + 5 * math.log(C) + 2 * C + 3 + 8)
    fp64 = N * 2.0 ** -53 * ((w * b).abs().sum() + loss.abs() * den) + 2.0 ** -52 * loss.abs() * den
    return float(loss), float((per.sum() + fp64) / den), float(den)


def ce2d_bwd(x, target, weight, gout=None):
    """-> (dx [B, C, H, W], per-entry gate) in fp64; gout None stands for 1."""
    C = x.shape[1]
    counted, t, w, m, d, p, _, _ = _ce_pixels(x, target, weight)
    G = (1.0 if gout is None else gout) / w.sum()
    onehot = F.one_hot(t, C).permute(0, 3, 1, 2).to(F64) * counted[:, None].to(F64)
    Gw = (G * w)[:, None]
    dx = Gw * (p - onehot)
    bound = Gw.abs() * (U * (p * (d.abs() + 2 * C + 9) + 4 * (p - onehot).abs() + 8 * (p + onehot)) + 2.0 ** -126) + 2.0 ** -148
    return torch.where(counted[:, None], dx, torch.zeros_like(dx)), bound


def _emulate_ce_pixels(x, target, weight, mutate):
    x = x.float()
    C = x.shape[1]
    counted, t, _ = ce_weights(target, weight, C)
    m = torch.zeros_like(x[:, 0]) if mutate == "no_max" else x.max(1).values
    e = torch.exp(x - m[:, None])
    s = torch.zeros_like(m)
    for c in range(C):
        s = s + e[:, c]
    wsel = x.argmax(1) if mutate == "argmax_weight" else t
    w = weight.float()[wsel] if weight is not None else torch.ones_like(m)
    w = torch.where(counted, w, torch.zeros_like(w))
    return x, counted, t, w, m, e, s


def emulate_ce2d_fwd(x, target, weight, mutate=None):
    """fp32 per pixel, fp64 across pixels, as ce2d_kernel<false> -> (loss, den).  mutate: "count_uncounted" (uncounted
    pixels add weight[0] to the weight sum), "argmax_weight" (the argmax class's weight instead of the target's),
    "no_max" (no max subtraction: expf overflows from logits of about 89 on)."""
    x, counted, t, w, m, e, s = _emulate_ce_pixels(x, target, weight, mutate)
    xt = x.gather(1, t[:, None]).squeeze(1)
    num = (w * ((m + torch.log(s)) - xt)).double().sum()
    wden = w
    if mutate == "count_uncounted":
        w0 = weight.float()[0] if weight is not None else torch.ones(())
        wden = torch.where(counted, w, w0.expand_as(w))
    den = wden.double().sum()
    return float(num / den), float(den)


def emulate_ce2d_bwd(x, target, weight, gout=None, mutate=None):
    """fp32 as ce2d_kernel<true>, the weight sum from the forward's emulation.  mutate as emulate_ce2d_fwd, plus
    "next_image" (image b's gradient computed from image b + 1's planes)."""
    _, den = emulate_ce2d_fwd(x, target, weight, mutate if mutate != "next_image" else None)
    gscale = (torch.tensor(1.0 if gout is None else gout, dtype=F64) / den).float()     # inf / NaN when den = 0
    xs = x.roll(-1, 0) if mutate == "next_image" else x
    x, counted, t, w, m, e, s = _emulate_ce_pixels(xs, target, weight, mutate)
    inv = 1.0 / s
    onehot = F.one_hot(t, x.shape[1]).permute(0, 3, 1, 2).float() * counted[:, None].float()
    dx = (gscale * w)[:, None] * (e * inv[:, None] - onehot)
    return torch.where(counted[:, None], dx, torch.zeros_like(dx))


# ---------------------------------------------------------------------------------------------------------------------
# lf_seg_lane_maps / _line: out [B, C, H, W] -> maps [B, nl, H, W]
# ---------------------------------------------------------------------------------------------------------------------
def lane_maps(out, nl, mask_rows, gt_line=None):
    """The reference's formulation: torch.max(out, 1)[1] (the first maximum), lane k's map (arg == k+1) * (k+1), rows
    < mask_rows zeroed; a lane flagged in gt_line takes image 0 / lane 0's map."""
    arg = torch.max(out, 1)[1]
    H = out.shape[2]
    keep = (torch.arange(H, device=out.device) >= mask_rows).view(1, H, 1)
    maps = torch.stack([torch.where((arg == k + 1) & keep, float(k + 1), 0.0) for k in range(nl)], 1).float()
    if gt_line is not None:
        flag = (gt_line != 0)[:, :, None, None]
        maps = torch.where(flag, maps[0:1, 0:1].expand_as(maps), maps)
    return maps


# ---------------------------------------------------------------------------------------------------------------------
# shapes shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------
LIN_B = [1, 7, 8, 9, 16, 17, 32, 33, 64, 65, 96, 130]
LIN_K = [1, 31, 32, 255, 256, 257, 700, 2048, 32768]
LIN_O = [1, 3, 4, 9, 12, 128, 256, 320]
LIN_CLASSES = ["randn", "heavy", "relu"]


def linear_cases():
    """(B, K, O, relu, bias, db, operand class): a sampled product in which every B appears three times and every K
    four times, cycling O, the flags and the operand classes."""
    out = []
    for i, B in enumerate(LIN_B):
        for j in range(3):
            n = 3 * i + j
            out.append((B, LIN_K[(i + 4 * j) % len(LIN_K)], LIN_O[(i + 3 * j) % len(LIN_O)], n % 2 == 0, n % 3 != 1,
                        n % 4 != 3, LIN_CLASSES[n % 3]))
    return out


LIN_PRODUCTION = [(K, O, relu) for K, O, relu in ((32768, 128, True), (128, 4, False), (128, 12, False), (128, 3, False),
                                                  (128, 5, False), (2048, 256, False), (2048, 320, False))]

ROWMEAN_C = [1, 3, 64, 100, 128, 255, 256]
ROWMEAN_W = [1, 2, 63, 64, 65, 1000]
ROWMEAN_H = [1, 32]
HORIZON = (32, 64, 64)          # the horizon head's (H, W, C): AvgPool2d((1, 64)) over 64 channels, C*H = 2048

def operand(shape, cls, g, device="cpu"):
    """randn; heavy-tailed randn * exp(2 randn); or a ReLU output (half exact zeros)."""
    t = torch.randn(shape, generator=g, device=device)
    if cls == "relu":
        return t.clamp_min(0)
    if cls == "heavy":
        return t * torch.exp(2 * torch.randn(shape, generator=g, device=device))
    return t


CE_LOGITS = ["randn","randn30", "ties", "spread80", "big1e4"]
CE_WEIGHTS = ["none", "positive", "zero_class"]
CE_TARGETS = ["in_range", "mixed", "none"]
CE_GOUT = [None, 1.0, -3.5, 0.0]


def ce_cases():
    """(C, weight mode, target mode, gout, logits) for C = 1..8 and every target mode, cycling the rest."""
    out = []
    for C in range(1, 9):
        for j, tm in enumerate(CE_TARGETS):
            out.append((C, CE_WEIGHTS[(C + j) % 3], tm, CE_GOUT[(C + 2 * j) % 4], CE_LOGITS[(2 * C + j) % 5]))
    return out


def ce_logits(shape, kind, g, device="cpu"):
    t = torch.randn(shape, generator=g, device=device)
    if kind == "randn30":
        return t * 30
    if kind == "ties":
        return torch.randint(-2, 3, shape, generator=g, device=device).float()
    if kind == "spread80":
        return torch.rand(shape, generator=g, device=device) * 160 - 80
    if kind == "big1e4":
        t[:, -1] = 1e4                                  # one class far above the rest: every other expf underflows to 0
        return t
    return t


def ce_targets(shape, C, mode, g, device="cpu"):
    t = torch.randint(0, C, shape, generator=g, device=device)
    if mode == "none":
        return torch.full(shape, -100, dtype=torch.long, device=device)
    if mode == "mixed":
        bad = torch.tensor([-100, -1, C, C + 5], device=device)
        pick = torch.randint(0, 8, shape, generator=g, device=device)
        t = torch.where(pick < 4, bad[pick.clamp_max(3)], t)        # half the pixels uncounted, every kind of miss
    return t


def ce_weight(C, mode, g, device="cpu"):
    if mode == "none":
        return None
    w = torch.rand(C, generator=g, device=device) * 2 + 0.25
    if mode == "zero_class":
        w[C // 2] = 0.0
    return w
