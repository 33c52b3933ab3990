"""fp64 restatements of the CUDA-core kernels' contracts (include/lanefit_b200.h): lf_conv_f32, lf_wgrad_f32 and the
split reductions, BatchNorm forward / apply / backward, the 2x2 max pool and its gradient, the output ConvTranspose2d,
the layout changes and lf_pack_gather -- plus the per-entry gates the GPU tests hold the kernels to.

Everything here is torch float64 on whatever device the operands live on (the CPU in tests/test_f32_contract_cpu.py,
the GPU in the kernel tests, where only the reference arithmetic runs in fp64).  The formulas are the header's, written
on the same strided views the C structs describe: a "spec" is a SimpleNamespace carrying the integer fields of the
struct under the struct's names, the tensors are flat 1-D buffers.

Gates.  An fp32 chain of k fused multiply-adds / adds, each rounded once, is within k * 2^-24 * S of the exact sum,
S = sum |term| (first-order; the +c below covers the second-order part at the chain lengths used here).
  lf_conv_f32   k = ntaps*Cin rounded up to the kernel's 16-wide K step (the padded steps add exact zeros) + bias + add_src
  lf_wgrad_f32  k = the pixels of the split: no thread accumulates more than that, and the fixed-order combine of the
                pixel groups (<= 64 adds) is inside c; the reduced result adds one add per split
  lf_colsum     k = pixels per block; lf_vec_reduce / lf_wgrad_reduce: k = nsplit
  lf_outconv_*  forward 16 FMAs + bias; data gradient 4L products; weight gradient 16 pixels per thread, 5 shuffle
                steps and 8 warp sums per 4096-pixel block
Pool, layout and pack kernels move or select values: exact equality.  BatchNorm: see bn_stat_bounds.
"""
import math
from types import SimpleNamespace as NS

import torch

U = 2.0 ** -24                      # fp32 unit round-off
F64 = torch.float64


def gate(k, S, c=8):
    return (k + c) * U * S


def excess(got, ref, bound):
    """max |got - ref| / bound over the entries (0/0 counts as 0, x/0 as inf)."""
    err = (got.to(F64) - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    return float(r.max()) if r.numel() else 0.0


def pixels(N, Hs, Ws, device="cpu"):
    m = torch.arange(N * Hs * Ws, device=device)
    return m // (Hs * Ws), (m // Ws) % Hs, m % Ws


def gather(flat, H, W, cstride, coff, C, n, y, x):
    """[M, C] fp64 rows flat[((n*H + y)*W + x)*cstride + coff + c], zero where (y, x) is outside [0,H) x [0,W)."""
    ok = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    base = ((n * H + y.clamp(0, H - 1)) * W + x.clamp(0, W - 1)) * cstride + coff
    idx = base[:, None] + torch.arange(C, device=flat.device)[None, :]
    v = flat[idx].to(F64)
    return torch.where(ok[:, None], v, torch.zeros_like(v))


# ---------------------------------------------------------------------------------------------------------------------
# lf_conv_f32
# ---------------------------------------------------------------------------------------------------------------------
def conv_spec(N, Hin, Win, Cin, Hout, Wout, Cout, CoutPad, phase, in_cstride=None, out_cstride=None, out_coff=0, relu=0):
    s = NS(N=N, Hin=Hin, Win=Win, Cin=Cin, in_cstride=in_cstride or Cin, Hout=Hout, Wout=Wout,
           out_cstride=out_cstride or Cout, out_coff=out_coff, Cout=Cout, CoutPad=CoutPad, relu=relu)
    for k in ("Hs", "Ws", "osy", "osx", "oy0", "ox0", "isy", "isx"):
        setattr(s, k, phase[k])
    s.ntaps = len(phase["taps"])
    s.dy, s.dx, s.wtap = ([t[i] for t in phase["taps"]] for i in range(3))
    return s


def conv_out_offsets(s, device="cpu", ignore_coff=False):
    n, j, i = pixels(s.N, s.Hs, s.Ws, device)
    pix = (n * s.Hout + j * s.osy + s.oy0) * s.Wout + i * s.osx + s.ox0
    return (pix * s.out_cstride + (0 if ignore_coff else s.out_coff))[:, None] + torch.arange(s.Cout, device=device)[None, :]


def conv_f32(s, inp, wmat, bias=None, mask_src=None, add_src=None, add_mask=None, m_limit=None, tap_shift=None,
             ignore_coff=False):
    """-> (ref [M, Cout], S [M, Cout], off [M, Cout] flat output indices).  Mutations: m_limit (pixels >= m_limit left
    out: a dropped pixel tile), tap_shift = (t, ddx) (tap t read ddx pixels to the side), ignore_coff."""
    dev = inp.device
    n, j, i = pixels(s.N, s.Hs, s.Ws, dev)
    w = wmat.to(F64).view(-1, s.Cin, s.CoutPad)
    acc = torch.zeros(n.numel(), s.Cout, dtype=F64, device=dev)
    S = torch.zeros_like(acc)
    for t in range(s.ntaps):
        ddx = tap_shift[1] if tap_shift is not None and tap_shift[0] == t else 0
        A = gather(inp, s.Hin, s.Win, s.in_cstride, 0, s.Cin, n, j * s.isy + s.dy[t], i * s.isx + s.dx[t] + ddx)
        Wt = w[s.wtap[t], :, :s.Cout]
        acc += A @ Wt
        S += A.abs() @ Wt.abs()
    if bias is not None:
        acc += bias.to(F64)[None, :s.Cout]
        S += bias.to(F64).abs()[None, :s.Cout]
    if s.relu:
        acc = acc.clamp_min(0)
    off = conv_out_offsets(s, dev, ignore_coff)
    if mask_src is not None:
        acc = torch.where(mask_src[off] > 0, acc, torch.zeros_like(acc))
    if add_src is not None:
        ad = add_src[off].to(F64)
        if add_mask is not None:
            ad = torch.where(add_mask[off] > 0, ad, torch.zeros_like(ad))
        acc = acc + ad
        S = S + ad.abs()
    if m_limit is not None:
        acc, S, off = acc[:m_limit], S[:m_limit], off[:m_limit]
    return acc, S, off


def conv_ksteps(s):
    return ((s.ntaps * s.Cin + 15) // 16) * 16 + 2


# ---------------------------------------------------------------------------------------------------------------------
# lf_wgrad_f32 and the reductions
# ---------------------------------------------------------------------------------------------------------------------
def wgrad_spec(N, plan, Hp, Wp, Cp, Hq, Wq, Cq, p_cstride=None, p_coff=0, q_cstride=None, q_coff=0, nsplit=1):
    s = NS(N=N, Hs=plan["Hs"], Ws=plan["Ws"], Hp=Hp, Wp=Wp, Cp=Cp, p_cstride=p_cstride or Cp, p_coff=p_coff,
           psy=plan["psy"], psx=plan["psx"], Hq=Hq, Wq=Wq, Cq=Cq, q_cstride=q_cstride or Cq, q_coff=q_coff,
           qsy=plan["qsy"], qsx=plan["qsx"], ntaps=len(plan["ptaps"]), nsplit=nsplit)
    s.pdy, s.pdx = [t[0] for t in plan["ptaps"]], [t[1] for t in plan["ptaps"]]
    s.qdy, s.qdx = [t[0] for t in plan["qtaps"]], [t[1] for t in plan["qtaps"]]
    s.CpPad, s.CqPad = -(-Cp // 64) * 64, -(-Cq // 64) * 64
    return s


def wgrad_f32(s, P, Q, m0=0, m1=None, tap_shift=None):
    """Pixels [m0, m1) of the domain -> (G [ntaps, Cp, Cq], S of G, qsum [Cq], S of qsum).  qsum is the column sum of
    tap 0's Q rows (the bias gradient when Q is dense)."""
    dev = P.device
    n, j, i = (t[m0:m1] for t in pixels(s.N, s.Hs, s.Ws, dev))
    G = torch.zeros(s.ntaps, s.Cp, s.Cq, dtype=F64, device=dev)
    S = torch.zeros_like(G)
    qsum = Sq = None
    for t in range(s.ntaps):
        ddx = tap_shift[1] if tap_shift is not None and tap_shift[0] == t else 0
        Pm = gather(P, s.Hp, s.Wp, s.p_cstride, s.p_coff, s.Cp, n, j * s.psy + s.pdy[t], i * s.psx + s.pdx[t] + ddx)
        Qm = gather(Q, s.Hq, s.Wq, s.q_cstride, s.q_coff, s.Cq, n, j * s.qsy + s.qdy[t], i * s.qsx + s.qdx[t])
        G[t] = Pm.T @ Qm
        S[t] = Pm.abs().T @ Qm.abs()
        if t == 0:
            qsum, Sq = Qm.sum(0), Qm.abs().sum(0)
    return G, S, qsum, Sq


def ws_plan(s, want_qsum):
    """Which kernel lf_wgrad_f32 runs: the plan of the small-channel kernel (all taps in one CTA), or (None, reason) when
    the tile kernel serves the shape.  Needed by the tests to know each split's pixel range (rounded up to PXS pixels)
    and to steer cases into every branch; lf_wgrad_f32_nsplit (> 0 iff a plan exists, = min(2 * SMs, ceil(M / 4 PXS)))
    is held against it."""
    p_same = all((s.pdy[t], s.pdx[t]) == (s.pdy[0], s.pdx[0]) for t in range(s.ntaps))
    q_same = all((s.qdy[t], s.qdx[t]) == (s.qdy[0], s.qdx[0]) for t in range(s.ntaps))
    if s.ntaps > 1 and p_same == q_same:
        return None, "both_or_neither_gathered"
    if s.Cp > 16 and s.Cq > 16:
        return None, "wide"
    taps_on_p = s.ntaps == 1 or not p_same
    if not taps_on_p and (want_qsum or s.Cq % 16 != 0):
        return None, "taps_on_q_qsum_or_cq"
    LU = s.ntaps * s.Cp if taps_on_p else s.Cp
    LV = s.Cq if taps_on_p else s.ntaps * s.Cq
    if LU % 4 or LV % 16:
        return None, "lu_lv_granularity"
    TPG = (LU // 4) * (LV // 16)
    if TPG > 256 or TPG < 1:
        return None, "too_many_threads"
    G = 256 // TPG
    threads = -(-G * TPG // 32) * 32
    PXG = 4 if G >= 8 else (16 if G >= 2 else 32)
    PXS = PXG * G
    per_px4 = (LU + LV) // 4
    if per_px4 > threads:
        return None, "fetch_wider_than_cta"
    ppp = threads // per_px4
    tile_floats = 2 * PXS * (LU + LV)
    if G > 1 and LU * LV + LV > tile_floats:
        return None, "reduction_scratch"
    if tile_floats * 4 > 96 * 1024:
        return None, "smem"
    return NS(taps_on_p=taps_on_p, LU=LU, LV=LV, G=G, PXG=PXG, PXS=PXS, ppp=ppp, passes=-(-PXS // ppp)), None


def tile_pxs(s):
    """Pixels per step of the tile kernel's four instantiations: 16-pixel (8 for 16 x 16) steps per thread group."""
    sp, sq = s.Cp <= 16, s.Cq <= 16
    return 128 if (sp and sq) else (64 if (sp or sq) else 16)


def split_ranges(M, nsplit, PXS):
    per = -(-M // nsplit)
    per = -(-per // PXS) * PXS
    return [(min(M, k * per), min(M, min(M, k * per) + per)) for k in range(nsplit)]


def reduce_ref(partial, nsplit, ntaps, Cp, Cq, CpPad, CqPad):
    """partial [nsplit][ntaps][CpPad][CqPad] (flat fp32) -> (sum over splits [ntaps, Cp, Cq] fp64, S)."""
    p = partial[:nsplit * ntaps * CpPad * CqPad].to(F64).view(nsplit, ntaps, CpPad, CqPad)[:, :, :Cp, :Cq]
    return p.sum(0), p.abs().sum(0)


def reduce_offsets(ntaps, Cp, Cq, st, sp, sq, device="cpu"):
    t, cp, cq = torch.meshgrid(torch.arange(ntaps, device=device), torch.arange(Cp, device=device),
                               torch.arange(Cq, device=device), indexing="ij")
    return t * st + cp * sp + cq * sq


# ---------------------------------------------------------------------------------------------------------------------
# BatchNorm2d, training mode, dense [npix][C]
# ---------------------------------------------------------------------------------------------------------------------
def bn_forward(x, gamma, beta, eps, momentum=None, running_mean=None, running_var=None, biased_running=False):
    """x [npix, C] -> dict(mean, var (biased), invstd, scale, shift, running_mean, running_var), all fp64.
    biased_running: the mutation that feeds the biased variance into the running statistic."""
    x = x.to(F64)
    n = x.shape[0]
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    scale = gamma.to(F64) * invstd
    r = dict(mean=mean, var=var, invstd=invstd, scale=scale, shift=beta.to(F64) - mean * scale)
    if running_mean is not None:
        unb = var if (biased_running or n <= 1) else var * n / (n - 1)
        r["running_mean"] = (1 - momentum) * running_mean.to(F64) + momentum * mean
        r["running_var"] = (1 - momentum) * running_var.to(F64) + momentum * unb
    return r


def _per_image(drop, npix, pix_per_image):
    img = torch.arange(npix, device=drop.device) // pix_per_image
    return drop.to(F64)[img]


def bn_apply(x, scale, shift, pix_per_image=1, drop=None, res=None, relu=False):
    """y = relu?((x*scale + shift) * drop[n]? + res?) and T = the magnitude the fp32 roundings scale with."""
    x = x.to(F64)
    y = x * scale.to(F64) + shift.to(F64)
    T = (x * scale.to(F64)).abs() + shift.to(F64).abs()
    if drop is not None:
        d = _per_image(drop, x.shape[0], pix_per_image)
        y, T = y * d, T * d.abs()
    if res is not None:
        y, T = y + res.to(F64), T + res.to(F64).abs()
    return (y.clamp_min(0) if relu else y), T


def bn_gated(dy, pix_per_image=1, ymask=None, drop=None):
    g = dy.to(F64)
    if ymask is not None:
        g = torch.where(ymask > 0, g, torch.zeros_like(g))
    gated = g
    if drop is not None:
        g = g * _per_image(drop, g.shape[0], pix_per_image)
    return g, gated


def bn_backward_sums(dy, x, mean, invstd, pix_per_image=1, ymask=None, drop=None):
    """s1 = sum g, s2 = sum g*xhat with xhat = (x - mean)*invstd, and the sums of magnitudes."""
    g, _ = bn_gated(dy, pix_per_image, ymask, drop)
    xhat = (x.to(F64) - mean.to(F64)) * invstd.to(F64)
    return g.sum(0), (g * xhat).sum(0), g.abs().sum(0), (g * xhat).abs().sum(0)


def bn_backward_dx(dy, x, mean, invstd, gamma, c1, c2, pix_per_image=1, ymask=None, drop=None):
    """dx = gamma*invstd*(g - c1 - xhat*c2), gated = dy*(ymask>0), T = magnitude for the gate."""
    g, gated = bn_gated(dy, pix_per_image, ymask, drop)
    xhat = (x.to(F64) - mean.to(F64)) * invstd.to(F64)
    k = gamma.to(F64) * invstd.to(F64)
    dx = k * (g - c1.to(F64) - xhat * c2.to(F64))
    T = k.abs() * (g.abs() + c1.to(F64).abs() + 2 * (xhat * c2.to(F64)).abs() + (mean.to(F64) * invstd.to(F64) * c2.to(F64)).abs())
    return dx, gated, T


def bn_terms_per_thread(npix, C, nblk):
    """Longest fp32 chain of the statistics kernels: a block takes ceil(npix / nblk) pixels and spreads them over
    256 / (C/4) pixel lanes; everything after the per-thread sums is fp64."""
    lanes = 256 // (C // 4)
    return -(-(-(-npix // nblk)) // lanes)


def bn_stat_bounds(x, T, eps):
    """Closed-form bounds on the forward statistics from the kernels' stated arithmetic: per-thread fp32 sums of at most
    T terms (sum x: T adds; sum x^2: T FMAs), fp64 afterwards, var = E[x^2] - mean^2, results rounded to fp32.
      |d mean|   <= (T+1) u E|x|
      |d var|    <= 3 (T+1) u E[x^2]        ((T+1) u E[x^2] from the second sum, 2|mean| |d mean| <= 2 (T+1) u E[x^2])
      |d invstd| <= invstd * (|d var| / (2 (var + eps)) + 2u)
    so relative to sigma^2 the variance error grows like 3 (T+1) u (1 + (mean/sigma)^2)."""
    x = x.to(F64)
    ex2 = (x * x).mean(0)
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    dmean = (T + 1) * U * x.abs().mean(0)
    dvar = 3 * (T + 1) * U * ex2
    rel_is = dvar / (2 * (var + eps)) + 2 * U
    return dmean, dvar, rel_is


def bn_envelope_ratio(T, tol=1e-4):
    """|mean|/sigma at which the bound above on the relative invstd error (hence on every normalised activation of O(1))
    reaches tol: 1.5 (T+1) u (1 + r^2) = tol."""
    return math.sqrt(max(tol / (1.5 * (T + 1) * U) - 1.0, 0.0))


# ---------------------------------------------------------------------------------------------------------------------
# 2x2 / stride-2 max pool into a channel slice
# ---------------------------------------------------------------------------------------------------------------------
_POOL_POS = ((0, 0), (0, 1), (1, 0), (1, 1))


def _pool_windows(inp, N, Hin, Win, C, in_cstride):
    n, oy, ox = pixels(N, Hin // 2, Win // 2, inp.device)
    return n, oy, ox, torch.stack([gather(inp, Hin, Win, in_cstride, 0, C, n, 2 * oy + a, 2 * ox + b) for a, b in _POOL_POS])


def maxpool2_fwd(inp, N, Hin, Win, C, in_cstride, out_cstride, out_coff, scale=None, shift=None):
    """-> (values [npix_out, C], flat output offsets).  scale / shift: the eval form relu(pool*scale[coff+c] + shift[coff+c])."""
    n, oy, ox, v = _pool_windows(inp, N, Hin, Win, C, in_cstride)
    m = v.max(0).values
    c = torch.arange(C, device=inp.device)
    if scale is not None:
        m = (m * scale.to(F64)[out_coff + c] + shift.to(F64)[out_coff + c]).clamp_min(0)
    off = (((n * (Hin // 2) + oy) * (Win // 2) + ox) * out_cstride + out_coff)[:, None] + c[None, :]
    return m, off


def maxpool2_bwd(inp, N, Hin, Win, C, in_cstride, d_out, out_cstride, out_coff, din_cstride, last_wins=False):
    """-> (gradient values [4, npix_out, C] for the four window positions, flat d_in offsets [4, npix_out, C]): the whole
    gradient goes to the first maximum in the order (0,0), (0,1), (1,0), (1,1) (last_wins: the mutation)."""
    n, oy, ox, v = _pool_windows(inp, N, Hin, Win, C, in_cstride)
    best, arg = v[0], torch.zeros_like(v[0], dtype=torch.long)
    for k in range(1, 4):
        better = (v[k] >= best) if last_wins else (v[k] > best)
        best, arg = torch.where(better, v[k], best), torch.where(better, torch.full_like(arg, k), arg)
    c = torch.arange(C, device=inp.device)
    g = d_out[(((n * (Hin // 2) + oy) * (Win // 2) + ox) * out_cstride + out_coff)[:, None] + c[None, :]].to(F64)
    vals = torch.stack([torch.where(arg == k, g, torch.zeros_like(g)) for k in range(4)])
    offs = torch.stack([(((n * Hin + 2 * oy + a) * Win + 2 * ox + b) * din_cstride)[:, None] + c[None, :] for a, b in _POOL_POS])
    return vals, offs


# ---------------------------------------------------------------------------------------------------------------------
# Decoder.output_conv: ConvTranspose2d(Cin -> L, 2, stride 2); x NHWC, out planar [N, L, 2H, 2W], w [Cin][L][2][2]
# ---------------------------------------------------------------------------------------------------------------------
def outconv_fwd(x, w, bias):
    """x [N,H,W,Cin], w [Cin,L,2,2], bias [L] or None -> (out [N,L,2H,2W], S)."""
    x, w = x.to(F64), w.to(F64)
    N, H, W, _ = x.shape
    L = w.shape[1]
    o = torch.einsum("njic,clab->nljaib", x, w).reshape(N, L, 2 * H, 2 * W)
    S = torch.einsum("njic,clab->nljaib", x.abs(), w.abs()).reshape(N, L, 2 * H, 2 * W)
    if bias is not None:
        o, S = o + bias.to(F64)[None, :, None, None], S + bias.to(F64).abs()[None, :, None, None]
    return o, S


def outconv_bwd_data(d_out, w):
    """d_out [N,L,2H,2W] -> (d_x [N,H,W,Cin], S)."""
    g, w = d_out.to(F64), w.to(F64)
    N, L, Ho, Wo = g.shape
    g = g.view(N, L, Ho // 2, 2, Wo // 2, 2)
    return torch.einsum("nljaib,clab->njic", g, w), torch.einsum("nljaib,clab->njic", g.abs(), w.abs())


def outconv_bwd_weight(x, d_out, p0=0, p1=None):
    """Pixels [p0, p1) of the N*H*W input pixels -> (dw [Cin,L,2,2], S, db [L], S of db)."""
    x, g = x.to(F64), d_out.to(F64)
    N, H, W, Cin = x.shape
    L = g.shape[1]
    xr = x.reshape(N * H * W, Cin)[p0:p1]
    gr = g.view(N, L, H, 2, W, 2).permute(0, 2, 4, 1, 3, 5).reshape(N * H * W, L, 2, 2)[p0:p1]
    return (torch.einsum("pc,plab->clab", xr, gr), torch.einsum("pc,plab->clab", xr.abs(), gr.abs()),
            gr.sum((0, 2, 3)), gr.abs().sum((0, 2, 3)))


# ---------------------------------------------------------------------------------------------------------------------
# lf_pack_gather
# ---------------------------------------------------------------------------------------------------------------------
PACK_INDEX_MASK, PACK_TF32_HI, PACK_TF32_LO = 0x1fffffff, 0x20000000, 0x40000000


def tf32_round(v):
    """fp32 -> the nearest value with the 13 low mantissa bits clear (ties away from zero: add half, truncate)."""
    b = v.contiguous().view(torch.int32).to(torch.int64) & 0xffffffff
    b = ((b + 0x1000) & 0xffffe000) & 0xffffffff
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b)
    return b.to(torch.int32).view(torch.float32)


def pack_gather(src, idx, bf16=False):
    """dst[k] = idx[k] >= 0 ? src[idx[k] & MASK] : 0; with the HI / LO flag the TF32 hi part of that value or the TF32
    rounding of value - hi (an exact fp32 difference); bf16: rounded to nearest even."""
    idx = idx.to(torch.int64)
    sel = torch.where(idx >= 0, idx & PACK_INDEX_MASK, torch.zeros_like(idx))
    v = torch.where(idx >= 0, src[sel], torch.zeros((), dtype=src.dtype, device=src.device))
    hi = tf32_round(v)
    lo = tf32_round(v - hi)
    v = torch.where((idx >= 0) & ((idx & PACK_TF32_HI) != 0), hi, torch.where((idx >= 0) & ((idx & PACK_TF32_LO) != 0), lo, v))
    return v.to(torch.bfloat16) if bf16 else v


# ---------------------------------------------------------------------------------------------------------------------
# shapes shared by the CPU and GPU tests
# ---------------------------------------------------------------------------------------------------------------------
def _plans():
    from lanedetection_end2end_b200 import net_plans
    return net_plans


def production_wgrads(N=2, H=256, W=512):
    """(name, plan, Hp, Wp, Cp, Hq, Wq, Cq, bias gradient requested) of every lf_wgrad_f32 call of a training step in fp32
    mode: ERFNet's trunk as ops_net hands it over (channels padded to 4) and the Classification heads' convolutions."""
    out = []
    for name, cin, cc, h, w in (("stem", 4, 16, H, W), ("down16_64", 16, 48, H // 2, W // 2), ("down64_128", 64, 64, H // 4, W // 4)):
        out.append((name, _plans().conv_wgrad_plan(h, w, 3, 3, 2, 1, 1, 1, 1), h, w, cin, h // 2, w // 2, cc, True))
    for name, ci, co, h, w in (("up128_64", 128, 64, H // 8, W // 8), ("up64_16", 64, 16, H // 4, W // 4)):
        out.append((name, _plans().convT_wgrad_plan(h, w, 3, 1), h, w, ci, 2 * h, 2 * w, co, False))
    for C, h, w, dils in ((64, H // 4, W // 4, (1,)), (128, H // 8, W // 8, (1, 2, 4, 8, 16)), (16, H // 2, W // 2, (1,))):
        for d in dils:
            out.append(("v3x1_c%d_d%d" % (C, d), _plans().conv_wgrad_plan(h, w, 3, 1, 1, d, 0, d, 1), h, w, C, h, w, C, True))
            out.append(("h1x3_c%d_d%d" % (C, d), _plans().conv_wgrad_plan(h, w, 1, 3, 1, 0, d, 1, d), h, w, C, h, w, C, True))
    h, w = H // 8, W // 8
    out.append(("head_conv1", _plans().conv_wgrad_plan(h, w, 1, 1, 1, 0, 0, 1, 1), h, w, 128, h, w, 128, True))
    for name, ci, co in (("head_conv2", 128, 128), ("head_conv3", 128, 64), ("head_conv4", 64, 64)):
        out.append((name, _plans().conv_wgrad_plan(h, w, 3, 3, 1, 1, 1, 1, 1), h, w, ci, h, w, co, True))
    return out


# one shape per branch of the plan: (Cp, Cq, ntaps, gathered side, bias gradient) -> expectation
PLAN_BRANCHES = [
    ((4, 16, 9, "p", True), dict(taps_on_p=True, G=28)),                 # stem: G >= 8, 4-pixel steps
    ((16, 48, 9, "p", True), dict(taps_on_p=True, G=2)),                 # G in 2..7
    ((64, 16, 9, "q", False), dict(taps_on_p=False, G=1)),               # taps on Q, one group
    ((16, 16, 3, "p", True), dict(taps_on_p=True, G=21)),
    ((16, 16, 1, "p", True), dict(taps_on_p=True, G=64)),                # one tap counts as taps on P
    ((64, 16, 9, "q", True), "taps_on_q_qsum_or_cq"), ((16, 12, 9, "q", False), "taps_on_q_qsum_or_cq"),
    ((64, 64, 9, "p", True), "wide"), ((16, 16, 3, "none", True), "both_or_neither_gathered"),
    ((16, 12, 3, "p", True), "lu_lv_granularity"), ((128, 16, 9, "p", True), "too_many_threads"),
]


def branch_spec(key):
    Cp, Cq, nt, side, _ = key
    taps = [(a - 1, b - 1) for a in range(3) for b in range(3)][:nt] if nt > 1 else [(0, 0)]
    zero = [(0, 0)] * nt
    plan = dict(Hs=12, Ws=20, psy=1, psx=1, qsy=1, qsx=1, ptaps=taps if side == "p" else zero, qtaps=taps if side == "q" else zero)
    return wgrad_spec(2, plan, 12, 20, Cp, 12, 20, Cq)
