"""The contract of the 3-tap tensor-core convolution (lf_conv1d_tc, lf_conv1d_tc_x3, lf_conv1d_tc_bf16,
lf_conv1d_tc_fp8 in csrc/conv_tc.cu) restated in fp64, and the per-entry gate its results are held to.

* Operands, bit for bit as the kernel feeds the tensor core (quantisers from tcg_contract.py):
    - TF32: activations tf32_rna (the kernel rounds each slab in shared memory); the weights are read from `wpack` as
      their fp32 bits, which wgmma .tf32 truncates (tf32_trunc; the ties class of the GPU tests pins it);
    - 3xTF32: the activations split hi = tf32_rna(a), lo = tf32_rna(a - hi); the weights pre-split by the packer
      (ops_net.split_tf32); the products hi*hi + hi*lo + lo*hi, lo*lo dropped;
    - BF16: bf16_rne on both operands (a bf16 `in` is already exact);
    - FP8: a_q = e4m3_rne_satfinite(fl32(x * fl32(448 / x_amax[n]))) per image n (0 where x_amax[n] = 0); the weights
      are the e4m3 bytes of `wpack` as given (pack_weights quantises each output channel co with w_scale[co]).  The
      exact sums are dequantised with dq[n, co] = fl32(fl32(x_amax[n] / 448) * w_scale[co]), the factor the kernel
      forms: ref = dq * sum a_q w_q, S = dq * sum |a_q w_q|.
* The reference: out[n,y,x,co] = sum_t sum_ci a_q[n, (y,x) + tap_t, ci] * w_q[co, t*C + ci] and S = sum |a_q w_q| per
  entry, in fp64 (products of quantised operands are exact there), zero outside the image.  Taps are any three (dy, dx):
  {-d, 0, +d} for the forward, {+d, 0, -d} for the input gradient, anything on the per-tap plan.
* The epilogue, in the kernel's order: + bias, ReLU (relu bit 0), mask_src > 0 or the affine mask fma(x, scale, shift) > 0
  (exact in fp64: x * scale has at most 48 significant bits, and one rounding keeps the sign), + add_src (gated by
  add_mask > 0), ReLU (relu bit 1).  ReLU and the masks do not widen an error (ReLU is 1-Lipschitz, the masks are exact),
  so the gate needs no special case where a pre-ReLU value is within it of zero.
* The gate: |got - ref| <= (c_tc + steps * 2^-23) * S' per entry, S' = S + |bias| + |add_src|, steps = 3 * C / 32 (one
  rounded FADD per tap and 32-channel chunk: each is summed from zero on the tensor core and added to the running fp32
  sum), + 1 for the 3xTF32 acs + acc or the FP8 dequantising multiply, + 1 per epilogue add.  c_tc covers the tensor
  core's in-instruction accumulation (and for 3xTF32 the correction terms, which it accumulates over all taps and
  chunks).
* FP8 out_amax: out_amax[n] is exactly the max |stored value| of image n (of the bf16 values for a bf16 `out`); an
  image whose stored outputs are all zero leaves its zero-initialised entry untouched.
* Per-CTA partials: row r of colsum_partial / stats_partial is the sum over the tiles m = r, r + m_ctas, ... of the
  kernel's stored (fp32) output: the sum, and the sum of squares or (affine mask) of out * x.  Each thread of the
  epilogue adds 8 rows per tile in one fp32 chain, and the 16 chains of a column are combined in fp64: chains of
  8 x tiles per CTA.  The tile map comes from lf_conv1d_tc_plan (TA, TB, vertical, m_ctas).
"""
import torch

from oracle import fp8_oracle
from tcg_contract import (C_TC_CEILING as _TCG_CEILING, LF_BF16, LF_F32, TC_BF16, TC_TF32, TC_X3, ULP,  # noqa: F401
                          bf16_rna, bf16_rne, gate_excess, rel_err, split_tf32, tc_usage, tf32_rna, tf32_rne, tf32_trunc,
                          with_low_bits)

TC_FP8 = 3                                 # lf_conv1d_tc_plan's precision of lf_conv1d_tc_fp8
KCH = 32                                   # channels per chunk (one 128-byte swizzle row of fp32)
TILE = 128                                 # pixels per tile
E4M3_MIN_NORMAL = 2.0 ** -6
# c_tc per precision (0 = TF32, 1 = 3xTF32, 2 = BF16, 3 = FP8).  Ceilings as for the tcg kernels
# (tcg_contract.C_TC_CEILING): well below the half-step of the operand rounding, so that the rounding mutations keep
# breaking the gate.  FP8: the H100's e4m3 wgmma sums the 32 products of one k32 step with fewer mantissa bits than fp32,
# aligned to the group's largest product.  Measured on an H100 80GB HBM3 (700 W): about 2^-15.4 of the sum of |products|
# on Gaussian activations, but up to 2^-10.1 over the FP8 cases of tests/test_conv_tc_contract_gpu.py, from the
# heavy-tailed ones, where one product dominates each group and the other 31 lose their low bits against it (the same
# error with activations that are e4m3 values already, x_amax = 448 and inv = 1: none of it is quantisation).  2^-9
# keeps 2.1x headroom over that; the ceiling 2^-8 stays 8x below e4m3's smallest relative half-step (2^-5).
C_TC = {TC_TF32: 2.0 ** -21, TC_X3: 2.0 ** -21, TC_BF16: 2.0 ** -21, TC_FP8: 2.0 ** -9}
C_TC_CEILING = {**_TCG_CEILING, TC_FP8: 2.0 ** -8}
PREC_NAMES = {TC_TF32: "tf32", TC_X3: "tf32x3", TC_BF16: "bf16", TC_FP8: "fp8"}
ENTRIES = {TC_TF32: "lf_conv1d_tc", TC_X3: "lf_conv1d_tc_x3", TC_BF16: "lf_conv1d_tc_bf16", TC_FP8: "lf_conv1d_tc_fp8"}


def tap_list(vertical, dil, transposed=False):
    """[(dy, dx)] * 3 in weight-slot order: {-d, 0, +d} (forward) or {+d, 0, -d} (input gradient) along one axis."""
    sgn = -1 if transposed else 1
    return [((sgn * (t - 1) * dil, 0) if vertical else (0, sgn * (t - 1) * dil)) for t in range(3)]


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def e4m3_rne(v):
    """cvt.rn.satfinite.e4m3x2.f32: round fp32 to e4m3 (nearest even, subnormals kept), saturated to +-448; as fp32."""
    return fp8_oracle.e4m3(v)


def e4m3_ftz(v):
    """e4m3 rounding with the subnormal results flushed to zero (NOT what the kernel does: a sensitivity check)."""
    q = e4m3_rne(v)
    return torch.where(q.abs() < E4M3_MIN_NORMAL, torch.zeros_like(q), q)


def e4m3_rtz(v):
    """e4m3 rounding toward zero (NOT what the kernel does: a sensitivity check): the nearest value, one code lower in
    magnitude wherever that rounded away from zero."""
    q = e4m3_rne(v)
    b = q.to(torch.float8_e4m3fn).view(torch.uint8)
    down = (b.to(torch.int16) - 1).clamp_min(0).to(torch.uint8).view(torch.float8_e4m3fn).float()
    return torch.where((q.abs() > v.abs()) & (q != 0), down, q)


def fp8_inv(x_amax):
    """[N] fp32: 448 / x_amax[n], IEEE division as the kernel's __fdiv_rn, 0 where x_amax[n] = 0."""
    return fp8_oracle.inverse_scale(x_amax.float())


def fp8_dq(x_amax, w_scale):
    """[N, C] fp32: the dequantisation factors fl32(fl32(x_amax[n] / 448) * w_scale[co])."""
    return fp8_oracle.scale(x_amax.float()).view(-1, 1) * w_scale.float().view(1, -1)


def act_terms(x, prec, rounding=None, x_amax=None):
    """The activation operand(s) the tensor core multiplies, fp64: [a_q] or, for 3xTF32, [a_hi, a_lo].
    rounding: override the kernel's rounding (the sensitivity checks).  FP8: x_amax [N] is the per-image scale."""
    x = x.float()
    if prec == TC_FP8:
        v = x * fp8_inv(x_amax).view(-1, 1, 1, 1)          # one fp32 multiply, rounded to nearest
        return [(rounding or e4m3_rne)(v).double()]
    if prec == TC_X3:
        hi = (rounding or tf32_rna)(x)
        return [hi.double(), tf32_rna(x - hi).double()]
    if rounding is None:
        rounding = tf32_rna if prec == TC_TF32 else bf16_rne
    return [rounding(x).double()]


def weight_terms(wpack, prec, rounding=None):
    """The weight operand(s) [C][3C] as the tensor core reads `wpack`, fp64: TF32 truncation of the fp32 bits, the
    pre-split pair [w_hi, w_lo] of a [2][C][3C] 3xTF32 operand, or the bf16 values."""
    if prec == TC_X3:
        return [wpack[0].double(), wpack[1].double()]
    if prec == TC_BF16:
        return [wpack.double()]
    if prec == TC_FP8:
        return [wpack.view(torch.float8_e4m3fn).double()]
    return [(rounding or tf32_trunc)(wpack).double()]


def fp8_weight_scale(w):
    """[C] fp32 w_scale of the FP8 operand of the [C][3C] slot matrix w: max |w[co]| / 448."""
    return fp8_oracle.scale(w.float().abs().amax(1))


def pack_weights(w, prec):
    """The packed operand ([C][3C] fp32) in the form the entry point takes.  FP8: [C][3C] uint8 holding the e4m3 bytes
    of w[co] * (448 / max |w[co]|), each output channel quantised on its own (its w_scale: fp8_weight_scale)."""
    if prec == TC_FP8:
        wf = w.float()
        q = e4m3_rne(wf * fp8_oracle.inverse_scale(wf.abs().amax(1)).view(-1, 1))
        return q.to(torch.float8_e4m3fn).view(torch.uint8).contiguous()
    if prec == TC_X3:
        hi, lo = split_tf32(w)
        return torch.stack([hi, lo]).contiguous()
    if prec == TC_BF16:
        return w.to(torch.bfloat16).contiguous()
    return w.float().contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def shifted(a, dy, dx):
    """b[n, y, x] = a[n, y + dy, x + dx], zero outside the image (TMA's out-of-bounds fill)."""
    N, H, W, C = a.shape
    out = torch.zeros_like(a)
    y0, y1, x0, x1 = max(0, -dy), min(H, H - dy), max(0, -dx), min(W, W - dx)
    if y0 < y1 and x0 < x1:
        out[:, y0:y1, x0:x1] = a[:, y0 + dy:y1 + dy, x0 + dx:x1 + dx]
    return out


def _tap_operand(a, t, taps, C, mut):
    dy, dx = taps[t]
    if mut.get("shift_tap") == t:                        # the tap read one pixel off along x
        dx += 1
    s = shifted(a, dy, dx)
    if mut.get("halo_zero") is not None and mut["halo_zero"][0] == t:
        # rows of the tap's view that lie before the destination's tile along the conv axis (inside the image) read as 0
        _, TA, vertical = mut["halo_zero"]
        N, H, W, _ = a.shape
        off = dy if vertical else dx
        p = torch.arange(H if vertical else W, device=a.device)
        src = p + off
        bad = (src >= 0) & (src < p.numel()) & (torch.div(src, TA, rounding_mode="floor") < torch.div(p, TA, rounding_mode="floor"))
        s = s * (~bad).to(s.dtype).view((1, -1, 1, 1) if vertical else (1, 1, -1, 1))
    if mut.get("drop_chunk") is not None and mut["drop_chunk"][0] == t:
        cb = mut["drop_chunk"][1]
        s[..., cb * KCH:(cb + 1) * KCH] = 0
    return s.reshape(-1, C)


def conv_fp64(x, wpack, prec, taps, a_round=None, w_round=None, scales=None, **mut):
    """(ref, S) [N*H*W, C] in fp64 of the bare convolution (no epilogue), from the quantised operands; FP8: dequantised,
    scales = (x_amax [N], w_scale [C]).
    Mutations (sensitivity checks): shift_tap = t; drop_chunk = (t, cb); halo_zero = (t, TA, vertical);
    drop_lo_hi (3xTF32: a_lo * w_hi dropped); a_round / w_round: other operand roundings; next_image_scale (FP8: image n
    quantised and dequantised with image n+1's x_amax, the last with image 0's)."""
    N, H, W, C = x.shape
    x_amax = None
    if prec == TC_FP8:
        x_amax, w_scale = scales
        if mut.get("next_image_scale"):
            x_amax = x_amax.roll(-1)
    A = act_terms(x, prec, a_round, x_amax)
    Wt = weight_terms(wpack, prec, w_round)
    if prec == TC_X3:
        pairs = [(0, 0), (0, 1)] + ([] if mut.get("drop_lo_hi") else [(1, 0)])
    else:
        pairs = [(0, 0)]
    ref = torch.zeros(N * H * W, C, dtype=torch.float64, device=x.device)
    S = torch.zeros_like(ref)
    for t in range(3):
        views = [_tap_operand(a, t, taps, C, mut) for a in A]
        for i, j in pairs:
            w = Wt[j][:, t * C:(t + 1) * C]
            ref += views[i] @ w.t()
            S += views[i].abs() @ w.abs().t()
    if prec == TC_FP8:
        dq = per_pixel(fp8_dq(x_amax, w_scale).double(), H * W)
        ref, S = ref * dq, S * dq
    return ref, S


def per_pixel(t, pixels_per_image):
    """[N, ...] -> [N * pixels_per_image, ...]: each image's row repeated for its pixels (NHW order)."""
    return t.repeat_interleave(pixels_per_image, 0)


def image_amax(out, N):
    """[N] fp32: the per-image max |stored value| FP8 reduces into out_amax (0 for an all-zero image)."""
    return out.float().abs().reshape(N, -1).amax(1)


def epilogue(z, S, bias=None, relu=0, mask_src=None, mask_affine=None, add_src=None, add_mask=None):
    """(out, S', adds): the kernel's epilogue applied in fp64 to the convolution z [P, C], the gate's magnitude S' and
    the number of rounded epilogue adds.  Tensors in NHWC (any float dtype)."""
    C = z.shape[1]
    v, Sp, adds = z, S, 0
    if bias is not None:
        b = bias.double().view(1, C)
        v, Sp, adds = v + b, Sp + b.abs(), adds + 1
    if relu & 1:
        v = v.clamp_min(0)
    if mask_src is not None:
        m = mask_src.double().reshape(-1, C)
        if mask_affine is not None:
            m = m * mask_affine[0].double().view(1, C) + mask_affine[1].double().view(1, C)
        v = torch.where(m > 0, v, torch.zeros_like(v))
    if add_src is not None:
        a = add_src.double().reshape(-1, C)
        if add_mask is not None:
            a = torch.where(add_mask.double().reshape(-1, C) > 0, a, torch.zeros_like(a))
        v, Sp, adds = v + a, Sp + a.abs(), adds + 1
    if relu & 2:
        v = v.clamp_min(0)
    return v, Sp, adds


def steps(C, prec, adds):
    """Rounded fp32 operations per output entry beyond the tensor core's own: one add per tap and chunk, the 3xTF32
    acs + acc or the FP8 dequantising multiply, and the epilogue's adds."""
    return 3 * C // KCH + (1 if prec in (TC_X3, TC_FP8) else 0) + adds


def excess(got, ref, S, nsteps, prec, c_tc=None):
    """max |got - ref| / gate over the entries (<= 1 passes)."""
    return gate_excess(got, ref, S, nsteps, prec, C_TC[prec] if c_tc is None else c_tc)


# ---------------------------------------------------------------------------------------------------------------------
# per-CTA partials
# ---------------------------------------------------------------------------------------------------------------------
def tile_map(N, H, W, plan, device=None):
    """(cta row, k = the tile's place in that CTA's sequence, r = row in the tile) of every pixel in NHW order:
    tile m = (n * tiles_b + tb) * tiles_a + ta runs on CTA row m % m_ctas as its (m // m_ctas)-th tile; row
    r = (position along the axis in the tile) * TB + (position across)."""
    TA, TB, vert, m = plan["TA"], plan["TB"], plan["vertical"], plan["m_ctas"]
    n, y, x = torch.meshgrid(torch.arange(N, device=device), torch.arange(H, device=device), torch.arange(W, device=device),
                             indexing="ij")
    pa, pb = (y, x) if vert else (x, y)
    tiles_a, tiles_b = (H if vert else W) // TA, (W if vert else H) // TB
    mt = (n * tiles_b + pb // TB) * tiles_a + pa // TA
    r = (pa % TA) * TB + pb % TB
    return (mt % m).reshape(-1), (mt // m).reshape(-1), r.reshape(-1)


def tiles_per_cta(N, H, W, plan):
    total = N * H * W // TILE
    return (total + plan["m_ctas"] - 1) // plan["m_ctas"]


def partial_fp64(vals, rows, m_ctas):
    """[m_ctas, C] fp64 sums of vals [P, C] over the pixels of each CTA row."""
    out = torch.zeros(m_ctas, vals.shape[1], dtype=torch.float64, device=vals.device)
    return out.index_add_(0, rows, vals.double())


def partial_steps(N, H, W, plan):
    """fp32 adds in the chain of one partial entry: 8 rows per tile and tile, + 1 for the final rounding."""
    return 8 * tiles_per_cta(N, H, W, plan) + 1


# ---------------------------------------------------------------------------------------------------------------------
# a kernel-faithful fp32 emulation (the CPU tests hold it to the gate)
# ---------------------------------------------------------------------------------------------------------------------
def emulate(x, wpack, prec, taps, plan, bias=None, relu=0, mask_src=None, mask_affine=None, add_src=None, add_mask=None,
            scales=None):
    """(out [P, C] fp32, colsum [m_ctas, C] fp32, stats [m_ctas, 2, C] fp64) as the kernel forms them: each tap and
    32-channel chunk summed from zero (here exactly, then rounded to fp32), added to the fp32 sum with a rounded add;
    3xTF32's correction terms summed apart and added last; FP8's sum times its fp32 dequantisation factor, rounded; the
    epilogue in fp32; the partials as fp32 chains of 8 rows per tile, the 16 chains of a column combined in fp64 (FP8
    takes no partials: its out_amax is image_amax(out))."""
    N, H, W, C = x.shape
    A = act_terms(x, prec, x_amax=scales[0] if prec == TC_FP8 else None)
    Wt = weight_terms(wpack, prec)
    P = N * H * W
    acc = torch.zeros(P, C, dtype=torch.float32, device=x.device)
    small = torch.zeros(P, C, dtype=torch.float64, device=x.device)
    for cb in range(C // KCH):
        for t in range(3):
            ch = slice(cb * KCH, (cb + 1) * KCH)
            views = [shifted(a, *taps[t])[..., ch].reshape(-1, KCH) for a in A]
            wcols = [w[:, t * C + cb * KCH:t * C + (cb + 1) * KCH] for w in Wt]
            acc = acc + (views[0] @ wcols[0].t()).float()
            if prec == TC_X3:
                small += views[0] @ wcols[1].t() + views[1] @ wcols[0].t()
    o = small.float() + acc if prec == TC_X3 else acc
    if prec == TC_FP8:
        o = o * per_pixel(fp8_dq(*scales), H * W)
    if bias is not None:
        o = o + bias.float().view(1, C)
    if relu & 1:
        o = o.clamp_min(0)
    if mask_src is not None:
        m = mask_src.double().reshape(-1, C)
        if mask_affine is not None:
            m = m * mask_affine[0].double().view(1, C) + mask_affine[1].double().view(1, C)
        o = torch.where(m > 0, o, torch.zeros_like(o))
    if add_src is not None:
        a = add_src.float().reshape(-1, C)
        if add_mask is not None:
            a = torch.where(add_mask.reshape(-1, C) > 0, a, torch.zeros_like(a))
        o = o + a
    if relu & 2:
        o = o.clamp_min(0)
    od = o.double()
    prod = od * (mask_src.double().reshape(-1, C) if mask_affine is not None else od)   # exact in fp64, as inside the fma
    rows, k, r = tile_map(N, H, W, plan, x.device)
    m, tpc = plan["m_ctas"], tiles_per_cta(N, H, W, plan)
    sums = []
    for v in (od, prod):
        # chain (cta, r0 = r % 16, channel) runs over (k, j = r // 16)
        E = torch.zeros(m, tpc, 8, 16, C, dtype=torch.float64, device=x.device)
        E[rows, k, r // 16, r % 16] = v
        s = torch.zeros(m, 16, C, dtype=torch.float32, device=x.device)
        for kk in range(tpc):
            for j in range(8):
                s = (s.double() + E[:, kk, j]).float()
        sums.append(s.double().sum(1))
    return o, sums[0].float(), torch.stack(sums, 1)


# ---------------------------------------------------------------------------------------------------------------------
# the plan query
# ---------------------------------------------------------------------------------------------------------------------
def query_plan(prec, in_dtype, N, H, W, C, taps):
    """(rc, plan dict or None) of lf_conv1d_tc_plan: what the entry point of precision prec launches (or refuses) for
    these arguments under the variant set now."""
    import ctypes
    from lanedetection_end2end_b200 import _capi
    dy = (ctypes.c_int * 3)(*[t[0] for t in taps])
    dx = (ctypes.c_int * 3)(*[t[1] for t in taps])
    info = (ctypes.c_int * _capi.TC_PLAN_INFO)()
    rc = _capi.lib().lf_conv1d_tc_plan(prec, in_dtype, N, H, W, C, dy, dx, info)
    return rc, (dict(zip(_capi.TC_PLAN_FIELDS, list(info))) if rc == 0 else None)


def plan_key(prec, in_dtype, C, plan):
    """The kernel instantiation and shared-memory plan a launch reached: (C, precision, bf16 input, resident weights,
    slab, 3xTF32 lo plan, single stage).  lo plan: "2" / "1" buffers after the ring, "stg" over the staging tile,
    "stg+" over it and reaching back before it; "-" for TF32 / BF16 / FP8."""
    lo = "-"
    if prec == TC_X3:
        lo = ("stg+" if plan["lo_bytes"] else "stg") if plan["lo_stg"] else str(plan["n_lo"])
    return (C, PREC_NAMES[prec], bool(in_dtype == LF_BF16), bool(plan["res"]), bool(plan["slab"]), lo, plan["stages"] == 1)


# ---------------------------------------------------------------------------------------------------------------------
# coverage: one launch per planner outcome
# ---------------------------------------------------------------------------------------------------------------------
# The shapes the planner is asked about: extents, dilations (up to beyond every extent) and both variants.
UNIVERSE_EXTENTS = (4, 8, 16, 32, 40, 64, 80, 128, 160, 256)
UNIVERSE_DILS = tuple(range(1, 33)) + (40, 48, 64, 80, 100, 124, 127, 128)

# (precision, bf16 input, C, H, W, vertical, dilation, variant) -> the plan_key it reaches
COVERAGE = [
    ((TC_TF32, False, 128, 32, 4, True, 1, 2), (128, "tf32", False, False, False, "-", False)),
    ((TC_TF32, False, 128, 32, 40, False, 8, 2), (128, "tf32", False, False, True, "-", False)),
    ((TC_TF32, False, 128, 32, 40, False, 14, 2), (128, "tf32", False, False, True, "-", True)),
    ((TC_TF32, False, 128, 32, 32, True, 1, 2), (128, "tf32", False, True, True, "-", False)),
    ((TC_TF32, False, 128, 32, 64, True, 2, 1), (128, "tf32", False, False, False, "-", False)),
    ((TC_TF32, False, 64, 32, 40, False, 14, 2), (64, "tf32", False, False, True, "-", True)),
    ((TC_TF32, False, 64, 32, 4, True, 1, 2), (64, "tf32", False, True, False, "-", False)),
    ((TC_TF32, False, 64, 32, 32, True, 1, 2), (64, "tf32", False, True, True, "-", False)),
    ((TC_TF32, False, 64, 64, 128, False, 1, 1), (64, "tf32", False, True, False, "-", False)),
    ((TC_BF16, False, 128, 32, 40, False, 14, 2), (128, "bf16", False, False, True, "-", False)),
    ((TC_BF16, False, 128, 32, 40, False, 17, 2), (128, "bf16", False, False, True, "-", True)),
    ((TC_BF16, False, 128, 32, 4, True, 1, 2), (128, "bf16", False, True, False, "-", False)),
    ((TC_BF16, False, 128, 32, 32, True, 1, 2), (128, "bf16", False, True, True, "-", False)),
    ((TC_BF16, False, 64, 32, 40, False, 17, 2), (64, "bf16", False, False, True, "-", True)),
    ((TC_BF16, False, 64, 32, 4, True, 1, 2), (64, "bf16", False, True, False, "-", False)),
    ((TC_BF16, False, 64, 32, 32, True, 1, 2), (64, "bf16", False, True, True, "-", False)),
    ((TC_BF16, True, 128, 32, 40, False, 32, 2), (128, "bf16", True, False, True, "-", False)),
    ((TC_BF16, True, 128, 32, 4, True, 1, 2), (128, "bf16", True, True, False, "-", False)),
    ((TC_BF16, True, 128, 32, 32, True, 1, 2), (128, "bf16", True, True, True, "-", False)),
    ((TC_BF16, True, 128, 32, 64, False, 4, 1), (128, "bf16", True, True, False, "-", False)),
    ((TC_BF16, True, 64, 32, 4, True, 1, 2), (64, "bf16", True, True, False, "-", False)),
    ((TC_BF16, True, 64, 32, 32, True, 1, 2), (64, "bf16", True, True, True, "-", False)),
    ((TC_X3, False, 128, 32, 40, False, 2, 2), (128, "tf32x3", False, False, True, "1", False)),
    ((TC_X3, False, 128, 32, 32, True, 1, 2), (128, "tf32x3", False, False, True, "2", False)),
    ((TC_X3, False, 128, 32, 40, False, 4, 2), (128, "tf32x3", False, False, True, "stg", False)),
    ((TC_X3, False, 128, 32, 40, False, 6, 2), (128, "tf32x3", False, False, True, "stg+", False)),
    ((TC_X3, False, 128, 32, 40, False, 7, 2), (128, "tf32x3", False, False, True, "stg+", True)),
    ((TC_X3, False, 128, 32, 64, True, 1, 1), (128, "tf32x3", False, False, True, "2", False)),
    ((TC_X3, False, 64, 32, 40, False, 8, 2), (64, "tf32x3", False, False, True, "stg+", True)),
    ((TC_X3, False, 64, 32, 40, False, 2, 2), (64, "tf32x3", False, True, True, "1", False)),
    ((TC_X3, False, 64, 32, 32, True, 1, 2), (64, "tf32x3", False, True, True, "2", False)),
    ((TC_X3, False, 64, 32, 40, False, 4, 2), (64, "tf32x3", False, True, True, "stg", False)),
    ((TC_X3, False, 64, 32, 40, False, 6, 2), (64, "tf32x3", False, True, True, "stg+", False)),
    ((TC_X3, False, 64, 32, 40, False, 7, 2), (64, "tf32x3", False, True, True, "stg+", True)),
    ((TC_FP8, False, 128, 40, 160, True, 17, 2), (128, "fp8", False, False, True, "-", False)),
    ((TC_FP8, False, 128, 32, 256, True, 80, 2), (128, "fp8", False, False, True, "-", True)),
    ((TC_FP8, False, 128, 32, 4, True, 1, 2), (128, "fp8", False, True, False, "-", False)),
    ((TC_FP8, False, 128, 32, 64, True, 1, 2), (128, "fp8", False, True, True, "-", False)),
    ((TC_FP8, True, 128, 32, 64, False, 4, 1), (128, "fp8", True, True, False, "-", False)),
    ((TC_FP8, True, 128, 40, 80, True, 2, 2), (128, "fp8", True, True, True, "-", False)),
    ((TC_FP8, False, 64, 32, 256, True, 80, 2), (64, "fp8", False, False, True, "-", True)),
    ((TC_FP8, False, 64, 64, 128, False, 1, 1), (64, "fp8", False, True, False, "-", False)),
    ((TC_FP8, False, 64, 64, 128, True, 1, 2), (64, "fp8", False, True, True, "-", False)),
    ((TC_FP8, True, 64, 32, 4, True, 1, 2), (64, "fp8", True, True, False, "-", False)),
    ((TC_FP8, True, 64, 32, 32, True, 1, 2), (64, "fp8", True, True, True, "-", False)),
]


def with_variant(variant, fn):
    """fn() with lf_conv1d_tc_set_variant(variant) in force (process-wide), the default (2) restored after."""
    from lanedetection_end2end_b200 import _capi
    _capi.lib().lf_conv1d_tc_set_variant(variant)
    try:
        return fn()
    finally:
        _capi.lib().lf_conv1d_tc_set_variant(2)


def universe_keys():
    """{plan_key: first (prec, bf16 in, C, H, W, vertical, dil, variant) reaching it} over the universe of shapes."""
    found = {}
    for variant in (2, 1):
        def scan():
            for prec in (TC_TF32, TC_X3, TC_BF16, TC_FP8):
                for abf in ((False, True) if prec in (TC_BF16, TC_FP8) else (False,)):
                    for C in (64, 128):
                        for H in UNIVERSE_EXTENTS:
                            for W in UNIVERSE_EXTENTS:
                                for v in (True, False):
                                    for d in UNIVERSE_DILS:
                                        rc, pl = query_plan(prec, LF_BF16 if abf else LF_F32, 2, H, W, C, tap_list(v, d))
                                        if rc == 0:
                                            found.setdefault(plan_key(prec, LF_BF16 if abf else LF_F32, C, pl),
                                                             (prec, abf, C, H, W, v, d, variant))
        with_variant(variant, scan)
    return found
