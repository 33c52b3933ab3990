"""The contracts of the two run-time-table tensor-core kernels, lf_conv_tcg (csrc/conv_tcg.cu) and lf_wgrad_tcg
(csrc/wgrad_tcg.cu), restated in fp64, and the per-entry gate their results are held to.

* emulate_*: literal CPU restatements of lf_conv_tcg / lf_wgrad_tcg / lf_wgrad_reduce on the exact views and strides the
  host code put into the args structs (tests/test_net_plans.py runs the host code against them).
* Operand quantisers, bit for bit as the kernels apply them:
    - tf32_rna: round to nearest, ties away, low 13 mantissa bits cleared (tc_ptx.cuh tf32_rna).  wgrad_tcg.cu applies it
      to both operands, conv_tcg.cu to the activations;
    - split_tf32: the 3xTF32 pair hi = tf32_rna(v), lo = tf32_rna(v - hi) (== ops_net.split_tf32);
    - bf16_rne: cvt.rn.bf16x2.f32, round to nearest even (== torch's .to(torch.bfloat16));
    - tf32_trunc: what wgmma .tf32 does with an fp32 bit pattern it reads from shared memory as is (the lf_conv_tcg TF32
      weights, which the host does not round): the PTX ISA defines a .tf32 element as the upper 19 bits of the 32-bit
      container, so the low 13 mantissa bits are ignored -- truncation toward zero.  The GPU tests confirm it with
      weights whose low bits are exactly half a TF32 step, where truncation and rounding differ.
* The reference is formed from the quantised operands: ref = sum a_q * b_q in fp64, and S = sum |a_q * b_q| per output
  entry.  Products of quantised operands are exact in fp64, so ref - got is only the kernel's fp32 accumulation.
* gate(): |got - ref| <= (c_tc + steps * 2^-23) * S per entry, with steps = the FADDs the kernel spends on that entry
  (patches or k-steps per CTA, plus the partials reduced).  c_tc covers the tensor core's in-instruction accumulation,
  which does not round like IEEE adds (NOTES.md), and for 3xTF32 the dropped lo * lo term.
"""
import torch

# c_tc per LfWgradTcgArgs / LfConvTcgArgs precision (0 = TF32, 1 = 3xTF32, 2 = BF16).  On an H100 80GB HBM3 (700 W) the
# largest (|got - ref| - steps * 2^-23 * S) / S over tests/test_tcg_kernels_gpu.py was 9.8e-8 for TF32 and 1.6e-7 for
# 3xTF32 (both from lf_conv_tcg launches of 1-3 k-steps, where the FADD term is small); no BF16 entry needed any c_tc.
# The constants keep >= 4x headroom over that.  Ceilings: 2^-16 for TF32 and BF16, 2^-18 for 3xTF32.
C_TC = {0: 2.0 ** -21, 1: 2.0 ** -20, 2: 2.0 ** -21}
C_TC_CEILING = {0: 2.0 ** -16, 1: 2.0 ** -18, 2: 2.0 ** -16}
ULP = 2.0 ** -23

LF_F32, LF_BF16 = 0, 1
TC_TF32, TC_X3, TC_BF16 = 0, 1, 2
WGT_KP = 32          # pixels per lf_wgrad_tcg patch (one pipeline stage)
TG_BM = 128          # pixels per lf_conv_tcg tile


# ---------------------------------------------------------------------------------------------------------------------
# quantisers (fp32 in, fp32 out, bit for bit what the kernels feed the tensor core)
# ---------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.float().contiguous().view(torch.int32)


def tf32_rna(t):
    """Round to nearest TF32, ties away from zero, low 13 mantissa bits cleared (tc_ptx.cuh tf32_rna)."""
    return ((_bits(t) + 0x1000) & -8192).view(torch.float32)


def tf32_rne(t):
    """Round to nearest TF32, ties to even (NOT what the kernels do: the sensitivity checks use it)."""
    b = _bits(t)
    return ((b + 0x0fff + ((b >> 13) & 1)) & -8192).view(torch.float32)


def tf32_trunc(t):
    """The low 13 mantissa bits dropped: how wgmma .tf32 reads an fp32 bit pattern."""
    return (_bits(t) & -8192).view(torch.float32)


def split_tf32(t):
    """(hi, lo) of the 3xTF32 split: hi = tf32_rna(t), lo = tf32_rna(t - hi)."""
    t = t.float()
    hi = tf32_rna(t)
    return hi, tf32_rna(t - hi)


def bf16_rne(t):
    """cvt.rn.bf16.f32 (round to nearest even), as fp32; integer restatement of torch's bf16 cast for finite values."""
    b = _bits(t)
    return ((b + 0x7fff + ((b >> 16) & 1)) & -65536).view(torch.float32)


def bf16_rna(t):
    """bf16 rounding with ties away from zero (NOT what the kernels do: the sensitivity checks use it)."""
    return ((_bits(t) + 0x8000) & -65536).view(torch.float32)


def quantise(t, prec, rounding=None):
    """fp64 value the tensor core multiplies for an fp32 operand t at LfWgradTcgArgs precision prec: TF32 (RNA), the
    3xTF32 pair hi + lo, or bf16 (RNE).  rounding: override the TF32 / bf16 rounding (the sensitivity checks)."""
    if prec == TC_X3:
        hi, lo = split_tf32(t)
        return hi.double() + lo.double()
    if rounding is None:
        rounding = tf32_rna if prec == TC_TF32 else bf16_rne
    return rounding(t).double()


def with_low_bits(t, bits, width):
    """t with its `width` low mantissa bits replaced by `bits` (tie values: 0x1000 / 13 for TF32, 0x8000 / 16 for bf16)."""
    mask = (1 << width) - 1
    return ((_bits(t) & ~mask) | bits).view(torch.float32)


# ---------------------------------------------------------------------------------------------------------------------
# geometry
# ---------------------------------------------------------------------------------------------------------------------
def wgt_pick_patch(Hs, Ws):
    """(bx, by) of lf_wgrad_tcg's 32-pixel patch: the widest bx = 32 >> i with Ws % bx == 0 and Hs % (32 / bx) == 0."""
    x = WGT_KP
    while x >= 1:
        if Ws % x == 0 and Hs % (WGT_KP // x) == 0:
            return x, WGT_KP // x
        x >>= 1
    return None


def tg_pick_patch(Hs, Ws):
    """(bx, by) of lf_conv_tcg's 128-pixel tile."""
    x = TG_BM
    while x >= 1:
        if Ws % x == 0 and Hs % (TG_BM // x) == 0:
            return x, TG_BM // x
        x >>= 1
    return None


def patch_pixels(N, Hs, Ws, bx, by, device=None):
    """(n, y, x) of every pixel of the iteration domain, patch after patch in the kernel's patch order
    (p -> tx = p % tiles_x, ty = p / tiles_x % tiles_y, n = p / (tiles_x * tiles_y)); patch p = rows [bx*by*p, +bx*by)."""
    tiles_x, tiles_y = Ws // bx, Hs // by
    p = torch.arange(N * tiles_x * tiles_y, device=device).view(-1, 1)
    k = torch.arange(bx * by, device=device).view(1, -1)
    n = (p // (tiles_x * tiles_y)).expand(-1, bx * by)
    y = (p // tiles_x) % tiles_y * by + k // bx
    x = p % tiles_x * bx + k % bx
    return n.reshape(-1), y.reshape(-1), x.reshape(-1)


def cta_patch_ranges(total, nctas):
    """[(p_begin, p_end)] of every split-K CTA of lf_wgrad_tcg (empty ranges for CTAs beyond the patches)."""
    per = (total + nctas - 1) // nctas
    return [(min(total, c * per), min(total, c * per + per)) for c in range(nctas)], per


def gather(flat, off, H, W, sn, sy, sx, n, y, x, c0, nc):
    """[npix, nc] fp64: element (n, y, x, c0 + c) of the strided view at element offset `off` of `flat`, zero outside
    [0, H) x [0, W) (TMA's zero fill)."""
    ok = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    idx = off + n * sn + y.clamp(0, H - 1) * sy + x.clamp(0, W - 1) * sx
    idx = idx.view(-1, 1) + (c0 + torch.arange(nc, device=flat.device)).view(1, -1)
    return flat[idx] * ok.view(-1, 1).to(flat.dtype)


def exact_and_abs(A, B):
    """(A^T B, |A|^T |B|) in fp64 for A [k, m], B [k, n] of quantised operands."""
    return A.t() @ B, A.abs().t() @ B.abs()


# ---------------------------------------------------------------------------------------------------------------------
# the gate
# ---------------------------------------------------------------------------------------------------------------------
def gate_bound(S, steps, prec, c_tc=None):
    return ((C_TC[prec] if c_tc is None else c_tc) + steps * ULP) * S


def gate_excess(got, ref, S, steps, prec, c_tc=None):
    """max over entries of |got - ref| / bound (<= 1 passes); an entry with S = 0 must be exactly ref."""
    err = (got.double() - ref).abs()
    bound = gate_bound(S, steps, prec, c_tc)
    exact = S == 0
    if bool((err[exact] != 0).any()):
        return float("inf")
    return float((err[~exact] / bound[~exact]).max()) if bool((~exact).any()) else 0.0


def tc_usage(got, ref, S, steps):
    """max over entries of (|got - ref| - steps * 2^-23 * S) / S: the part of the error c_tc has to cover."""
    err = (got.double() - ref).abs()
    nz = S > 0
    if not bool(nz.any()):
        return 0.0
    return float(((err[nz] - steps * ULP * S[nz]) / S[nz]).max())


def rel_err(got, ref, S):
    """max over entries of |got - ref| / S."""
    nz = S > 0
    if not bool(nz.any()):
        return 0.0
    return float(((got.double() - ref).abs()[nz] / S[nz]).max())


# ---------------------------------------------------------------------------------------------------------------------
# literal CPU restatements of the contracts on the args structs (the host code's pointers resolved against `tensors`)
# ---------------------------------------------------------------------------------------------------------------------
def _locate(ptr, tensors):
    for t in tensors:
        if t.data_ptr() <= ptr < t.data_ptr() + t.numel() * t.element_size():
            return t, (ptr - t.data_ptr()) // t.element_size()
    raise AssertionError("pointer outside the known tensors")


def emulate_conv_tcg(a, tensors):
    """CPU restatement of the lf_conv_tcg contract (include/lanefit_b200.h) on the exact views / strides the host
    code put into LfConvTcgArgs; `tensors` = the CPU tensors the pointers refer to."""
    K = a.ntaps * a.Kc
    wt, woff = _locate(a.wg, tensors)
    Wg = wt.reshape(-1)[woff:woff + a.Ng * K].view(a.Ng, K).double()
    acc = torch.zeros(a.N, a.Hs, a.Ws, a.Ng, dtype=torch.float64)
    for t in range(a.ntaps):
        v = a.a[a.map[t]]
        base, off = _locate(v.ptr, tensors)
        # as_strided must stay inside the storage: gather explicitly with bounds checks (zero outside [0,H)x[0,W))
        flat = base.reshape(-1).double()
        ys = torch.arange(a.Hs) + a.dy[t]
        xs = torch.arange(a.Ws) + a.dx[t]
        ok = ((ys >= 0) & (ys < v.H)).view(1, -1, 1, 1) & ((xs >= 0) & (xs < v.W)).view(1, 1, -1, 1)
        idx = (off + torch.arange(a.N).view(-1, 1, 1, 1) * v.sn + ys.clamp(0, v.H - 1).view(1, -1, 1, 1) * v.sy
               + xs.clamp(0, v.W - 1).view(1, 1, -1, 1) * v.sx + torch.arange(a.Kc).view(1, 1, 1, -1))
        A = flat[idx] * ok
        acc += torch.einsum("nyxk,ck->nyxc", A, Wg[:, t * a.Kc:(t + 1) * a.Kc])
    if a.bias:
        bt, boff = _locate(a.bias, tensors)
        acc += bt.reshape(-1)[boff:boff + a.Ng].double()
    ot, ooff = _locate(a.out, tensors)
    oflat = ot.reshape(-1)
    oidx = (ooff + torch.arange(a.N).view(-1, 1, 1, 1) * a.osn + (torch.arange(a.Hs) * a.oy_mul + a.oy0).view(1, -1, 1, 1) * a.osy
            + torch.arange(a.Ws).view(1, 1, -1, 1) * a.osx + torch.arange(a.Ng).view(1, 1, 1, -1))
    oflat[oidx.reshape(-1)] = acc.reshape(-1).float()


def emulate_wgrad_tcg(a, tensors):
    """CPU restatement of the lf_wgrad_tcg contract: every CTA's partial holds 1/nctas of the total (so that the
    reduction that follows is exercised), computed in fp64.  The A views hold elements of a.a_dtype, B is fp32."""
    def view_gather(v, dy, dx, c0, nc, dtype):
        base, off = _locate(v.ptr, tensors)
        assert base.dtype == dtype, (base.dtype, dtype)
        flat = base.reshape(-1).double()
        ys, xs = torch.arange(a.Hs) + dy, torch.arange(a.Ws) + dx
        ok = ((ys >= 0) & (ys < v.H)).view(1, -1, 1, 1) & ((xs >= 0) & (xs < v.W)).view(1, 1, -1, 1)
        idx = (off + torch.arange(a.N).view(-1, 1, 1, 1) * v.sn + ys.clamp(0, v.H - 1).view(1, -1, 1, 1) * v.sy
               + xs.clamp(0, v.W - 1).view(1, 1, -1, 1) * v.sx + (c0 + torch.arange(nc)).view(1, 1, 1, -1))
        return flat[idx] * ok

    a_dtype = {LF_F32: torch.float32, LF_BF16: torch.bfloat16}[a.a_dtype]
    B = view_gather(a.b, 0, 0, 0, a.Nn, torch.float32)
    D = torch.zeros(a.nblocks * 32, a.Nn, dtype=torch.float64)
    for blk in range(a.nblocks):
        A = view_gather(a.a[a.map[blk]], a.dy[blk], a.dx[blk], a.cblk[blk] * 32, 32, a_dtype)
        D[blk * 32:(blk + 1) * 32] = torch.einsum("nyxc,nyxo->co", A, B)
    pt, poff = _locate(a.partial, tensors)
    part = pt.reshape(-1)[poff:poff + a.nctas * D.numel()].view(a.nctas, *D.shape)
    part[:] = (D / a.nctas).float()


def emulate_wgrad_reduce(args, tensors):
    """CPU restatement of lf_wgrad_reduce: dst[t*st + p*sp + q*sq] = sum over splits of partial[s][t][p][q]."""
    partial, nsplit, ntaps, cp, cq, cpp, cqp, dst, st_, sp, sq, _stream = args
    src = next(t for t in tensors if t.data_ptr() == partial)
    red = src.reshape(-1)[:nsplit * ntaps * cpp * cqp].view(nsplit, ntaps, cpp, cqp)[:, :, :cp, :cq].double().sum(0).float()
    res, _ = _locate(dst, tensors)   # by each tensor's own byte extent: a bf16 tensor just below dst is not the destination
    idx = ((dst - res.data_ptr()) // 4 + torch.arange(ntaps).view(-1, 1, 1) * st_ + torch.arange(cp).view(1, -1, 1) * sp
           + torch.arange(cq).view(1, 1, -1) * sq)
    res.reshape(-1)[idx.reshape(-1)] = red.reshape(-1)
