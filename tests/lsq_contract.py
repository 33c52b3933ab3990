"""The contract of the weighted least-squares layer (lf_lsq_fwd / lf_lsq_bwd in csrc/lsq.cu) restated in fp64 and exact
arithmetic, and the per-entry gate its results are held to.

* Plan: lf_lsq_plan reports the kernel (row-separable or general), the activation template, the lanes per CTA NL, the
  lane groups and the chunks per system; plan_py() restates that selection (and every refusal) in Python.
* Forward reference: a = act(o) and w = a^2 in fp64 from the exact inputs (f32, or bf16 widened exactly); the moments
  S_k = sum w y^k and T_k = sum w x y^k over the unmasked rows in fp64, y = yrow[r] on the row-separable plan and ytab[p]
  on the general one; Z_ij = S_{2d-i-j} + reg_ls delta_ij, X_i = T_{d-i}, solved EXACTLY (fractions.Fraction) for beta
  and Z^-1.  Masked rows are dropped, not multiplied by zero (their y may be non-finite).
* Forward gate, from the kernel's operation order:
    - per pixel, w carries the activation's error (ACT table below) and one fp32 rounding (v*v);
    - row-separable: per row the fp32 sums A_r = sum_c w, B_r = sum_c w x run through V sequential terms per thread
      (sa +=, sb = fmaf), ceil(W / (32 V)) column steps and the five-level packed warp butterfly, so every term passes
      through at most NADD = V + steps + 5 rounded adds: e_A,r <= sum_c e_w + NADD u sum_c w, e_B,r likewise with |x|;
      eps_S[k] = sum_r |y_r|^k e_A,r and eps_T[k] = sum_r |y_r|^k e_B,r, plus the fp64 part (y^k by k products, one fma
      per row, the warp, block and chunk sums, and the reference's own fp64 sums): (k + H + 16 + nchunks) u64 per term;
    - general: w is one fp32 product and everything after it fp64;
    - first order, keeping the structure of the perturbation (dZ = sum_r dA_r phi_r phi_r^T, dX = sum_r dB_r phi_r, phi_r
      = [y_r^d .. 1]; per pixel for the general kernel), which is what |Z^-1| (eps_X + E_Z |beta|) bounds from above:
          |dbeta| <= sum_r |Z^-1 phi_r| (e_A,r |phi_r^T beta| + e_B,r),   |dZ^-1| <= sum_r e_A,r |Z^-1 phi_r| |Z^-1 phi_r|^T;
      the fp64 part as |Z^-1| (eps_X + E_Z |beta|) and |Z^-1| E_Z |Z^-1|, E_Z[i][j] = eps_S[2d-i-j]; the fp64 solve:
      C_SOLVE (d+1) u64 |Z^-1| |Z| |Z^-1| (and that times |X| for beta, + (d+1) u64 |Z^-1| |X| for the product Z^-1 X);
      + the rounding of the exact answer to fp64;
    - safety factor 2 for second-order terms; a case is only in the linear regime (and counts as covered) when rho, the
      infinity norm of the bound on |Z^-1 dZ| in the basis scaled by max|y|^(d-i), is <= RHO_MAX.
* Backward reference per pixel: ref = m phi(o) (x - phi^T(y) beta) 2 phi^T(y) (Z^-1 g), phi(o) = a'(o) a(o), from the
  exact fp64 beta, Z^-1 (row-major, any matrix) and g handed to lf_lsq_bwd.  Gate, from the kernel's order (q, s by fp64
  Horner, q = q_hi + q_lo, ((x - q_hi) - q_lo) * 2s in fp32, phi in fp32):
      |got - ref| <= 2 [ |2s| (C1 u |phi| |x - q| + C2 2^-48 |phi| qa) + e_phi |x - q| |2s| + |phi| |x - q| C3 u64 sa ]
  qa = sum |beta_i| |y|^(d-i), sa = 2 sum (|Z^-1| |g|)_i |y|^(d-i); + half a bf16 ulp of the stored value for bf16 d_o.
* Activation error table, absolute bounds e_a (on a) and e_phi (on phi = a' a) per element, from the CUDA math library's
  documented accuracy (no fast-math): expf within 2 ulp, log1pf within 1 ulp, division and products correctly rounded.
  One fp32 ulp of v is at most 2^-23 |v| = 2u |v|, so expf is off by up to d_e = 4u relative and log1pf by up to
  d_l = 2u; a correctly rounded operation by up to u:
      none, abs, relu : exact
      square          : e_a = u a; e_phi = 2u |phi| (2 o exact, then two products)
      sigmoid         : s = 1 / (1 + e), e = expf(-o).  The relative error d_e of e reaches 1 + e scaled by e / (1 + e)
                        = 1 - s, then one rounding for 1 + e and one for the division:
                            e_a = (d_e (1 - s) + 2u) s
                        phi = (s (1 - s)) s from the rounded s: phi'(s) = 2s - 3s^2, three roundings (1 - s, two products):
                            e_phi = |2s - 3s^2| e_a + 3u |phi| + e_a^2
                        (the error of 1 - s is absolute, not relative, as s -> 1)
      softplus        : o > 20: a = o, phi = o exactly (torch's threshold 20, derivative 1 above it).  Else e = expf(o),
                        a = log1pf(e): d log1p(e) = de / (1 + e), so e's error reaches a as d_e sigma, sigma = e / (1 + e):
                            e_a = d_e sigma + d_l a
                        phi = (e / (1 + e)) log1pf(e): sigma from the same e with relative error d_e (1 - sigma) + 2u, the
                        product one more rounding:
                            e_phi = |phi| (d_e (1 - sigma) + 3u) + sigma e_a
  The first-order sums are scaled by SECOND for the products of the per-operation errors.  sigmoid, softplus and square
  add an absolute floor for subnormal results and for expf's overflow (sigmoid: s < 2.9e-39 once expf(-o) overflows).
"""
from fractions import Fraction

import numpy as np
import torch

U = 2.0 ** -24                       # fp32 unit round-off
U64 = 2.0 ** -53
TINY = 2.0 ** -140                   # absolute floor: subnormal results of the products, w = a^2 and d_o
ULP = 2.0 ** -23                     # one fp32 ulp relative to the value it belongs to (at most)
EXPF_ULP, LOG1PF_ULP = 2, 1          # CUDA math library accuracy of expf and log1pf
D_E, D_L = EXPF_ULP * ULP, LOG1PF_ULP * ULP
FLOOR = 2.0 ** -126                  # sigmoid / softplus: subnormal results, expf overflow
SECOND = 1.0 + 1e-6                  # second-order products of the per-operation errors (each <= 6u)
C_SOLVE = 8                          # fp64 Gauss-Jordan / Cholesky: C_SOLVE (d+1) u64 |Z^-1||Z||Z^-1|
C1, C2 = 6, 4                        # backward: rounded fp32 ops on x - q and the products; the q_hi + q_lo split
SAFETY = 2.0
RHO_MAX = 1e-2

LF_F32, LF_BF16 = 0, 1
ACTS = ("none", "square", "abs", "relu", "sigmoid", "softplus")     # index = LF_ACT_*
ACT_SQUARE, ACT_RUNTIME = 1, -1
THREADS, WARPS, MAXL = 256, 8, 4
INVALID, UNSUPPORTED = -1, -2


# ---------------------------------------------------------------------------------------------------------------------
# the plan (restated) and the query
# ---------------------------------------------------------------------------------------------------------------------
def pick_nchunks(B, groups, H, mask_rows, ctas_per_sm, sms):
    slots, units = sms * ctas_per_sm, B * groups
    ha = H - mask_rows if H - mask_rows > 0 else 1
    n_max = ha // WARPS if ha // WARPS > 1 else 1
    n_cap = (H + WARPS - 1) // WARPS
    best, best_score = 1, -1.0
    n = 1
    while n <= n_max and n <= n_cap:
        ctas = units * n
        waves = (ctas + slots - 1) // slots
        fill = float(ctas) / float(waves * slots)
        rows = float(ha) / n
        score = fill * (rows / (rows + 6.0))
        if score > best_score + 1e-9:
            best_score, best = score, n
        n += 1
    return best


def workspace_bytes(B, L, H, order):
    if B <= 0 or L <= 0 or H <= 0 or order < 0 or order > 4 or B * L * 4 > 65536:
        return 0
    return 65536 + B * L * ((H + WARPS - 1) // WARPS) * (3 * order + 2) * 8


def device_sms():
    """SMs the library sizes its grids for: the current device's, or 132 without one (as device_sms() in C)."""
    try:
        if torch.cuda.is_available():
            return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    except Exception:
        pass
    return 132


def plan_py(bwd, dtype, has_yrow, has_ytab, B, L, H, W, order, mask_rows, act, sms=None):
    """(rc, plan dict or None): the selection lf_lsq_fwd / lf_lsq_bwd make, restated."""
    sms = device_sms() if sms is None else sms
    if not (B > 0 and L > 0 and H > 0 and W > 0 and 0 <= order <= 4 and 0 <= mask_rows <= H and 0 <= act <= 5
            and dtype in (LF_F32, LF_BF16) and B <= 65535 and L <= 65535):
        return INVALID, None
    if not bwd and workspace_bytes(B, L, H, order) == 0:
        return UNSUPPORTED, None
    rowsep = bool(has_yrow) and W % (8 if dtype == LF_BF16 else 4) == 0
    if not rowsep and not has_ytab:
        return INVALID, None
    groups, nl = L, 1
    if rowsep:
        groups = (L + MAXL - 1) // MAXL
        nl = (L + groups - 1) // groups
    cps = 4 if bwd else (2 if rowsep else 4)
    return 0, dict(rowsep=int(rowsep), act_t=ACT_SQUARE if act == 1 else ACT_RUNTIME, nl=nl, groups=groups,
                   nchunks=pick_nchunks(B, groups, H, mask_rows, cps, sms), ctas_per_sm=cps, align=16 if rowsep else 0)


def query_plan(bwd, dtype, has_yrow, has_ytab, B, L, H, W, order, mask_rows, act):
    import ctypes
    from lanedetection_end2end_b200 import _capi
    info = (ctypes.c_int * _capi.LSQ_PLAN_INFO)()
    rc = _capi.lib().lf_lsq_plan(bwd, dtype, int(has_yrow), int(has_ytab), B, L, H, W, order, mask_rows, act, info)
    return rc, (dict(zip(_capi.LSQ_PLAN_FIELDS, list(info))) if rc == 0 else None)


def instance(bwd, dtype, plan):
    """The kernel template a launch runs: (direction, kernel, activation template, dtype, NL)."""
    return ("bwd" if bwd else "fwd", "rowsep" if plan["rowsep"] else "general",
            "square" if plan["act_t"] == ACT_SQUARE else "runtime", "bf16" if dtype == LF_BF16 else "f32",
            plan["nl"] if plan["rowsep"] else 1)


def all_instances():
    out = set()
    for bwd in (0, 1):
        for a in ("square", "runtime"):
            for dt in ("f32", "bf16"):
                out.add(("bwd" if bwd else "fwd", "general", a, dt, 1))
                for nl in (1, 2, 3, 4):
                    out.add(("bwd" if bwd else "fwd", "rowsep", a, dt, nl))
    return out


def chunk_rows(c, n, H, mask_rows):
    """(masked rows, unmasked rows) of chunk c of n, as lsq_chunk_rows splits them."""
    ha = H - mask_rows
    return (range(c * mask_rows // n, (c + 1) * mask_rows // n),
            range(mask_rows + c * ha // n, mask_rows + (c + 1) * ha // n))


# ---------------------------------------------------------------------------------------------------------------------
# activations
# ---------------------------------------------------------------------------------------------------------------------
def _sigmoid(o):
    from scipy.special import expit          # no overflow for any o, relative accuracy of a few u64 on both sides
    return expit(o)


def act64(o, act):
    """(a, phi = a'(o) a(o)) in fp64 of the exact inputs o (fp64 array)."""
    name = ACTS[act]
    if name == "none":
        return o.copy(), o.copy()
    if name == "square":
        return o * o, 2.0 * o ** 3
    if name == "abs":
        return np.abs(o), o.copy()
    if name == "relu":
        r = np.maximum(o, 0.0)
        return r, r.copy()
    if name == "sigmoid":
        s = _sigmoid(o)
        return s, s * s * _sigmoid(-o)           # s^2 (1 - s), without the cancellation of 1 - s
    big = o > 20.0
    a = np.where(big, o, np.log1p(np.exp(np.minimum(o, 20.0))))
    return a, np.where(big, o, _sigmoid(o) * a)


def act_err(o, act):
    """(e_a, e_phi): absolute bounds on the kernel's fp32 a and phi (table in the module docstring)."""
    name = ACTS[act]
    a, phi = act64(o, act)
    z = np.zeros_like(o)
    if name in ("none", "abs", "relu"):
        return z, z
    if name == "square":
        return U * a + TINY, 2 * U * np.abs(phi) + TINY
    if name == "sigmoid":
        s, c = a, _sigmoid(-o)                              # s and 1 - s
        ea = SECOND * (D_E * c + 2 * U) * s + FLOOR
        return ea, SECOND * (np.abs(2 * s * c - s * s) * ea + 3 * U * np.abs(phi)) + ea * ea + FLOOR
    big = o > 20.0
    sig, sc = _sigmoid(o), _sigmoid(-o)
    ea = SECOND * (D_E * sig + D_L * a) + FLOOR
    ephi = SECOND * (np.abs(phi) * (D_E * sc + 3 * U) + sig * ea) + FLOOR
    return np.where(big, 0.0, ea), np.where(big, 0.0, ephi)


def act_f32_torch(o32, act):
    """torch-CPU float32 activation (the masked output's reference)."""
    name = ACTS[act]
    t = torch.as_tensor(o32, dtype=torch.float32)
    if name == "none":
        return t.clone()
    if name == "square":
        return t * t
    if name == "abs":
        return t.abs()
    if name == "relu":
        return torch.relu(t)
    if name == "sigmoid":
        return torch.sigmoid(t)
    return torch.nn.functional.softplus(t)


# ---------------------------------------------------------------------------------------------------------------------
# exact solve
# ---------------------------------------------------------------------------------------------------------------------
def solve_exact(Z, X):
    """(beta, Z^-1) of one system from fp64 Z [n, n], X [n], by Gauss-Jordan in Fractions; None if singular."""
    n = len(X)
    M = [[Fraction(float(Z[i][j])) for j in range(n)] + [Fraction(int(i == j)) for j in range(n)] for i in range(n)]
    for c in range(n):
        p = next((r for r in range(c, n) if M[r][c] != 0), None)
        if p is None:
            return None
        M[c], M[p] = M[p], M[c]
        piv = M[c][c]
        M[c] = [v / piv for v in M[c]]
        for r in range(n):
            if r != c and M[r][c] != 0:
                f = M[r][c]
                M[r] = [vr - f * vc for vr, vc in zip(M[r], M[c])]
    inv = [row[n:] for row in M]
    Xf = [Fraction(float(v)) for v in X]
    beta = [sum((inv[i][j] * Xf[j] for j in range(n)), Fraction(0)) for i in range(n)]
    return np.array([float(b) for b in beta]), np.array([[float(v) for v in row] for row in inv])


# ---------------------------------------------------------------------------------------------------------------------
# forward reference and gate
# ---------------------------------------------------------------------------------------------------------------------
def forward_reference(o, xtab, yvals, H, W, order, mask_rows, act, reg_ls, rowsep, nchunks, dtype, mut=None):
    """Per system (beta, Z^-1, beta bound, Z^-1 bound, rho), all [B, L, ...] fp64 numpy, and the moments.
    o: [B, L, H, W] exact values (fp64 numpy); xtab [H*W]; yvals: yrow [H] (rowsep) or ytab [H*W] (general).
    mut: fp64 mutation -- ("drop_row", r), ("mask_rows", m), ("y_row", r), ("lane", l), ("x_shift",), ("w_eq_a",),
    ("no_reg",)."""
    mut = mut or ()
    kind = mut[0] if mut else None
    o = np.asarray(o, np.float64)
    B, L = o.shape[:2]
    d, n = order, order + 1
    mr = mut[1] if kind == "mask_rows" else mask_rows
    if kind == "lane":
        o = o.copy()
        o[:, mut[1]] = o[:, mut[1] - 1]
    x = np.asarray(xtab, np.float64).reshape(H, W)
    if kind == "x_shift":
        x = np.concatenate([x[:, 1:], x[:, -1:]], 1)
    if rowsep:
        y = np.repeat(np.asarray(yvals, np.float64).reshape(H, 1), W, 1)
    else:
        y = np.asarray(yvals, np.float64).reshape(H, W)
    if kind == "y_row":
        y = y.copy()
        y[mut[1]] = y[mut[1] + 1]
    rows = np.arange(mr, H)
    if kind == "drop_row":
        rows = rows[rows != mut[1]]
    ov, xv, yv = o[:, :, rows], x[rows], y[rows]
    a, _ = act64(ov, act)
    ea, _ = act_err(ov, act)
    w = a if kind == "w_eq_a" else a * a
    ew = 2 * np.abs(a) * ea + U * w + 2.0 ** -149
    ax, ay = np.abs(xv), np.abs(yv)
    R = len(rows)
    V = 8 if dtype == LF_BF16 else 4
    if rowsep:
        # fp32 row sums: the perturbation of Z is sum_r dA_r phi_r phi_r^T, of X sum_r dB_r phi_r
        nadd = V + -(-W // (32 * V)) + 5
        eA = ew.sum(-1) + nadd * U * w.sum(-1)                      # [B, L, R]
        eB = (ew * ax).sum(-1) + nadd * U * (w * ax).sum(-1)
        wt, wxt = w.sum(-1), (w * xv).sum(-1)
        yp = yv[:, 0] if R else np.zeros(0)
        nf = H + 16 + nchunks
    else:
        # general: per pixel one fp32 product, then fp64
        eA, eB = ew.reshape(B, L, -1), (ew * ax).reshape(B, L, -1)
        wt, wxt = w.reshape(B, L, -1), (w * xv).reshape(B, L, -1)
        yp = yv.reshape(-1)
        nf = R * W // THREADS + 29 + nchunks
    Phi = np.stack([yp ** (d - i) for i in range(n)], -1)             # [R or P, n], highest power first
    S = np.stack([np.einsum("blr,r->bl", wt, yp ** k) for k in range(2 * d + 1)], -1)
    T = np.stack([np.einsum("blr,r->bl", wxt, yp ** k) for k in range(d + 1)], -1)
    # fp64 part (y^k by k products, fma per row / pixel, warp, block and chunk sums, and the reference's own sums)
    epsS = np.stack([(k + nf) * U64 * np.einsum("blr,r->bl", np.abs(wt), np.abs(yp) ** k) for k in range(2 * d + 1)], -1)
    epsT = np.stack([(k + nf) * U64 * np.einsum("blr,r->bl", np.abs(wxt), np.abs(yp) ** k) for k in range(d + 1)], -1)
    reg = 0.0 if kind == "no_reg" else reg_ls
    I, J = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    Z = S[..., 2 * d - I - J] + reg * np.eye(n)
    X = T[..., d - np.arange(n)]
    EZ = epsS[..., 2 * d - I - J]
    eX = epsT[..., d - np.arange(n)]
    beta = np.full((B, L, n), np.nan)
    Zi = np.full((B, L, n, n), np.nan)
    bb = np.full((B, L, n), np.inf)
    bz = np.full((B, L, n, n), np.inf)
    rho = np.full((B, L), np.inf)
    cs = C_SOLVE * n * U64
    ymax = max(float(np.abs(yp).max()) if len(yp) else 1.0, 1e-30)
    D = np.array([ymax ** (d - i) for i in range(n)])                 # scaling of the linear-regime norm
    for b in range(B):
        for l in range(L):
            r = solve_exact(Z[b, l], X[b, l])
            if r is None:
                continue
            be, zi = r
            az, aZ, aX = np.abs(zi), np.abs(Z[b, l]), np.abs(X[b, l])
            Uv = np.abs(Phi @ zi.T)                                   # |Z^-1 phi_r| per row / pixel
            fit = np.abs(Phi @ be)                                    # |phi_r^T beta|
            dz32 = Uv.T @ (eA[b, l][:, None] * Uv)
            db32 = Uv.T @ (eA[b, l] * fit + eB[b, l])
            dzs = cs * az @ aZ @ az
            dz = dz32 + az @ EZ[b, l] @ az + dzs
            db = db32 + az @ (eX[b, l] + EZ[b, l] @ np.abs(be)) + dzs @ aX + n * U64 * az @ aX
            beta[b, l], Zi[b, l] = be, zi
            bb[b, l] = SAFETY * db + U64 * np.abs(be)
            bz[b, l] = SAFETY * dz + U64 * az
            M = (Uv.T @ (eA[b, l][:, None] * np.abs(Phi))) + az @ (EZ[b, l] + cs * aZ)   # bounds |Z^-1 dZ|
            rho[b, l] = float(((M * D[:, None]) / D[None, :]).sum(-1).max())   # D M D^-1
    return dict(beta=beta, zinv=Zi, bound_beta=bb, bound_zinv=bz, rho=rho, S=S, T=T)


def excess(got, ref, bound):
    """max |got - ref| / bound over the entries (<= 1 passes); a zero bound demands equality, NaN in ref demands NaN."""
    got, ref, bound = (np.asarray(v, np.float64) for v in (got, ref, bound))
    nan = np.isnan(ref)
    if (np.isnan(got) != nan).any():
        return float("inf")
    err = np.abs(got[~nan] - ref[~nan])
    bnd = bound[~nan]
    if not np.isfinite(err).all():
        return float("inf")
    zero = bnd == 0
    if (err[zero] != 0).any():
        return float("inf")
    return float((err[~zero] / bnd[~zero]).max()) if (~zero).any() else 0.0


def forward_excess(got_beta, got_zinv, ref):
    return max(excess(got_beta, ref["beta"], ref["bound_beta"]), excess(got_zinv, ref["zinv"], ref["bound_zinv"]))


def bf16_half_ulp(v):
    """Half a bf16 ulp of each (bf16) value: the most its rounding from fp32 can have moved it."""
    a = np.abs(np.asarray(v, np.float64))
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    return np.where(a > 0, 2.0 ** (np.maximum(e, -126) - 8), 2.0 ** -134)


def gate_use(got, ref, bound, rounding):
    """max over entries of (|got - ref| - rounding) / (bound - rounding): how much of the gate beyond the final bf16
    rounding an error uses (the headroom figure of the bf16 outputs, whose rounding can reach half an ulp exactly)."""
    got, ref, bound, rounding = (np.broadcast_to(np.asarray(v, np.float64), np.shape(ref)) for v in (got, ref, bound, rounding))
    live = bound > rounding
    if not live.any():
        return 0.0
    return float(((np.abs(got - ref) - rounding)[live] / (bound - rounding)[live]).max())


# ---------------------------------------------------------------------------------------------------------------------
# backward reference and gate
# ---------------------------------------------------------------------------------------------------------------------
def backward_reference(o, xtab, yvals, H, W, order, mask_rows, act, beta, zinv, g, rowsep, dtype, got=None, mut=None):
    """(ref, bound) [B, L, H, W] fp64 of lf_lsq_bwd.  got: the kernel's d_o (for the bf16 half-ulp term).
    mut: ("no_factor2",), ("zinv_t",), ("unmask_row",), ("flip_residual",)."""
    mut = mut or ()
    kind = mut[0] if mut else None
    o = np.asarray(o, np.float64)
    d, n = order, order + 1
    x = np.asarray(xtab, np.float64).reshape(1, 1, H, W)
    y = (np.repeat(np.asarray(yvals, np.float64).reshape(H, 1), W, 1) if rowsep
         else np.asarray(yvals, np.float64).reshape(H, W))[None, None]
    zi = np.swapaxes(zinv, -1, -2) if kind == "zinv_t" else zinv
    z = np.einsum("blij,blj->bli", zi, g)
    za = 2 * np.einsum("blij,blj->bli", np.abs(zi), np.abs(g))
    mr = mask_rows - 1 if kind == "unmask_row" else mask_rows
    with np.errstate(all="ignore"):
        q = sum(beta[..., i, None, None] * y ** (d - i) for i in range(n))
        qa = sum(np.abs(beta[..., i, None, None]) * np.abs(y) ** (d - i) for i in range(n))
        s = 2 * sum(z[..., i, None, None] * y ** (d - i) for i in range(n))
        sa = sum(za[..., i, None, None] * np.abs(y) ** (d - i) for i in range(n))
        _, phi = act64(o, act)
        _, ephi = act_err(o, act)
        r = (q - x) if kind == "flip_residual" else (x - q)
        ref = phi * r * s * (0.5 if kind == "no_factor2" else 1.0)
        bound = SAFETY * (np.abs(s) * (C1 * U * np.abs(phi) * np.abs(r) + C2 * 2.0 ** -48 * np.abs(phi) * qa)
                          + ephi * np.abs(r) * np.abs(s) + np.abs(phi) * np.abs(r) * 4 * n * U64 * sa) + TINY
        if dtype == LF_BF16:
            bound = bound + bf16_half_ulp(got)
    ref[:, :, :mr] = 0.0
    bound[:, :, :mr] = 0.0
    return ref, bound


# ---------------------------------------------------------------------------------------------------------------------
# kernel-faithful fp32 emulation (the CPU tests hold it to the gate)
# ---------------------------------------------------------------------------------------------------------------------
def ulp_shift(t, k):
    """fp32 values that differ from the exact values t (fp64) by as close to k fp32 ulps as stays within |k| ulps: what
    a math-library function within |k| ulp may return, at the edge of its bound in the direction of k."""
    t = np.asarray(t, np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        at = np.abs(t)
        e = np.floor(np.log2(np.where(at > 0, at, 1.0)))
        ulp = np.where(at >= 2.0 ** -126, 2.0 ** (e - 23), 2.0 ** -149)
        v = (t + k * ulp).astype(np.float32)
        far = np.abs(v.astype(np.float64) - t) > abs(k) * ulp
        v = np.where(far, np.nextafter(v, t.astype(np.float32)), v)
        return np.where(np.isfinite(t), v, t.astype(np.float32)).astype(np.float32)


def _exp_log(o32, sign, exp_ulps, log_ulps):
    """(e, log1p(e)) as the kernel's expf / log1pf give them: correctly rounded when the ulp arguments are None, else at
    the edge of the documented bound in their direction."""
    f = np.float32
    with np.errstate(over="ignore"):
        t = np.exp(sign * o32.astype(np.float64))
        e = t.astype(f) if exp_ulps is None else ulp_shift(t, exp_ulps)
        lt = np.log1p(e.astype(np.float64))
        return e, (lt.astype(f) if log_ulps is None else ulp_shift(lt, log_ulps))


def _act_f32(o32, act, exp_ulps=None, log_ulps=None):
    """The kernel's fp32 activation; expf / log1pf correctly rounded, or moved to the edge of their documented bounds."""
    f = np.float32
    name = ACTS[act]
    if name == "none":
        return o32.copy()
    if name == "square":
        return o32 * o32
    if name == "abs":
        return np.abs(o32)
    if name == "relu":
        return np.maximum(o32, f(0))
    with np.errstate(over="ignore"):
        if name == "sigmoid":
            e, _ = _exp_log(o32, -1.0, exp_ulps, log_ulps)
            return f(1) / (f(1) + e)
        e, l1p = _exp_log(o32, 1.0, exp_ulps, log_ulps)
        return np.where(o32 > f(20), o32, l1p)


def _dact_f32(o32, act, exp_ulps=None, log_ulps=None):
    f = np.float32
    name = ACTS[act]
    if name == "square":
        return f(2) * o32 * o32 * o32
    if name == "abs" or name == "none":
        return o32.copy()
    if name == "relu":
        return np.maximum(o32, f(0))
    with np.errstate(over="ignore", invalid="ignore"):
        if name == "sigmoid":
            e, _ = _exp_log(o32, -1.0, exp_ulps, log_ulps)
            s = f(1) / (f(1) + e)
            return s * (f(1) - s) * s
        e, l1p = _exp_log(o32, 1.0, exp_ulps, log_ulps)
        return np.where(o32 > f(20), o32, (e / (f(1) + e)) * l1p)


def emulate_forward_rowsep(o32, xtab, yrow, H, W, order, mask_rows, act, reg_ls, dtype, ulps=(None, None)):
    """(beta, Z^-1) as the row-separable kernel forms them: per thread V sequential fp32 terms, fp32 column steps, the
    xor butterfly (the packed reduction adds the same pairs), then fp64 per row and a fp64 solve.  ulps = (expf, log1pf)
    ulp offsets of the math library (None: correctly rounded)."""
    f = np.float32
    V = 8 if dtype == LF_BF16 else 4
    WV = W // V
    steps = -(-WV // 32)
    v = _act_f32(np.asarray(o32, f)[:, :, mask_rows:], act, *ulps)
    B, L, R = v.shape[:3]
    w = v * v
    x = np.asarray(xtab, f).reshape(H, W)[mask_rows:]
    pad = steps * 32 * V - W
    wp = np.concatenate([w, np.zeros((B, L, R, pad), f)], -1).reshape(B, L, R, steps, 32, V)
    xp = np.concatenate([x, np.zeros((R, pad), f)], -1).reshape(1, 1, R, steps, 32, V)
    A = np.zeros((B, L, R, 32), f)
    Bx = np.zeros((B, L, R, 32), f)
    for st in range(steps):
        sa = np.zeros((B, L, R, 32), f)
        sb = np.zeros((B, L, R, 32), f)
        for e in range(V):
            sa = sa + wp[..., st, :, e]
            sb = (wp[..., st, :, e].astype(np.float64) * xp[..., st, :, e] + sb).astype(f)   # fmaf
        A, Bx = A + sa, Bx + sb
    for m in (16, 8, 4, 2, 1):
        A, Bx = A[..., :m] + A[..., m:2 * m], Bx[..., :m] + Bx[..., m:2 * m]
    A, Bx = A[..., 0].astype(np.float64), Bx[..., 0].astype(np.float64)
    yr = np.asarray(yrow, np.float64)[mask_rows:]
    d, n = order, order + 1
    S = np.stack([(A * yr ** k).sum(-1) for k in range(2 * d + 1)], -1)
    T = np.stack([(Bx * yr ** k).sum(-1) for k in range(d + 1)], -1)
    I, J = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    Z = S[..., 2 * d - I - J] + reg_ls * np.eye(n)
    Zi = np.linalg.inv(Z)
    return np.einsum("blij,blj->bli", Zi, T[..., d - np.arange(n)]), Zi


def emulate_backward(o32, xtab, yvals, H, W, order, mask_rows, act, beta, zinv, g, rowsep, ulps=(None, None)):
    """d_o (fp32) in the kernel's per-pixel order (row-separable: q_hi + q_lo split and fp32 residual; general: fp64)."""
    f = np.float32
    o32 = np.asarray(o32, f)
    d, n = order, order + 1
    zs = 2.0 * np.einsum("blij,blj->bli", zinv, g)
    y = (np.repeat(np.asarray(yvals, np.float64).reshape(H, 1), W, 1) if rowsep
         else np.asarray(yvals, np.float64).reshape(H, W))[None, None]
    q = beta[..., 0, None, None] * np.ones_like(y)
    s = zs[..., 0, None, None] * np.ones_like(y)
    for i in range(1, n):
        q = q * y + beta[..., i, None, None]
        s = s * y + zs[..., i, None, None]
    x32 = np.asarray(xtab, f).reshape(1, 1, H, W)
    phi = _dact_f32(o32, act, *ulps)
    if rowsep:
        qh = q.astype(f)
        ql = (q - qh).astype(f)
        sf = s.astype(f)
        if ACTS[act] == "square":
            o3 = (o32 * o32) * o32
            out = o3 * (((x32 - qh) - ql) * (f(2) * sf))
        else:
            out = phi * (((x32 - qh) - ql) * sf)
    else:
        out = (phi.astype(np.float64) * (x32.astype(np.float64) - q) * s).astype(f)
    out = np.array(out, f)
    out[:, :, :mask_rows] = 0
    return out


def rowsep_tables(H, W, kind="bev"):
    """(xtab [H*W], ytab [H*W], yrow [H]) fp32 of a synthetic row-separable grid: x across the columns (with a row-dependent
    offset), y exactly constant along each row: kind "bev" y in [0, 1), "bp" y in (0, 255]."""
    r = np.arange(H, dtype=np.float64)[:, None]
    c = np.arange(W, dtype=np.float64)[None, :]
    x = (c * (512.0 / max(W, 1)) + 3.0 * r / max(H, 1)).astype(np.float32)
    yr = ((H - r[:, 0]) / (H + 1.0) if kind == "bev" else 255.0 - 200.0 * r[:, 0] / max(H, 1)).astype(np.float32)
    return x.reshape(-1), np.repeat(yr[:, None], W, 1).reshape(-1), yr


def nonsymmetric_backward_inputs(B, L, order, ymax, seed):
    """(beta, Z^-1, g) fp64 built by hand: beta_i y^(d-i) of order 100 for y up to ymax, and a non-symmetric Z^-1 (so a
    transposed coefficient load shows)."""
    rng = np.random.default_rng(seed)
    n = order + 1
    beta = rng.standard_normal((B, L, n)) * np.array([100.0 / max(ymax, 1e-3) ** (order - i) for i in range(n)])
    zinv = rng.standard_normal((B, L, n, n)) * 1e-3 + 1e-3 * np.triu(np.ones((n, n)), 1)
    g = rng.standard_normal((B, L, n))
    return beta, zinv, g


# ---------------------------------------------------------------------------------------------------------------------
# the GPU coverage table: one case per kernel instance and direction
# ---------------------------------------------------------------------------------------------------------------------
# (name, dtype, act, L, H, W, B, order, solver, reg_ls, mask_rows, grid, yrow given) -> fwd and bwd instance
COVERAGE = [
    ("sq_f32_nl1_cap", LF_F32, 1, 1, 256, 512, 1, 2, 0, 0.0, 0, "bev", True),
    ("sq_f32_nl2", LF_F32, 1, 2, 9, 100, 3, 1, 1, 1e-3, 1, "bp", True),
    ("sq_f32_nl3_part", LF_F32, 1, 5, 7, 132, 8, 0, 0, 0.0, 6, "bev", True),
    ("sq_f32_nl4_part", LF_F32, 1, 10, 1, 4, 2, 2, 0, 1.0, 0, "bev", True),
    ("sq_bf16_nl1", LF_BF16, 1, 1, 320, 640, 2, 3, 1, 0.0, 1, "bev", True),
    ("sq_bf16_nl2_allmasked", LF_BF16, 1, 2, 7, 8, 128, 2, 0, 1.0, 7, "bev", True),
    ("sq_bf16_nl3", LF_BF16, 1, 3, 9, 136, 5, 1, 0, 0.0, 0, "bp", True),
    ("sq_bf16_nl4_part", LF_BF16, 1, 7, 256, 512, 2, 4, 0, 0.0, 77, "bev", True),
    ("sigmoid_f32_nl1", LF_F32, 4, 1, 9, 640, 4, 0, 1, 1e-3, 8, "bev", True),
    ("softplus_f32_nl2", LF_F32, 5, 2, 256, 132, 1, 3, 0, 0.0, 52, "bev", True),
    ("abs_f32_nl3", LF_F32, 2, 3, 7, 4, 16, 1, 0, 1.0, 1, "bp", True),
    ("relu_f32_nl4", LF_F32, 3, 4, 320, 100, 2, 2, 1, 0.0, 0, "bp", True),
    ("none_bf16_nl1_allmasked", LF_BF16, 0, 1, 1, 8, 1, 0, 0, 1.0, 1, "bev", True),
    ("sigmoid_bf16_nl2", LF_BF16, 4, 2, 9, 512, 64, 4, 1, 1.0, 0, "bev", True),
    ("softplus_bf16_nl3_part", LF_BF16, 5, 5, 256, 136, 1, 2, 0, 1e-3, 1, "bp", True),
    ("none_bf16_nl4_part", LF_BF16, 0, 10, 7, 640, 3, 3, 0, 0.0, 0, "bev", True),
    ("sq_f32_general_w98", LF_F32, 1, 3, 9, 98, 2, 2, 0, 0.0, 1, "bev", True),
    ("sq_bf16_general_w100", LF_BF16, 1, 2, 7, 100, 4, 1, 1, 0.0, 0, "bp", True),
    ("softplus_f32_general", LF_F32, 5, 2, 256, 512, 1, 3, 0, 0.0, 77, "bev", False),
    ("sigmoid_bf16_general", LF_BF16, 4, 1, 320, 640, 2, 2, 1, 0.0, 64, "bp", False),
]
CASE_FIELDS = ("name", "dtype", "act", "L", "H", "W", "B", "order", "solver", "reg_ls", "mask_rows", "grid", "yrow")


def case_dict(case):
    return dict(zip(CASE_FIELDS, case))


def case_operands(c, seed=0):
    """(o fp32 array (bf16-exact for bf16 cases), xtab, ytab, yrow) of a coverage case: values of both signs, the softplus
    threshold (19.9, 20, 20.1) and large |o| (+-30, +-100) planted in every unmasked row of the activations that care."""
    rng = np.random.default_rng(1000 + seed + sum(map(ord, c["name"])))
    B, L, H, W = c["B"], c["L"], c["H"], c["W"]
    o = (rng.standard_normal((B, L, H, W)) * 1.5 + 0.3).astype(np.float32)
    if ACTS[c["act"]] == "softplus":
        o[..., 0:3] = np.array([19.9, 20.0, 20.1], np.float32)[:min(3, W)] if W >= 3 else 20.0
    if ACTS[c["act"]] == "sigmoid" and W >= 4:
        o[..., 0:4] = np.array([30.0, -30.0, 100.0, -100.0], np.float32)
    if c["dtype"] == LF_BF16:
        o = torch.from_numpy(o).bfloat16().float().numpy()
    xtab, ytab, yrow = rowsep_tables(H, W, c["grid"])
    return o, xtab, ytab, yrow


def forward_mutations(c, plan):
    """The fp64 mutations of the forward that apply to a case; each must break the gate.  A regularisation below 1e-3
    of the pixel count cannot move beta past the gate, so dropping it is only asked to show where it is larger."""
    H, L, mask_rows = c["H"], c["L"], c["mask_rows"]
    m = []
    if mask_rows < H:
        r = mask_rows
        if plan["nchunks"] > 1:                       # first row of chunk 1: a chunk boundary
            r = min(max(chunk_rows(1, plan["nchunks"], H, mask_rows)[1].start, mask_rows), H - 1)
        m += [("drop_row", r), ("mask_rows", mask_rows + 1), ("x_shift",), ("w_eq_a",)]
        if c["order"] > 0 and H - mask_rows >= 2:
            m.append(("y_row", mask_rows))
    if mask_rows > 0:
        m.append(("mask_rows", mask_rows - 1))
    if c["reg_ls"] and c["reg_ls"] >= 1e-3 * (H - mask_rows) * c["W"]:
        m.append(("no_reg",))
    if plan["rowsep"] and L % plan["nl"]:
        m.append(("lane", L - 1))
    return m


def backward_mutations(c):
    if c["mask_rows"] >= c["H"]:
        return []
    return ([("no_factor2",), ("flip_residual",)] + ([("zinv_t",)] if c["order"] > 0 else [])     # 1x1 at order 0
            + ([("unmask_row",)] if c["mask_rows"] > 0 else []))
