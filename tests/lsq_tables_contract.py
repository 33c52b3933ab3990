"""The contract of the least-squares layer's table entry points (csrc/lsq.cu) restated in fp64 and exact arithmetic, on
top of tests/lsq_contract.py (imported as lc: its references, gates, activations and emulations are reused):

  rowsums    lf_lsq_fwd_rowsums[_keep]                       lsq_fwd_rowsums[_keep]_kernel<ACT_T, BF16, NL>
  grid_grad  lf_lsq_grid_grad[_per_image]                    lsq_grid_grad[_pi]_kernel
  per_image  lf_lsq_{fwd,bwd}_per_image                      lsq_fwd_rowsep_pi_kernel<ACT_T, BF16, NL, ROWSUMS, KEEP>,
                                                             lsq_bwd_rowsep_pi[_keep]_kernel<ACT_T, BF16, NL>
  lanes      lf_lsq_*_lanes (Lmap > L: a prefix fit)         lsq_{fwd,bwd}_{rowsep,general}_lanes_kernel, run-time
                                                             per_image flag

* Instances: launched() restates which (kernel, ACT_T, dtype, NL, ROWSUMS, KEEP, per_image) one call runs, from
  lc.plan_py (or the library's own lf_lsq_plan) and the dispatch in lsq.cu; all_instances() is every one a call can reach.
* Row sums: (A_r, B_r, C_r) = sum_c (w, w x, w c) in fp64 over the kept pixels of an unmasked row, w = (keep act(o))^2.
  The kernel adds, per lane, V sequential terms per column step (sa +=, sb = fmaf(w, x, sb), sc = fmaf(w, c, sc), c an
  exact integer), then the column steps' partials into one fp32 accumulator per row (`#pragma unroll UNR` unrolls the
  loop but does not split the accumulator: without fast-math the compiler does not reassociate fp32 additions), then a
  five-level warp butterfly.  So each term passes through at most NADD = V + ceil(W / (32 V)) + 5 rounded adds, as in
  lc.forward_reference:
      e_A <= sum_c ew + NADD u sum_c w,   e_B likewise with |x|,   e_C likewise with c,
  ew = 2 |a| e_a + u w + 2^-149 per pixel (e_a from lc.act_err; 0 where keep is 0: the kernel stores +0.0 there).  The
  gate is SECOND (e + W u64 S) + TINY, the second term for the fp64 reference's own sums.  Were the column steps split
  over UNR partial accumulators added in order at the end, a chain would be V + ceil(steps / UNR) + min(UNR, steps) - 1 + 5
  <= NADD; the CPU test runs both orders.  Rows < mask_rows are not written.
* Grid gradient, per row r >= mask_rows, summed over the systems s of the call (all B L, or image b's L):
      z = Zinv g,  phi = [y^d .. y 1],  phi' = d phi / dy,
      g_alpha = sum_s (phi.z) C,  g_gamma = sum_s (phi.z) A,
      g_y'    = -sum_s [ (phi'.z)(B - (phi.beta) A) - (phi.z)(phi'.beta) A ]
  evaluated EXACTLY (fractions.Fraction) from the kernel's own fp32 row sums and yrow and the fp64 beta, Zinv, g handed
  to it.  The kernel evaluates the same expression in fp64, so |got - exact| <= gamma_k S with S the expression in
  absolute values (|Zinv| |g| for z, |y| for y, and B + |phi.beta| A for the residual) and k the longest chain of
  roundings from an input to an output, counted from lsq_grid_grad_row:
      powers of y by products: d;  k y^(k-1) by pwm = pwm y + pw: 2 d on top of the powers' d;  z_i: n products and adds;
      phi.z, phi'.z, phi.beta, phi'.beta: n + 1;  the row's terms: 6;  the sum over the nbl systems: nbl
      k = 3 d + 3 n + 7 + nbl,  gate = SECOND (k + 2) u64 S   (+2: the exact value's rounding to fp64, and slack).
  Masked rows are exactly 0.
* Per-image fit: lc.forward_reference / lc.backward_reference per image on that image's xtab[b], yrow[b], with the
  nchunks of the B-image plan.  Prefix fit: the references on o[:, :L] of a [B, Lmap, H, W] map; d_o of lanes
  [L, Lmap) must be +0.0 bit for bit.
* Emulations in the kernel's order: emulate_rowsums (fp32), emulate_grid_grad (fp64); the fits reuse lc.emulate_*.
* Mutations, each of which must put the emulation (and the GPU result) outside the gate:
  grid gradient: Zinv transposed, g_y' with the sign of dL/dy, the -(phi.z)(phi'.beta) A term dropped, A and C swapped,
  the row sums of row r + 1, row mask_rows - 1 included; per image: the sum over every image, every image on image 0's
  tables; prefix fit: lanes read with stride L instead of Lmap; row sums: the column index one off.
"""
from fractions import Fraction

import numpy as np

import lsq_contract as lc

U, U64 = lc.U, lc.U64

# ---------------------------------------------------------------------------------------------------------------------
# instances
# ---------------------------------------------------------------------------------------------------------------------
# (kernel, activation template, dtype, NL, ROWSUMS, KEEP, per_image); "-" where a kernel has no such parameter


def entry_name(bwd, per_image=False, rowsums=False, keep=False, lanes=False):
    """The C entry point of a (direction, table kind, row sums, keep map, prefix fit) combination."""
    sfx = "_lanes" if lanes else ""
    if per_image:
        return ("lf_lsq_bwd_per_image" if bwd else "lf_lsq_fwd_per_image") + sfx
    if bwd:
        return "lf_lsq_bwd" + ("_keep" if keep else "") + sfx
    return "lf_lsq_fwd" + ("_rowsums" if rowsums else "") + ("_keep" if keep else "") + sfx


def launched(entry, dtype, act, B, L, Lmap, H, W, order, mask_rows, has_yrow=True, has_ytab=False, keep=False,
             rowsums=False, plan=None):
    """(rc, instance) of one call of `entry` (the per-image entry points take keep / rowsums as optional operands, the
    others by name).  plan(bwd, dtype, has_yrow, has_ytab, B, L, H, W, order, mask_rows, act) -> (rc, plan dict):
    lc.plan_py (default, with 132 SMs) or lc.query_plan."""
    if entry in ("lf_lsq_grid_grad", "lf_lsq_grid_grad_per_image"):
        pi = int(entry.endswith("per_image"))
        return 0, ("grid_grad_pi" if pi else "grid_grad", "-", "-", 0, 0, 0, pi)
    plan = plan or (lambda *a: lc.plan_py(*a, sms=132))
    bwd = "_bwd" in entry
    lanes = entry.endswith("_lanes")
    pi = "per_image" in entry
    rs = int(not bwd and (rowsums if pi else "rowsums" in entry))
    kp = int(keep if pi else "_keep" in entry)
    if not lanes:
        Lmap = L
    if not (L <= Lmap <= 65535):
        return lc.INVALID, None
    if pi or rs:
        has_yrow, has_ytab = True, False        # these entry points plan with yrow and without ytab
    rc, p = plan(int(bwd), dtype, has_yrow, has_ytab, B, L, H, W, order, mask_rows, act)
    if rc != 0:
        return rc, None
    if (pi or rs) and not p["rowsep"]:
        return lc.INVALID, None
    a = "square" if p["act_t"] == lc.ACT_SQUARE else "runtime"
    dt = "bf16" if dtype == lc.LF_BF16 else "f32"
    d = "bwd" if bwd else "fwd"
    if lanes and Lmap > L:
        if p["rowsep"]:
            return 0, (d + "_rowsep_lanes", a, dt, p["nl"], rs, kp, int(pi))
        return 0, (d + "_general_lanes", a, dt, 1, 0, kp, 0)
    if pi:
        return 0, (d + "_rowsep_pi", a, dt, p["nl"], rs, kp, 1)
    if rs:
        return 0, ("fwd_rowsums", a, dt, p["nl"], 1, kp, 0)
    # the plain kernels (tests/lsq_contract.py and the keep tests cover them)
    return 0, (d + ("_rowsep" if p["rowsep"] else "_general"), a, dt, p["nl"] if p["rowsep"] else 1, 0, kp, 0)


def all_instances():
    """Every instance the table entry points can reach."""
    out = {("grid_grad", "-", "-", 0, 0, 0, 0), ("grid_grad_pi", "-", "-", 0, 0, 0, 1)}
    for a in ("square", "runtime"):
        for dt in ("f32", "bf16"):
            for kp in (0, 1):
                out.add(("fwd_general_lanes", a, dt, 1, 0, kp, 0))
                out.add(("bwd_general_lanes", a, dt, 1, 0, kp, 0))
                for nl in (1, 2, 3, 4):
                    out.add(("fwd_rowsums", a, dt, nl, 1, kp, 0))
                    out.add(("bwd_rowsep_pi", a, dt, nl, 0, kp, 1))
                    for pi in (0, 1):
                        out.add(("bwd_rowsep_lanes", a, dt, nl, 0, kp, pi))
                    for rs in (0, 1):
                        out.add(("fwd_rowsep_pi", a, dt, nl, rs, kp, 1))
                        for pi in (0, 1):
                            out.add(("fwd_rowsep_lanes", a, dt, nl, rs, kp, pi))
    return out


def case_calls(c):
    """(entry, keep, rowsums) of every call a coverage case makes: on a row-separable plan every table entry point,
    keep and row sums on and off; on the general plan the prefix fits (the only table entry points it can take)."""
    rowsep = lc.plan_py(0, c["dtype"], c["yrow"], True, c["B"], c["L"], c["H"], c["W"], c["order"], c["mask_rows"],
                        c["act"], sms=132)[1]["rowsep"]
    calls = []
    for kp in (False, True):
        calls += [(entry_name(0, keep=kp, lanes=True), kp, False), (entry_name(1, keep=kp, lanes=True), kp, False)]
        if not rowsep:
            continue
        calls += [(entry_name(0, rowsums=True, keep=kp), kp, True), (entry_name(0, rowsums=True, keep=kp, lanes=True), kp, True),
                  (entry_name(1, per_image=True), kp, False), (entry_name(1, per_image=True, lanes=True), kp, False)]
        for rs in (False, True):
            calls += [(entry_name(0, per_image=True), kp, rs), (entry_name(0, per_image=True, lanes=True), kp, rs)]
    if rowsep:
        calls += [("lf_lsq_grid_grad", False, True), ("lf_lsq_grid_grad_per_image", False, True)]
    return calls


def case_instance(c, call, plan=None):
    entry, kp, rs = call
    return launched(entry, c["dtype"], c["act"], c["B"], c["L"], c["Lmap"], c["H"], c["W"], c["order"], c["mask_rows"],
                    c["yrow"], True, kp, rs, plan)


# ---------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------
def keep_map(H, W, seed):
    """A keep map with isolated holes, whole masked columns and a masked corner; any nonzero byte keeps a pixel."""
    rng = np.random.default_rng(seed)
    k = (rng.uniform(size=(H, W)) > 0.2).astype(np.uint8)
    k[:, 1:min(3, W)] = 0
    k[:H // 3, W - W // 4:] = 0
    k[k != 0] = rng.integers(1, 256, size=int((k != 0).sum()))
    return k


def zeroed(o, keep, act):
    """o with the pixels keep drops replaced by a value whose activation is exactly 0 in lc.act64."""
    fill = -np.inf if lc.ACTS[act] in ("sigmoid", "softplus") else 0.0
    return np.where(keep[None, None] != 0, o, fill)


def per_image_tables(xtab, yrow, B, H, W):
    """(xtab [B, H*W], yrow [B, H]) fp32: image b's x scaled by 1 + b / 4 and moved by 3 b, its y scaled by 1 + b / 10,
    so that every power of y, and so every coefficient of the fit, differs between images."""
    x = np.asarray(xtab, np.float64).reshape(1, H * W)
    y = np.asarray(yrow, np.float64).reshape(1, H)
    b = np.arange(B, dtype=np.float64)[:, None]
    return (x * (1.0 + 0.25 * b) + 3.0 * b).astype(np.float32), (y * (1.0 + 0.1 * b)).astype(np.float32)


def case_operands(c, seed=0):
    """(o [B, Lmap, H, W] fp32 (bf16-exact for bf16 cases), xtab, ytab, yrow, per-image xtab, per-image yrow, keep) of a
    coverage case: lc.case_operands' values (softplus threshold, large |o| for sigmoid) on every one of the Lmap lanes."""
    o, xtab, ytab, yrow = lc.case_operands(dict(c, L=c["Lmap"]), seed)
    xs, ys = per_image_tables(xtab, yrow, c["B"], c["H"], c["W"])
    return o, xtab, ytab, yrow, xs, ys, keep_map(c["H"], c["W"], 7 + sum(map(ord, c["name"])))


def stride_l_view(o, L):
    """What the prefix-fit kernels would read without the b * (Lmap - L) shift: the first B L maps of o, as [B, L, H, W]."""
    B, _, H, W = o.shape
    return np.ascontiguousarray(o).reshape(-1)[:B * L * H * W].reshape(B, L, H, W)


# ---------------------------------------------------------------------------------------------------------------------
# row sums
# ---------------------------------------------------------------------------------------------------------------------
def nadd(W, dtype):
    V = 8 if dtype == lc.LF_BF16 else 4
    return V + -(-W // (32 * V)) + 5


def rowsums_reference(o, xtab, H, W, mask_rows, act, dtype, keep=None, mut=None):
    """(ref, bound) [B, L, H - mask_rows, 3] fp64 of the unmasked rows' (A, B, C).  o: exact values (fp64) [B, L, H, W].
    mut: ("col_shift",) -- C with the column index one off."""
    mr = mask_rows
    ov = np.asarray(o, np.float64)[:, :, mr:]
    a, _ = lc.act64(ov, act)
    ea, _ = lc.act_err(ov, act)
    if keep is not None:
        kk = (np.asarray(keep)[mr:] != 0)[None, None]
        a, ea = np.where(kk, a, 0.0), np.where(kk, ea, 0.0)
    w = a * a
    ew = np.where(w > 0, 2 * np.abs(a) * ea + U * w + 2.0 ** -149, 2 * np.abs(a) * ea)
    x = np.asarray(xtab, np.float64).reshape(H, W)[mr:]
    cols = np.arange(W, dtype=np.float64) + (1.0 if mut and mut[0] == "col_shift" else 0.0)
    k = nadd(W, dtype)
    ref, bound = [], []
    for f in (1.0, x, cols):
        af = np.abs(f) * np.ones_like(w)
        s = (w * af).sum(-1)
        ref.append((w * f).sum(-1))
        bound.append(lc.SECOND * ((ew * af).sum(-1) + k * U * s + W * U64 * s) + lc.TINY)
    return np.stack(ref, -1), np.stack(bound, -1)


def emulate_rowsums(o32, xtab, H, W, mask_rows, act, dtype, keep=None, split=1, ulps=(None, None)):
    """(A, B, C) [B, L, H - mask_rows, 3] as the kernel forms them in fp32: per lane V sequential terms per column step,
    the column steps into `split` partial accumulators (1: the kernel; the unroll factor UNR: a compiler that split
    them) added in order at the end, then the xor butterfly."""
    f = np.float32
    V = 8 if dtype == lc.LF_BF16 else 4
    WV = W // V
    steps = -(-WV // 32)
    mr = mask_rows
    v = lc._act_f32(np.asarray(o32, f)[:, :, mr:], act, *ulps)
    if keep is not None:
        v = np.where((np.asarray(keep)[mr:] != 0)[None, None], v, f(0))
    w = (v * v).astype(f)
    Bn, L, R = w.shape[:3]
    pad = steps * 32 * V - W
    wp = np.concatenate([w, np.zeros((Bn, L, R, pad), f)], -1).reshape(Bn, L, R, steps, 32, V)
    x = np.asarray(xtab, f).reshape(H, W)[mr:]
    xp = np.concatenate([x, np.zeros((R, pad), f)], -1).reshape(1, 1, R, steps, 32, V)
    cp = np.concatenate([np.arange(W, dtype=f), np.zeros(pad, f)]).reshape(steps, 32, V)
    acc = np.zeros((3, split, Bn, L, R, 32), f)
    for st in range(steps):
        sa = np.zeros((Bn, L, R, 32), f)
        sb = np.zeros((Bn, L, R, 32), f)
        sc = np.zeros((Bn, L, R, 32), f)
        for e in range(V):
            we = wp[..., st, :, e]
            sa = sa + we
            sb = (we.astype(np.float64) * xp[..., st, :, e] + sb).astype(f)       # fmaf
            sc = (we.astype(np.float64) * cp[st, :, e] + sc).astype(f)
        for i, s in enumerate((sa, sb, sc)):
            acc[i, st % split] = acc[i, st % split] + s
    tot = acc[:, 0]
    for p in range(1, split):
        tot = tot + acc[:, p]
    for m in (16, 8, 4, 2, 1):
        tot = tot[..., :m] + tot[..., m:2 * m]
    return np.moveaxis(tot[..., 0], 0, -1).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# grid gradient
# ---------------------------------------------------------------------------------------------------------------------
def gg_chain(order, nbl):
    n = order + 1
    return 3 * order + 3 * n + 7 + nbl


def _gg_groups(B, L, per_image):
    """Systems summed into each output: [range(B L)] for the shared tables, [range(b L, b L + L)] per image."""
    return [range(b * L, b * L + L) for b in range(B)] if per_image else [range(B * L)]


def grid_grad_reference(rowsums, yrow, beta, zinv, gbeta, B, L, H, order, mask_rows, per_image):
    """(ref, bound): [H, 3] (shared tables) or [B, H, 3] (per image) fp64.  rowsums [B L, H, 3] (the kernel's fp32 values),
    yrow [H] or [B, H], beta [B L, n], zinv [B L, n, n], gbeta [B L, n].  ref is the exact value rounded to fp64."""
    n = order + 1
    rs = np.asarray(rowsums, np.float64).reshape(B * L, H, 3)
    beta, zinv, gbeta = (np.asarray(v, np.float64).reshape(B * L, *s) for v, s in
                         ((beta, (n,)), (zinv, (n, n)), (gbeta, (n,))))
    yr = np.asarray(yrow, np.float64).reshape(-1, H)
    F = Fraction
    zF = [[sum((F(zinv[s, i, j]) * F(gbeta[s, j]) for j in range(n)), F(0)) for i in range(n)] for s in range(B * L)]
    bF = [[F(v) for v in beta[s]] for s in range(B * L)]
    za = np.abs(zinv) @ np.abs(gbeta)[..., None]
    za = za[..., 0]                                                     # [S, n]  |Zinv| |g|
    groups = _gg_groups(B, L, per_image)
    ref = np.zeros((len(groups), H, 3))
    bound = np.zeros((len(groups), H, 3))
    for gi, sys_ in enumerate(groups):
        y64 = yr[gi if per_image else 0]
        k = gg_chain(order, len(sys_))
        for r in range(mask_rows, H):
            y = F(float(y64[r]))
            phi = [y ** (order - i) for i in range(n)]
            dphi = [(order - i) * y ** (order - i - 1) if order - i > 0 else F(0) for i in range(n)]
            ay = abs(float(y64[r]))
            aphi = np.array([ay ** (order - i) for i in range(n)])
            adphi = np.array([(order - i) * ay ** (order - i - 1) if order - i > 0 else 0.0 for i in range(n)])
            ga = gg = gy = F(0)
            sa = sg = sy = 0.0
            for s in sys_:
                A, Bs, C = (F(float(v)) for v in rs[s, r])
                z, bt = zF[s], bF[s]
                pz = sum((p * q for p, q in zip(phi, z)), F(0))
                dz = sum((p * q for p, q in zip(dphi, z)), F(0))
                pb = sum((p * q for p, q in zip(phi, bt)), F(0))
                db = sum((p * q for p, q in zip(dphi, bt)), F(0))
                gg += pz * A
                ga += pz * C
                gy += dz * (Bs - pb * A) - pz * db * A
                apz, adz = float(aphi @ za[s]), float(adphi @ za[s])
                apb, adb = float(aphi @ np.abs(beta[s])), float(adphi @ np.abs(beta[s]))
                aA, aB, aC = abs(rs[s, r, 0]), abs(rs[s, r, 1]), abs(rs[s, r, 2])
                sg += apz * aA
                sa += apz * aC
                sy += adz * (aB + apb * aA) + apz * adb * aA
            ref[gi, r] = (float(ga), float(gg), float(-gy))
            bound[gi, r] = lc.SECOND * (k + 2) * U64 * np.array([sa, sg, sy])
    return (ref if per_image else ref[0]), (bound if per_image else bound[0])


def emulate_grid_grad(rowsums, yrow, beta, zinv, gbeta, B, L, H, order, mask_rows, per_image, mut=None, below=None):
    """g_rowp in fp64 in lsq_grid_grad_row's order (vectorised over rows), or a mutation of it:
    ("zinv_t",), ("dy_sign",), ("drop_term",), ("swap_ac",), ("next_row",), ("all_images",), ("image0_y",), and
    ("row_below_mask",) with below = the fp64 row sums [B L, 3] of row mask_rows - 1."""
    kind = mut[0] if mut else None
    n = order + 1
    rs = np.asarray(rowsums, np.float64).reshape(B * L, H, 3).copy()
    beta, zinv, gbeta = (np.asarray(v, np.float64).reshape(B * L, *s) for v, s in
                         ((beta, (n,)), (zinv, (n, n)), (gbeta, (n,))))
    yr = np.asarray(yrow, np.float64).reshape(-1, H)
    if kind == "zinv_t":
        zinv = np.swapaxes(zinv, 1, 2)
    if kind == "swap_ac":
        rs = rs[..., [2, 1, 0]]
    if kind == "next_row":
        rs[:, :-1] = rs[:, 1:]
    mr = mask_rows
    if kind == "row_below_mask":
        mr = mask_rows - 1
        rs[:, mr] = np.asarray(below, np.float64).reshape(B * L, 3)
    if kind == "image0_y":
        yr = np.repeat(yr[:1], yr.shape[0], 0)
    groups = _gg_groups(B, L, per_image and kind != "all_images")
    if kind == "all_images":
        groups = groups * B
    out = np.zeros((len(groups), H, 3))
    rows = np.arange(mr, H)
    for gi, sys_ in enumerate(groups):
        y = yr[gi if per_image else 0][rows]
        with np.errstate(all="ignore"):
            phi = np.zeros((n, len(rows)))
            dphi = np.zeros((n, len(rows)))
            pw, pwm = np.ones_like(y), np.zeros_like(y)
            for i in range(order, -1, -1):
                phi[i], dphi[i] = pw, pwm
                pwm = pwm * y + pw
                pw = pw * y
            ga = np.zeros_like(y)
            gg = np.zeros_like(y)
            gy = np.zeros_like(y)
            for s in sys_:
                pz = dz = pb = db = 0.0
                for i in range(n):
                    z = 0.0
                    for j in range(n):
                        z += zinv[s, i, j] * gbeta[s, j]
                    pz = pz + phi[i] * z
                    dz = dz + dphi[i] * z
                    pb = pb + phi[i] * beta[s, i]
                    db = db + dphi[i] * beta[s, i]
                A, Bs, C = rs[s, rows, 0], rs[s, rows, 1], rs[s, rows, 2]
                gg = gg + pz * A
                ga = ga + pz * C
                gy = gy + (dz * (Bs - pb * A) if kind == "drop_term" else dz * (Bs - pb * A) - pz * db * A)
        out[gi, rows] = np.stack([ga, gg, gy if kind == "dy_sign" else -gy], -1)
    return out if per_image else out[0]


def grid_grad_mutations(c, per_image):
    """The mutations of the grid gradient that apply to a case (at order 0 phi' = 0, Zinv is 1 x 1 and y is not used)."""
    H, mr = c["H"], c["mask_rows"]
    if mr >= H:
        return []
    m = [("swap_ac",), ("next_row",)] if H - mr >= 2 else [("swap_ac",)]
    if c["order"] > 0:
        m += [("zinv_t",), ("dy_sign",), ("drop_term",)]
    if mr > 0:
        m.append(("row_below_mask",))
    if per_image:
        m += [("all_images",)] + ([("image0_y",)] if c["order"] > 0 else [])
    return m


def row_below_mask(o, xtab, H, W, mask_rows, act, dtype, keep=None):
    """The fp64 row sums [B, L, 3] of row mask_rows - 1 (xtab [H*W], or [B, H*W] per image)."""
    xs = np.asarray(xtab).reshape(-1, H * W)
    parts = [rowsums_reference(o[b:b + 1], xs[b if len(xs) > 1 else 0], H, W, mask_rows - 1, act, dtype, keep)[0][:, :, 0]
             for b in range(o.shape[0])]
    return np.concatenate(parts)


# ---------------------------------------------------------------------------------------------------------------------
# fits on per-image tables and prefix fits
# ---------------------------------------------------------------------------------------------------------------------
def per_image_forward_reference(o, xs, ys, H, W, order, mask_rows, act, reg_ls, nchunks, dtype, mut=None):
    """lc.forward_reference per image on its own tables; mut ("image0",): every image on image 0's tables."""
    parts = []
    for b in range(o.shape[0]):
        t = 0 if mut and mut[0] == "image0" else b
        parts.append(lc.forward_reference(o[b:b + 1], xs[t], ys[t], H, W, order, mask_rows, act, reg_ls, True, nchunks,
                                          dtype))
    return {k: np.concatenate([p[k] for p in parts]) for k in ("beta", "zinv", "bound_beta", "bound_zinv", "rho")}


def per_image_backward_reference(o, xs, ys, H, W, order, mask_rows, act, beta, zinv, g, dtype, got, mut=None):
    refs, bounds = [], []
    for b in range(o.shape[0]):
        t = 0 if mut and mut[0] == "image0" else b
        r, bd = lc.backward_reference(o[b:b + 1], xs[t], ys[t], H, W, order, mask_rows, act, beta[b:b + 1],
                                      zinv[b:b + 1], g[b:b + 1], True, dtype, None if got is None else got[b:b + 1])
        refs.append(r)
        bounds.append(bd)
    return np.concatenate(refs), np.concatenate(bounds)


def emulate_per_image_forward(o32, xs, ys, H, W, order, mask_rows, act, reg_ls, dtype):
    parts = [lc.emulate_forward_rowsep(o32[b:b + 1], xs[b], ys[b], H, W, order, mask_rows, act, reg_ls, dtype)
             for b in range(o32.shape[0])]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def emulate_per_image_backward(o32, xs, ys, H, W, order, mask_rows, act, beta, zinv, g):
    return np.concatenate([lc.emulate_backward(o32[b:b + 1], xs[b], ys[b], H, W, order, mask_rows, act, beta[b:b + 1],
                                               zinv[b:b + 1], g[b:b + 1], True) for b in range(o32.shape[0])])


# ---------------------------------------------------------------------------------------------------------------------
# the GPU coverage table
# ---------------------------------------------------------------------------------------------------------------------
# (name, dtype, act, L, Lmap, H, W, B, order, solver, reg_ls, mask_rows, grid, yrow given); every case runs every
# entry point of case_calls().  Sizes keep the exact solves and the exact grid gradient small: B L systems of at most
# 5 x 5 each, and at most B L H = 3 840 (row, system) pairs in Fractions.
COVERAGE = [
    ("sq_f32_nl1_h129_w132", lc.LF_F32, 1, 1, 2, 129, 132, 3, 2, 0, 0.0, 0, "bev", True),
    ("sq_f32_nl2_w4", lc.LF_F32, 1, 2, 9, 9, 4, 4, 1, 1, 1e-3, 1, "bp", True),
    ("sq_f32_nl3_L5_h127", lc.LF_F32, 1, 5, 6, 127, 8, 3, 0, 0, 0.0, 120, "bev", True),
    ("sq_f32_nl4_L7_h1", lc.LF_F32, 1, 7, 9, 1, 136, 3, 2, 0, 1.0, 0, "bev", True),
    ("sq_bf16_nl1_h320_cap", lc.LF_BF16, 1, 1, 3, 320, 8, 3, 4, 0, 0.0, 0, "bev", True),
    ("sq_bf16_nl2_allmasked", lc.LF_BF16, 1, 2, 4, 64, 136, 5, 3, 0, 1.0, 64, "bev", True),
    ("sq_bf16_nl3_L6", lc.LF_BF16, 1, 6, 7, 33, 16, 3, 1, 1, 0.0, 5, "bp", True),
    ("sq_bf16_nl4_w264", lc.LF_BF16, 1, 4, 5, 128, 264, 3, 2, 0, 0.0, 52, "bev", True),
    ("sigmoid_f32_nl1_h127", lc.LF_F32, 4, 1, 3, 127, 136, 3, 0, 1, 1e-3, 8, "bev", True),
    ("softplus_f32_nl2_h129", lc.LF_F32, 5, 2, 3, 129, 132, 3, 3, 0, 0.0, 52, "bev", True),
    ("abs_f32_nl3_w4", lc.LF_F32, 2, 3, 9, 7, 4, 16, 1, 0, 1.0, 1, "bp", True),
    ("relu_f32_nl4_h320_cap", lc.LF_F32, 3, 4, 5, 320, 100, 3, 2, 1, 0.0, 0, "bp", True),
    ("none_bf16_nl1_h1_allmasked", lc.LF_BF16, 0, 1, 2, 1, 8, 3, 0, 0, 1.0, 1, "bev", True),
    ("sigmoid_bf16_nl2", lc.LF_BF16, 4, 2, 5, 9, 512, 8, 4, 1, 1.0, 0, "bev", True),
    ("softplus_bf16_nl3_L5", lc.LF_BF16, 5, 5, 9, 64, 136, 3, 2, 0, 1e-3, 1, "bp", True),
    ("none_bf16_nl4_L7", lc.LF_BF16, 0, 7, 8, 7, 640, 3, 3, 0, 0.0, 0, "bev", True),
    ("sq_f32_general_w98", lc.LF_F32, 1, 3, 4, 9, 98, 3, 2, 0, 0.0, 1, "bev", True),
    ("sq_bf16_general_w100", lc.LF_BF16, 1, 2, 5, 7, 100, 3, 1, 1, 0.0, 0, "bp", True),
    ("softplus_f32_general", lc.LF_F32, 5, 2, 3, 129, 64, 3, 3, 0, 0.0, 77, "bev", False),
    ("sigmoid_bf16_general", lc.LF_BF16, 4, 1, 2, 127, 96, 3, 2, 1, 0.0, 64, "bp", False),
]
CASE_FIELDS = ("name", "dtype", "act", "L", "Lmap", "H", "W", "B", "order", "solver", "reg_ls", "mask_rows", "grid",
               "yrow")


def case_dict(case):
    return dict(zip(CASE_FIELDS, case))
