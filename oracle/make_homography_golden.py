"""Generate tests/golden/homography_lsq_*.npz for the learned homography (--learn_homography) from the UNMODIFIED
reference's own ``ProjectiveGridGenerator``, ``Weighted_least_squares`` and ``backprojection_loss`` on the CPU, in
float64 (TEST INFRASTRUCTURE; run in the build container: ``python -m oracle.make_homography_golden``).

The reference builds M once with cv2; here M and M^-1 come from theta [5] (get_homography's source corners shifted, see
lanedetection_end2end_b200/homography.py) through a differentiable float64 8x8 solve, and the reference's modules run
on them, so autograd reaches theta.  The loss's y' and Y56 are recomputed from M(theta) by the reference's own formulas
(BP/Loss_crit.py:166-188).  Inputs are oracle/inputs.py's lane maps (regenerated bit-identically; sha256 stored) and
loss targets.

Stored per case: theta, beta, d_o sampled (summarize), theta.grad and, per entry of theta, the sum of the absolute
per-pixel and per-constant terms of the chain rule (``gtheta_abs``) -- the scale a cancelling total is gated against.
"""
import json
import os
import zlib
from math import ceil

import numpy as np
import torch

from . import inputs
from . import reference_import as ri
from .make_golden import GOLDEN_DIR, summarize

CASES = [
    # name, L, order, mask_pct, act, reg_ls, cholesky, B
    ("homography_lsq_l4_d3", 4, 3, 0.2, "square", 0.0, False, 2),
    ("homography_lsq_l2_d2_chol", 2, 2, 0.3, "square", 0.0, True, 2),
    ("homography_lsq_l2_d1_reg_relu", 2, 1, 0.3, "relu", 1.0, False, 2),
]
THETA = np.array([0.004, -0.003, 0.006, -0.005, 0.01], dtype=np.float32)


def warp_fp64(theta, R):
    """M(theta), M^-1(theta) [3,3] float64 by the 8x8 perspective solve (m22 = 1), differentiable in theta."""
    w = 2 * R
    f = lambda v: float(np.float32(v))
    t = theta
    sx = torch.stack([f(0.45 * w) + t[0] * w, f(0.55 * w) + t[1] * w, f(0.02 * w) + t[2] * w, f(0.97 * w) + t[3] * w])
    top = f(0.20 * R) + t[4] * R
    bot = torch.tensor(f(R - 1), dtype=torch.float64)
    sy = torch.stack([top, top, bot, bot])
    dx = torch.tensor([f(0.45 * w), f(0.55 * w), f(0.45 * w), f(0.55 * w)], dtype=torch.float64)
    dy = torch.tensor([f(0.20 * R), f(0.20 * R), f(R - 1), f(R - 1)], dtype=torch.float64)

    def solve(x, y, X, Y):
        z, o = torch.zeros_like(x), torch.ones_like(x)
        A = torch.cat([torch.stack([x, y, o, z, z, z, -X * x, -X * y], 1), torch.stack([z, z, z, x, y, o, -Y * x, -Y * y], 1)])
        m = torch.linalg.solve(A, torch.cat([X, Y]))
        return torch.cat([m, torch.ones(1, dtype=torch.float64)]).view(3, 3)

    return solve(sx, sy, dx, dy), solve(dx, dy, sx, sy)


def loss_constants(ns, args, M, Minv, B):
    """backprojection_loss with M, M^-1 of theta: __init__'s own formulas on the given matrices."""
    crit = ns.Loss_crit.backprojection_loss(args)
    y_d = (torch.arange(160, 720, 10) - 80).double() / 2.5
    y_prime = (M[1, 1:2] * y_d + M[1, 2:]) / (M[2, 1:2] * y_d + M[2, 2:])
    y_eval = 255 - y_prime
    ones = torch.ones(56).double()
    Y = torch.stack([y_eval ** k for k in range(args.order, 0, -1)] + [ones], 1)
    crit.Y = Y.unsqueeze(0).repeat(B, 1, 1)
    crit.y_prime = y_prime.unsqueeze(0).repeat(B, 1).unsqueeze(2)
    crit.M_inv = Minv.unsqueeze(0).repeat(B, 1, 1)
    return crit, y_prime


def run_case(case):
    name, L, order, mask_pct, act, reg_ls, chol, B = case
    ns = ri.import_reference("Backprojection_Loss")
    H, W = 256, 512
    seed = zlib.crc32(name.encode()) % 100000
    o_np = inputs.make_lane_maps(B, L, H, W, seed=seed).astype(np.float32)
    if act == "relu":
        o_np = ((o_np - 0.3) * 4.0).astype(np.float32)
    x_gt, valid = inputs.make_loss_targets(B, 4, seed=seed + 1)
    args = ri.make_args(ns, ["--resize", str(H), "--order", str(order), "--batch_size", str(B), "--nclasses", str(L)])
    zero_rows = ceil(H * mask_pct)
    idx_row = torch.linspace(0, zero_rows - 1, zero_rows).long()
    size = torch.Size([B, L, H, W])

    theta = torch.from_numpy(THETA).double().requires_grad_(True)
    M, Minv = warp_fp64(theta, H)
    grid = ns.LSQ_layer.ProjectiveGridGenerator(size, M.unsqueeze(0).expand(B, 3, 3), True)
    grid.retain_grad()
    ls = ns.LSQ_layer.Weighted_least_squares(size, L, order, True, reg_ls, chol)
    ls.tensor_ones = ls.tensor_ones.double()
    ls.reg_ls = ls.reg_ls.double()
    o = torch.from_numpy(o_np).double().requires_grad_(True)
    masked = ns.LSQ_layer.activation_layer(act, True)(o).index_fill(2, idx_row, 0)
    betas = [b for b in ls(masked, grid) if b is not None][:L]
    crit, y_prime = loss_constants(ns, args, M, Minv, B)
    y_prime.retain_grad()
    crit.M_inv.retain_grad()
    loss = 0
    for l in range(L):
        ll, _ = crit(betas[l], torch.from_numpy(x_gt[:, l]), torch.from_numpy(valid[:, l]))
        loss = loss + ll
    loss = loss / L
    loss.backward()

    # |terms| of the chain rule: per pixel of the grid (dL/dgrid . dgrid/dtheta_j), per sample row and per entry of M^-1
    def grid_of(t):
        Mt, _ = warp_fp64(t, H)
        return ns.LSQ_layer.ProjectiveGridGenerator(torch.Size([1, L, H, W]), Mt.unsqueeze(0), True)[0]

    def consts_of(t):
        Mt, Mit = warp_fp64(t, H)
        y_d = (torch.arange(160, 720, 10) - 80).double() / 2.5
        return torch.cat([((Mt[1, 1] * y_d + Mt[1, 2]) / (Mt[2, 1] * y_d + Mt[2, 2])), Mit.reshape(-1)])

    th = theta.detach()
    g_grid = grid.grad.sum(0)                                       # [HW, 2]: the expanded batch shares one grid
    g_const = torch.cat([y_prime.grad.reshape(-1) if y_prime.grad is not None else torch.zeros(56, dtype=torch.float64),
                         crit.M_inv.grad.sum(0).reshape(-1)])
    absterm = np.zeros(5)
    for j in range(5):
        e = torch.zeros(5, dtype=torch.float64)
        e[j] = 1.0
        _, jg = torch.func.jvp(grid_of, (th,), (e,))
        _, jc = torch.func.jvp(consts_of, (th,), (e,))
        absterm[j] = float((g_grid * jg).abs().sum() + (g_const * jc).abs().sum())

    beta = torch.stack([b.squeeze(-1) for b in betas], 1)
    out = {"meta": json.dumps(dict(name=name, L=L, order=order, mask_pct=mask_pct, act=act, reg_ls=reg_ls, cholesky=chol,
                                   B=B, H=H, W=W, seed=seed)),
           "input_sha": inputs.sha256_of(o_np, x_gt, valid),
           "theta": THETA, "x_gt": x_gt, "valid": valid,
           "beta_f64": beta.detach().numpy(), "loss_f64": np.array(float(loss)),
           "gtheta_f64": theta.grad.numpy().copy(), "gtheta_abs": absterm}
    summarize("grad_f64", o.grad, 4096, out)
    return name, out


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for case in CASES:
        name, out = run_case(case)
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
        print(name, "gtheta", out["gtheta_f64"], "abs", out["gtheta_abs"])


if __name__ == "__main__":
    main()
