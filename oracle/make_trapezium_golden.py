"""Generate tests/golden/trapezium_*.npz for --trapezium_mask from the UNMODIFIED reference's own modules on the CPU
(TEST INFRASTRUCTURE; run in the build container: ``python -m oracle.make_trapezium_golden``).

Each case builds the reference's ``Net`` (BP or BEV variant) and takes the masks its constructor builds and leaves
unused: ``idx_row``, ``idx_col1``, ``idx_col2`` and ``idx_mask`` (BP/Networks/LSQ_layer.py:236-246,
Birds_Eye_View_Loss/Networks/LSQ_layer.py:257-266).  It applies them to the ACTIVATED maps, as the commented lines'
own comment asks ("the mask zeroes the weight maps the least-squares layer fits"):

    masked = activation(o).index_fill(2, idx_row, 0).index_fill(3, idx_col1, 0).index_fill(3, idx_col2, 0)
                          .masked_fill(idx_mask, 0)

and runs the reference's ``Weighted_least_squares`` on them in float32 and float64.  The scalar the gradients come
from is the linear loss sum(beta * g) with a stored g = dL/dbeta (oracle/inputs.make_grad_beta), the same upstream
gradient the lsq_*.npz fixtures use.  The --learn_homography case fits on the warp of theta (make_homography_golden's
float64 8x8 solve) so autograd reaches theta.

Stored per case: keep (uint8 [H, W], 1 where no mask is set), beta in f32 / f64, masked (sampled), the loss, d_o
(sampled) in f32 / f64 and, for the warp case, theta and dL/dtheta (f32: the
fp32 maps and fit on the fp32 warp of the same float64 theta).
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
from .make_homography_golden import THETA, warp_fp64

CASES = [
    # name, variant, L, order, act, reg_ls, resize, mask_pct, extra reference flags, learned warp
    ("trapezium_bp_l4_d3_clas", "Backprojection_Loss", 4, 3, "square", 0.0, 256, 0.2, ["--clas", "True"], False),
    ("trapezium_bp_l2_d2_reg_relu", "Backprojection_Loss", 2, 2, "relu", 1.0, 256, 0.3, [], False),
    ("trapezium_bp_l4_d3_homography", "Backprojection_Loss", 4, 3, "square", 0.0, 256, 0.2, [], True),
    ("trapezium_bp_l2_d2_r320", "Backprojection_Loss", 2, 2, "square", 0.0, 320, 0.3, [], False),
    ("trapezium_bev_l2_d2", "Birds_Eye_View_Loss", 2, 2, "square", 0.0, 256, 0.3, [], False),
    ("trapezium_bev_l4_d2_clas", "Birds_Eye_View_Loss", 4, 2, "square", 0.0, 256, 0.3, ["--clas", "True"], False),
]
CASE_FIELDS = ("name", "variant", "L", "order", "act", "reg_ls", "resize", "mask_pct", "flags", "warp")
B = 2


def case_dict(case):
    return dict(zip(CASE_FIELDS, case))


def case_inputs(c):
    """(o [B, L, H, W] float32, g = dL/dbeta [B, L, order+1] float64), regenerated bit-identically from the name."""
    H = c["resize"]
    seed = zlib.crc32(c["name"].encode()) % 100000
    o = inputs.make_lane_maps(B, c["L"], H, 2 * H, seed=seed)
    if c["act"] == "relu":
        o = (o - 0.3) * 4.0          # negative inputs too
    return o.astype(np.float32), inputs.make_grad_beta(B, c["L"], c["order"], seed=7)


def reference_net(ns, c):
    args = ri.make_args(ns, ["--nclasses", str(c["L"]), "--order", str(c["order"]), "--batch_size", str(B),
                             "--resize", str(c["resize"]), "--mask_percentage", str(c["mask_pct"])] + list(c["flags"]))
    return ns.LSQ_layer.Net(args)


def apply_masks(net, a):
    """The reference constructor's masks on the activated maps a [B, L, H, W]."""
    m = a.index_fill(2, net.idx_row, 0)
    m = m.index_fill(3, net.idx_col1, 0)
    m = m.index_fill(3, net.idx_col2, 0)
    return m.masked_fill(net.idx_mask[:a.shape[0], :a.shape[1]].bool(), 0)


def run_case(case):
    c = case_dict(case)
    ns = ri.import_reference(c["variant"])
    L, order, H = c["L"], c["order"], c["resize"]
    W = 2 * H
    torch.manual_seed(0)
    net = reference_net(ns, c)
    keep = (apply_masks(net, torch.ones(1, 1, H, W)) != 0)[0, 0].numpy().astype(np.uint8)
    assert ceil(H * c["mask_pct"]) == len(net.idx_row)
    o_np, g_np = case_inputs(c)
    size = torch.Size([B, L, H, W])
    out = {"meta": json.dumps(dict((k, v) for k, v in c.items())),
           "input_sha": inputs.sha256_of(o_np, g_np), "keep": keep, "g": g_np}
    actf = ns.LSQ_layer.activation_layer(c["act"], True)
    ls = ns.LSQ_layer.Weighted_least_squares(size, L, order, True, c["reg_ls"], False)
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        ls.tensor_ones = ls.tensor_ones.to(dt)
        ls.reg_ls = ls.reg_ls.to(dt)
        theta = None
        if c["warp"]:
            theta = torch.from_numpy(THETA).double().requires_grad_(True)
            M, _ = warp_fp64(theta, H)
            grid = ns.LSQ_layer.ProjectiveGridGenerator(size, M.to(dt).unsqueeze(0).expand(B, 3, 3), True)
        elif c["variant"] == "Backprojection_Loss":
            grid = net.grid.to(dt)
        else:
            grid = net.project_layer(net.M).to(dt)
        # --resize 320: the homography's vanishing line gives non-finite grid rows, all inside the masked top rows; the
        # reference's 0 * inf there is NaN, the kernel never reads those rows.  Zero them so the fit sees what it means.
        grid = torch.where(torch.isfinite(grid), grid, torch.zeros_like(grid))
        o = torch.from_numpy(o_np).to(dt).requires_grad_(True)
        masked = apply_masks(net, actf(o))
        betas = [b for b in ls(masked, grid) if b is not None][:L]
        beta = torch.stack([b.squeeze(-1) for b in betas], 1)          # [B, L, order+1]
        loss = (beta * torch.from_numpy(g_np).to(beta.dtype)).sum()
        loss.backward()
        out["beta_" + tag] = beta.detach().double().numpy()
        out["loss_" + tag] = np.array(float(loss.detach()))
        summarize("grad_" + tag, o.grad, 4096, out)
        if theta is not None:
            out["theta"] = THETA
            out["gtheta_" + tag] = theta.grad.numpy().copy()
        if tag == "f64":
            summarize("masked_f64", masked, 4096, out)
    return c["name"], out


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for case in CASES:
        name, out = run_case(case)
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
        print(name, "kept %.4f" % out["keep"].mean(), "loss", float(out["loss_f64"]),
              "gtheta" if "gtheta_f64" in out else "", out.get("gtheta_f64", ""))


if __name__ == "__main__":
    main()
