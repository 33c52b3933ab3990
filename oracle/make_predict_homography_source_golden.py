"""Generate tests/golden/predict_homography_source_*.npz for the predicted per-image homography in the source-corner
parametrisation (--predict_homography_corners source) from the UNMODIFIED reference's own modules on the CPU, in float64
(TEST INFRASTRUCTURE; run in the build container: ``python -m oracle.make_predict_homography_source_golden``).

The chain, per case (B images):
  encoder map E [B, 128, 32, 64] -> the reference's ``Spatial_transformer_net`` (loaded as make_predict_homography_golden
  loads it, BatchNorm in training mode) with a 5-output ``fully_connected2`` -> z [B, 5] -> theta = tanh(z) / 64 ->
  get_homography(resize)'s source corners shifted by theta (x of the four corners by theta_0..3 * 2R, the top row by
  theta_4 * R) -> per image a float64 torch solve of the 8x8 perspective system (differentiable, for dL/dz) ->
  the reference's ``ProjectiveGridGenerator`` fed the per-image M -> act(o) with the row mask (and, with
  --trapezium_mask, the reference constructor's column / corner masks) -> the reference's ``Weighted_least_squares`` ->
  the reference's ``backprojection_loss`` with M_inv, y_prime and Y set per image, averaged over the lanes.

Stored per case: z, each image's M and M^-1 from ``cv2.getPerspectiveTransform`` on the shifted corners in float32 (as
get_homography calls it), beta, the loss, dL/dz and per entry the sum of the absolute chain-rule terms through the grid
and the loss constants (``gz_abs``), as make_predict_homography_golden stores them.  Unlike the destination
parametrisation, the loss depends on z here, but its total can still cancel far below its terms (2 lanes far from their
targets), so dL/dz is gated against ``gz_abs``; and the branch's backward is pinned, as there, on a fixed cotangent
v [B, 5]: sampled gradients of sum(z * v) with respect to the encoder map and the branch's weights.
"""
import json
import os
import zlib
from math import ceil

import cv2
import numpy as np
import torch

from . import inputs
from .make_golden import GOLDEN_DIR, summarize
from .make_predict_homography_golden import SAMPLED, branch_weights, encoder_map, load_least_squares_net

CASES = [
    # name, L, order, mask_pct, trapezium, B
    ("predict_homography_source_l2_d2", 2, 2, 0.3, False, 2),
    ("predict_homography_source_l4_d3_trapezium", 4, 3, 0.2, True, 2),
]


def source_branch_weights(seed):
    """branch_weights(seed) with a 5-output fully_connected2, drawn at the same scale (float32 numpy)."""
    w = branch_weights(seed)
    rng = np.random.default_rng(seed + 1000)
    w["fully_connected2.weight"] = (rng.standard_normal((5, 128)) * 0.05).astype(np.float32)
    w["fully_connected2.bias"] = (rng.standard_normal(5) * 0.01).astype(np.float32)
    return w


def cotangent(B, seed):
    """The fixed cotangent v [B, 5] float64 of the branch's backward check."""
    return np.random.default_rng(seed).standard_normal((B, 5))


def source_corners(theta, R):
    """(src [4, 2], dst [4, 2]) of get_homography(resize) with the source corners shifted by theta [5]; float64 torch,
    differentiable in theta."""
    f = lambda v: float(np.float32(v))
    w = 2 * R
    c = lambda v: torch.as_tensor(v, dtype=torch.float64)
    top, bot = f(0.20 * R) + theta[4] * R, c(f(R - 1))
    src = torch.stack([torch.stack([f(0.45 * w) + theta[0] * w, top]), torch.stack([f(0.55 * w) + theta[1] * w, top]),
                       torch.stack([f(0.02 * w) + theta[2] * w, bot]), torch.stack([f(0.97 * w) + theta[3] * w, bot])])
    dst = c([[f(0.45 * w), f(0.20 * R)], [f(0.55 * w), f(0.20 * R)], [f(0.45 * w), f(R - 1)], [f(0.55 * w), f(R - 1)]])
    return src, dst


def perspective(src, dst):
    """M (m22 = 1) mapping src to dst by a float64 torch solve of the 8x8 system cv2.getPerspectiveTransform sets up."""
    rows, rhs = [], []
    z, o = torch.zeros((), dtype=torch.float64), torch.ones((), dtype=torch.float64)
    for i in range(4):
        x, y, X, Y = src[i, 0], src[i, 1], dst[i, 0], dst[i, 1]
        rows.append(torch.stack([x, y, o, z, z, z, -X * x, -X * y]))
        rhs.append(X)
        rows.append(torch.stack([z, z, z, x, y, o, -Y * x, -Y * y]))
        rhs.append(Y)
    h = torch.linalg.solve(torch.stack(rows), torch.stack(rhs))
    return torch.cat([h, o.view(1)]).view(3, 3)


def run_case(case, ns, lsn):
    from . import reference_import as ri
    from lanedetection_end2end_b200.Networks.LSQ_layer import trapezium_keep
    name, L, order, mask_pct, trapezium, B = case
    H, W = 256, 512
    seed = zlib.crc32(name.encode()) % 100000
    o_np = inputs.make_lane_maps(B, L, H, W, seed=seed).astype(np.float32)
    E_np = encoder_map(B, seed + 2)
    x_gt, valid = inputs.make_loss_targets(B, 4, seed=seed + 1)
    x_gt = (x_gt * 0.5 + 380.0)                              # targets near where these warps put the lanes
    args = ri.make_args(ns, ["--resize", str(H), "--order", str(order), "--batch_size", str(B), "--nclasses", str(L)])
    zero_rows = ceil(H * mask_pct)
    size = torch.Size([B, L, H, W])

    st = lsn.Spatial_transformer_net((32, 64), 128)
    st.fully_connected2 = torch.nn.Linear(128, 5)
    st = st.double().train()
    st.load_state_dict({k: torch.from_numpy(v).double() for k, v in source_branch_weights(seed + 3).items()}, strict=False)
    E = torch.from_numpy(E_np).double().requires_grad_(True)
    z = st(E)
    z.retain_grad()
    theta = torch.tanh(z) / 64
    pairs = [source_corners(theta[b], H) for b in range(B)]
    M = torch.stack([perspective(s, d) for s, d in pairs])
    Minv = torch.stack([perspective(d, s) for s, d in pairs])
    # cv2 on the same corners in float32, as get_homography calls it
    cv = [(cv2.getPerspectiveTransform(s.detach().numpy().astype(np.float32), d.numpy().astype(np.float32)),
           cv2.getPerspectiveTransform(d.numpy().astype(np.float32), s.detach().numpy().astype(np.float32)))
          for s, d in pairs]
    M_cv, Minv_cv = np.stack([c[0] for c in cv]), np.stack([c[1] for c in cv])
    for a, b in ((M, M_cv), (Minv, Minv_cv)):
        assert np.abs(a.detach().numpy() - b).max() / np.abs(b).max() < 1e-5

    grid = ns.LSQ_layer.ProjectiveGridGenerator(size, M, True)
    ls = ns.LSQ_layer.Weighted_least_squares(size, L, order, True, 0.0, False)
    ls.tensor_ones = ls.tensor_ones.double()
    ls.reg_ls = ls.reg_ls.double()
    o = torch.from_numpy(o_np).double()
    idx_row = torch.linspace(0, zero_rows - 1, zero_rows).long()
    masked = ns.LSQ_layer.activation_layer("square", True)(o).index_fill(2, idx_row, 0)
    if trapezium:
        masked = masked * trapezium_keep(H, zero_rows).double()
    betas = [b for b in ls(masked, grid) if b is not None][:L]

    crit = ns.Loss_crit.backprojection_loss(args)
    y_d = (torch.arange(160, 720, 10) - 80).double() / 2.5
    y_prime = (M[:, 1, 1:2] * y_d + M[:, 1, 2:]) / (M[:, 2, 1:2] * y_d + M[:, 2, 2:])          # [B, 56]
    Y = torch.stack([(255 - y_prime) ** k for k in range(order, 0, -1)] + [torch.ones_like(y_prime)], 2)
    crit.Y, crit.y_prime, crit.M_inv = Y, y_prime.unsqueeze(2), Minv
    loss = 0
    for l in range(L):
        ll, _ = crit(betas[l], torch.from_numpy(x_gt[:, l]), torch.from_numpy(valid[:, l]))
        loss = loss + ll
    loss = loss / L
    grid.retain_grad()
    y_prime.retain_grad()
    Minv.retain_grad()
    Y.retain_grad()
    loss.backward()

    # |terms| of dL/dz_{b,j}: per grid pixel (dL/dgrid . dgrid/dz) and per loss constant (y', Y, M^-1), image by image
    zz = z.detach()

    def parts(zb):
        s, d = source_corners(torch.tanh(zb) / 64, H)
        Mb, Mi = perspective(s, d), perspective(d, s)
        gb = ns.LSQ_layer.ProjectiveGridGenerator(torch.Size([1, L, H, W]), Mb.unsqueeze(0), True)[0]
        yp = (Mb[1, 1] * y_d + Mb[1, 2]) / (Mb[2, 1] * y_d + Mb[2, 2])
        Yb = torch.stack([(255 - yp) ** k for k in range(order, 0, -1)] + [torch.ones_like(yp)], 1)
        return gb, yp, Yb, Mi

    gz_abs = np.zeros((B, 5))
    for b in range(B):
        for j in range(5):
            e = torch.zeros(5, dtype=torch.float64)
            e[j] = 1.0
            _, tang = torch.func.jvp(parts, (zz[b],), (e,))
            grads = (grid.grad[b], y_prime.grad[b], Y.grad[b], Minv.grad[b])
            gz_abs[b, j] = float(sum((g * t).abs().sum() for g, t in zip(grads, tang)))

    beta = torch.stack([b.squeeze(-1) for b in betas], 1)
    out = {"meta": json.dumps(dict(name=name, L=L, order=order, mask_pct=mask_pct, trapezium=trapezium, B=B, H=H, W=W,
                                   seed=seed)),
           "input_sha": inputs.sha256_of(o_np, E_np, x_gt, valid),
           "x_gt": x_gt, "valid": valid, "z_f64": z.detach().numpy(), "M_f64": M_cv, "Minv_f64": Minv_cv,
           "beta_f64": beta.detach().numpy(), "loss_f64": np.array(float(loss)), "gz_f64": z.grad.numpy().copy(),
           "gz_abs": gz_abs}
    # the branch's backward on a fixed cotangent (a second pass through the reference module's graph)
    E2 = torch.from_numpy(E_np).double().requires_grad_(True)
    st.zero_grad()
    v = torch.from_numpy(cotangent(B, seed + 4))
    (st(E2) * v).sum().backward()
    summarize("gE_v_f64", E2.grad, 4096, out)
    sd = dict(st.named_parameters())
    for k in SAMPLED:
        summarize("g_" + k + "_v_f64", sd[k].grad, 1024, out)
    return name, out


def main():
    from . import reference_import as ri
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    ns = ri.import_reference("Backprojection_Loss")
    lsn = load_least_squares_net(ri.REFERENCE_ROOT)
    for case in CASES:
        name, out = run_case(case, ns, lsn)
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), **out)
        print(name, "z", out["z_f64"].ravel(), "gz", out["gz_f64"].ravel(), "abs", out["gz_abs"].ravel(),
              "loss", float(out["loss_f64"]))


if __name__ == "__main__":
    main()
