"""Generate tests/golden/predict_homography_*.npz for the predicted per-image homography (--predict_homography) from the
UNMODIFIED reference's own modules on the CPU, in float64 (TEST INFRASTRUCTURE; run in the build container:
``python -m oracle.make_predict_homography_golden``).

The chain, per case (B images):
  encoder map E [B, 128, 32, 64] -> the reference's ``Spatial_transformer_net`` (Backprojection_Loss/Networks/
  Least_squares_net.py, BatchNorm in training mode) -> z [B, 3] -> delta = tanh(z) / 16 -> the reference ``DLT.forward``'s
  6x6 equations on the back-projection corners of get_homography(resize), in pixel units, one M per image -> the
  reference's ``ProjectiveGridGenerator`` fed the per-image M -> act(o) with the row mask (and, with --trapezium_mask, the
  reference constructor's column / corner masks) -> the reference's ``Weighted_least_squares`` -> the reference's
  ``backprojection_loss`` with M_inv, y_prime and Y set per image, averaged over the lanes.

Least_squares_net.py imports modules the reference does not ship and calls ``torch.gesv``: it is loaded from the
reference checkout with those imports stubbed (they are only used by networks this chain does not build) and
``torch.gesv`` shimmed to ``torch.linalg.solve``; nothing of it is copied.  The branch's weights come from
``branch_weights(seed)`` (a NumPy generator, so the GPU test rebuilds them without the reference), with a non-zero
``fully_connected2`` so that the images' warps differ.

Stored per case: z, M^-1, beta, the loss, dL/dz and per entry the sum of the absolute chain-rule terms through the grid
and the loss constants (``gz_abs``: the scale a cancelling total is gated against).  The loss does not depend on z in
exact arithmetic (NOTES.md "Predicted homography": the DLT moves the destination corners along a rectangle, an affine
change of the bird's-eye-view coordinates that the fit and the back-projection undo), so dL/dz is rounding and its
backward through the branch carries no signal to compare.  The branch's backward is pinned instead on a fixed cotangent
v [B, 3]: sampled gradients of sum(z * v) with respect to the encoder map and the branch's weights.
"""
import importlib.util
import json
import os
import sys
import types
import zlib
from math import ceil

import numpy as np
import torch

from . import inputs
from .make_golden import GOLDEN_DIR, summarize

CASES = [
    # name, L, order, mask_pct, trapezium, B
    ("predict_homography_l2_d2", 2, 2, 0.3, False, 2),
    ("predict_homography_l2_d2_trapezium", 2, 2, 0.3, True, 2),
    ("predict_homography_l4_d3", 4, 3, 0.2, False, 2),
    ("predict_homography_l4_d3_trapezium", 4, 3, 0.2, True, 2),
]
ENC = (128, 32, 64)              # the ERFNet encoder map the branch reads
SAMPLED = ("conv1.weight", "conv2.weight", "conv3.weight", "conv4.weight", "conv4_bn.weight", "fully_connected1.weight",
           "fully_connected2.weight", "fully_connected2.bias")


def branch_weights(seed):
    """The branch's parameters under the reference's state_dict names (float32 numpy; BatchNorm weight 1, bias 0 as
    nn.BatchNorm2d starts), drawn at the scale of a fan-in init."""
    rng = np.random.default_rng(seed)
    shapes = [("conv1", (128, 128, 1, 1)), ("conv2", (128, 128, 3, 3)), ("conv3", (64, 128, 3, 3)), ("conv4", (64, 64, 3, 3)),
              ("conv5", (64, 64, 3, 3)), ("fully_connected1", (128, 64 * 16 * 32)), ("fully_connected2", (3, 128))]
    w = {}
    for name, shp in shapes:
        fan_in = int(np.prod(shp[1:]))
        scale = 0.05 if name == "fully_connected2" else np.sqrt(2.0 / fan_in)
        w[name + ".weight"] = (rng.standard_normal(shp) * scale).astype(np.float32)
        w[name + ".bias"] = (rng.standard_normal(shp[0]) * 0.01).astype(np.float32)
    for name, c in (("conv1_bn", 128), ("conv2_bn", 128), ("conv3_bn", 64), ("conv4_bn", 64)):
        w[name + ".weight"] = np.ones(c, np.float32)
        w[name + ".bias"] = np.zeros(c, np.float32)
    return w


def cotangent(B, seed):
    """The fixed cotangent v [B, 3] float64 of the branch's backward check."""
    return np.random.default_rng(seed).standard_normal((B, 3))


def encoder_map(B, seed):
    """A ReLU-like encoder map E [B, 128, 32, 64] float32."""
    rng = np.random.default_rng(seed)
    return np.maximum(rng.standard_normal((B,) + ENC), 0.0).astype(np.float32)


def load_least_squares_net(root):
    """The reference's Least_squares_net module, its missing imports stubbed and torch.gesv shimmed."""
    path = os.path.join(root, "Backprojection_Loss", "Networks", "Least_squares_net.py")
    stubs = {"Networks.segnet_long": ["SegNet"], "Networks.Enet_vanilla": ["ENet"], "Networks.unet": ["UNet", "_DecoderBlock"],
             "Networks.vision": ["ResNet18"]}
    saved = {k: sys.modules.get(k) for k in list(stubs) + ["Networks"]}
    try:
        if "Networks" not in sys.modules:
            pkg = types.ModuleType("Networks")
            pkg.__path__ = []
            sys.modules["Networks"] = pkg
        for mod, names in stubs.items():
            m = types.ModuleType(mod)
            for n in names:
                setattr(m, n, type(n, (torch.nn.Module,), {}))
            sys.modules[mod] = m
        if not hasattr(torch, "gesv"):
            torch.gesv = lambda b, a: (torch.linalg.solve(a, b), None)
        spec = importlib.util.spec_from_file_location("reference_least_squares_net", path)
        lsn = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(lsn)
        return lsn
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def dlt_pixel(delta, R):
    """DLT.forward's 6x6 system (A h = B, rows as the reference orders them) on get_homography(resize)'s corners in
    pixel units, one image: delta [3] -> M [3, 3] (m22 = 1), differentiable.  The reference adds delta to normalised
    destination corners; here delta_0 / delta_1 move the left / right column by delta * 2R and delta_2 the top row by
    delta * R."""
    f = lambda v: float(np.float32(v))
    w = 2 * R
    xs_bl, xs_br, xs_tl, xs_tr = f(0.02 * w), f(0.97 * w), f(0.45 * w), f(0.55 * w)
    ys1, ys2 = f(R - 1), f(0.20 * R)                         # source bottom / top rows
    yd1 = f(R - 1)                                           # destination bottom row (fixed)
    xd_l, xd_r = f(0.45 * w) + delta[0] * w, f(0.55 * w) + delta[1] * w
    yd2 = f(0.20 * R) + delta[2] * R
    z, o = torch.zeros((), dtype=torch.float64), torch.ones((), dtype=torch.float64)
    c = lambda v: torch.as_tensor(v, dtype=torch.float64)
    A = torch.stack([
        torch.stack([z, z, z, c(-ys1), -o, c(ys1 * yd1)]),
        torch.stack([c(xs_bl), c(ys1), o, z, z, -ys1 * xd_l]),
        torch.stack([c(xs_br), c(ys1), o, z, z, -ys1 * xd_r]),
        torch.stack([z, z, z, c(-ys2), -o, ys2 * yd2]),
        torch.stack([c(xs_tl), c(ys2), o, z, z, -ys2 * xd_l]),
        torch.stack([c(xs_tr), c(ys2), o, z, z, -ys2 * xd_r])])
    Bv = torch.stack([c(-yd1), xd_l, xd_r, -yd2, xd_l, xd_r])
    h = torch.gesv(Bv.unsqueeze(1), A)[0].squeeze(1)         # the reference's solve, shimmed to torch.linalg.solve
    return torch.stack([h[0], h[1], h[2], z, h[3], h[4], z, h[5], o]).view(3, 3)


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

    st = lsn.Spatial_transformer_net((32, 64), 128).double().train()
    st.load_state_dict({k: torch.from_numpy(v).double() for k, v in branch_weights(seed + 3).items()}, strict=False)
    E = torch.from_numpy(E_np).double().requires_grad_(True)
    z = st(E)
    z.retain_grad()
    delta = torch.tanh(z) / 16
    Ms = [dlt_pixel(delta[b], H) for b in range(B)]
    M = torch.stack(Ms)
    Minv = torch.stack([torch.linalg.inv(m) / torch.linalg.inv(m)[2, 2] for m in Ms])

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
        d = torch.tanh(zb) / 16
        Mb = dlt_pixel(d, H)
        gb = ns.LSQ_layer.ProjectiveGridGenerator(torch.Size([1, L, H, W]), Mb.unsqueeze(0), True)[0]
        yp = (Mb[1, 1] * y_d + Mb[1, 2]) / (Mb[2, 1] * y_d + Mb[2, 2])
        Yb = torch.stack([(255 - yp) ** k for k in range(order, 0, -1)] + [torch.ones_like(yp)], 1)
        Mi = torch.linalg.inv(Mb)
        return gb, yp, Yb, Mi / Mi[2, 2]

    gz_abs = np.zeros((B, 3))
    for b in range(B):
        for j in range(3):
            e = torch.zeros(3, dtype=torch.float64)
            e[j] = 1.0
            _, tang = torch.func.jvp(parts, (zz[b],), (e,))
            grads = (grid.grad[b], y_prime.grad[b], Y.grad[b], Minv.grad[b])
            gz_abs[b, j] = float(sum((g * t).abs().sum() for g, t in zip(grads, tang)))

    beta = torch.stack([b.squeeze(-1) for b in betas], 1)
    out = {"meta": json.dumps(dict(name=name, L=L, order=order, mask_pct=mask_pct, trapezium=trapezium, B=B, H=H, W=W,
                                   seed=seed)),
           "input_sha": inputs.sha256_of(o_np, E_np, x_gt, valid),
           "x_gt": x_gt, "valid": valid, "z_f64": zz.numpy(), "Minv_f64": Minv.detach().numpy(),
           "beta_f64": beta.detach().numpy(), "loss_f64": np.array(float(loss)),
           "gz_f64": z.grad.numpy().copy(), "gz_abs": gz_abs}
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
