"""--predict_homography_corners source on the GPU: each image's tables against lf_homography_tables bit for bit, the
backward against lf_homography_bwd and the host hooks, the reference modules' golden, a warp that learns, and the model:
graphed training against the eager loop, validation, test_model and every convolution mode."""
import numpy as np
import pytest
import torch

from test_epoch_gpu import paths  # noqa: F401  (the synthetic TuSimple directory fixture)
from test_predict_homography_gpu import _args, _loss_inputs

from lanedetection_end2end_b200 import _capi, homography as hg, ops_lsq

pytestmark = pytest.mark.gpu
DEV = "cuda"
p = _capi.ptr
SRC = ("--predict_homography", "True", "--predict_homography_corners", "source")


def _tables(z, R=256, mask_rows=77, corners="source"):
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = hg._PREDICTED_FUNCTIONS[corners].apply(z, R, mask_rows, 255.0, st)
    return out, st


def _z(B, seed, scale=1.0, nz=5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, nz, generator=g) * scale).to(DEV)


def _learned_tables(theta, R, mask_rows):
    f64 = dict(dtype=torch.float64, device=DEV)
    M, Minv, rowp, yk = torch.empty(9, **f64), torch.empty(9, **f64), torch.empty(R, 3, **f64), torch.empty(56, **f64)
    xtab, yrow = torch.empty(R * 2 * R, device=DEV), torch.empty(R, device=DEV)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    _capi.call("lf_homography_tables", p(theta.contiguous()), R, mask_rows, 255.0, p(M), p(Minv), p(rowp), p(xtab),
               p(yrow), p(yk), p(st), _capi.stream_ptr())
    return rowp, Minv, yk, M, xtab, yrow


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [256, 320])
def test_tables_are_the_learned_warps_bits(R):
    B, mask_rows = 6, int(np.ceil(0.3 * R))
    z = _z(B, 1)
    z[-1] = torch.tensor([30.0, -30.0, 30.0, -30.0, 30.0])          # a corner of the box
    (rowp, Minv, yk, M, xtab, yrow, theta), st = _tables(z, R, mask_rows)
    assert int(st.item()) == 0 and theta.dtype == torch.float32 and tuple(theta.shape) == (B, 5)
    assert torch.equal(theta, (torch.tanh(z.double()) / 64).float())
    for b in range(B):
        for got, want in zip((rowp[b], Minv[b], yk[b], M[b], xtab[b], yrow[b]), _learned_tables(theta[b], R, mask_rows)):
            assert torch.equal(got, want)
        th, Mh, Mih, rowph, ykh = hg.predicted_source_warp_host(z[b].cpu().numpy(), R)
        assert np.array_equal(th, theta[b].cpu().numpy())
        for got, ref in ((M[b], Mh), (Minv[b], Mih), (rowp[b, mask_rows:], rowph[mask_rows:]), (yk[b], ykh)):
            got = got.cpu().numpy().reshape(ref.shape)
            assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()


def _cotangents(B, R, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, R, 3, generator=g, dtype=torch.float64).to(DEV),
            torch.randn(B, 9, generator=g, dtype=torch.float64).to(DEV) * 1e-3,
            torch.randn(B, 56, generator=g, dtype=torch.float64).to(DEV) * 1e-2)


def _source_bwd(z, R, mask_rows, g_rowp, g_minv, g_yk):
    B = z.shape[0]
    g_z = torch.empty(B, 5, device=DEV)
    g_theta = torch.empty(B, 5, dtype=torch.float64, device=DEV)
    _capi.call("lf_predicted_homography_source_bwd", p(z), B, R, mask_rows, p(g_rowp), p(g_minv), p(g_yk), p(g_z),
               p(g_theta), _capi.stream_ptr())
    return g_z, g_theta


def test_backward_is_the_learned_warps_sum():
    """With every image on one theta, the images' dL/dtheta sum to lf_homography_bwd's on the summed cotangents within
    reassociation; image by image, g_theta is lf_homography_bwd's reduction."""
    R, B, mask_rows = 256, 4, 77
    z = _z(1, 2).expand(B, 5).contiguous()
    theta = (torch.tanh(z[0].double()) / 64).float()
    g_rowp, g_minv, g_yk = _cotangents(B, R, 3)
    g_z, g_theta = _source_bwd(z, R, mask_rows, g_rowp, g_minv, g_yk)
    want = np.zeros(5)
    sums = [t.sum(0).cpu().numpy().copy() for t in (g_rowp, g_minv, g_yk)]
    th = theta.cpu().numpy()
    assert _capi.lib().lf_homography_bwd_host(th.ctypes.data, R, mask_rows, *(s.ctypes.data for s in sums),
                                              want.ctypes.data) == 0
    got = g_theta.sum(0).cpu().numpy()
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    for b in range(B):
        one = torch.empty(5, device=DEV)
        _capi.call("lf_homography_bwd", p(theta), R, mask_rows, p(g_rowp[b].contiguous()), p(g_minv[b].contiguous()),
                   p(g_yk[b].contiguous()), p(one), _capi.stream_ptr())
        assert torch.equal(g_theta[b].float(), one)
    t = torch.tanh(z.double())
    want_z = (g_theta * ((1 - t * t) / 64)).float()
    assert (g_z - want_z).abs().max().item() <= 1e-6 * want_z.abs().max().item()


def test_backward_matches_the_host_hook():
    R, B, mask_rows = 256, 4, 77
    z = _z(B, 2).requires_grad_(True)
    (rowp, Minv, yk, *_), _ = _tables(z, R, mask_rows)
    g_rowp, g_minv, g_yk = _cotangents(B, R, 3)
    (rowp * g_rowp).sum().add((Minv * g_minv).sum()).add((yk * g_yk).sum()).backward()
    _, g_theta = _source_bwd(z.detach(), R, mask_rows, g_rowp, g_minv, g_yk)
    for b in range(B):
        zb = z[b].detach().cpu().numpy().astype(np.float32)
        ref, ref_theta = np.zeros(5), np.zeros(5)
        gr, gm, gy = (t[b].cpu().numpy().copy() for t in (g_rowp, g_minv, g_yk))
        rc = _capi.lib().lf_predicted_homography_source_bwd_host(zb.ctypes.data, R, mask_rows, gr.ctypes.data,
                                                                 gm.ctypes.data, gy.ctypes.data, ref.ctypes.data,
                                                                 ref_theta.ctypes.data)
        assert rc == 0
        got = z.grad[b].double().cpu().numpy()
        assert np.abs(got - ref.astype(np.float32)).max() <= 1e-6 * np.abs(ref).max()
        assert np.abs(g_theta[b].cpu().numpy() - ref_theta).max() <= 1e-12 * np.abs(ref_theta).max()


# ---------------------------------------------------------------------------------------------------------------------
# the reference modules
# ---------------------------------------------------------------------------------------------------------------------
GOLDEN_CASES = ["predict_homography_source_l2_d2", "predict_homography_source_l4_d3_trapezium"]


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_golden_reference_modules(case, capsys):
    """The branch, the per-image source-corner warps, the fit and the loss against the reference modules' float64 golden
    (oracle/make_predict_homography_source_golden.py), in the default tf32x3 mode, under the destination golden's gates:
    z and each image's M^-1 within 1e-5, beta within 1e-4 and the loss within 1e-5 (norm-wise); dL/dz per entry within
    1e-4 of the sum of its absolute chain-rule terms (the total can cancel far below them); and the branch's backward on a
    fixed cotangent -- sampled gradients of the encoder map and of the branch's weights -- within 1e-4."""
    import json
    import os
    import types
    from math import ceil
    from conftest import GOLDEN
    from oracle import inputs
    from oracle.make_predict_homography_golden import SAMPLED, encoder_map
    from oracle.make_predict_homography_source_golden import cotangent, source_branch_weights
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss, fused_backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import trapezium_keep
    zf = np.load(os.path.join(GOLDEN, case + ".npz"))
    meta = json.loads(str(zf["meta"]))
    B, L, H, W, order, seed = meta["B"], meta["L"], meta["H"], meta["W"], meta["order"], meta["seed"]
    o_np = inputs.make_lane_maps(B, L, H, W, seed=seed).astype(np.float32)
    E_np = encoder_map(B, seed + 2)
    assert inputs.sha256_of(o_np, E_np, zf["x_gt"], zf["valid"]) == str(zf["input_sha"])
    mask = ceil(H * meta["mask_pct"])
    keep = trapezium_keep(H, mask).cuda() if meta["trapezium"] else None
    mod = hg.PredictedHomography(H, mask, corners="source").cuda().train()
    mod.spatial_trans.load_state_dict({k: torch.from_numpy(v) for k, v in source_branch_weights(seed + 3).items()},
                                      strict=False)
    E = torch.from_numpy(E_np).cuda().requires_grad_(True)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    z = mod.spatial_trans(E)
    z.retain_grad()
    rowp, Minv, yk, M, xtab, yrow, theta = hg._PredictedSourceWarpFunction.apply(z, H, mask, 255.0, st)
    warp = hg.WarpTables(rowp, Minv, yk, M, xtab, yrow, H, W, delta=theta)
    mod.current = warp
    crit = backprojection_loss(_args("--order", str(order), "--nclasses", str(L), *SRC, L=L))
    crit.bind(types.SimpleNamespace(DLT=mod))
    o = torch.from_numpy(o_np).cuda()
    beta, _ = ops_lsq.lsq_warp(o, warp, order, mask, "square", 0.0, False, False, st, keep)
    loss, _ = fused_backprojection_loss(crit, [beta[:, l].unsqueeze(-1) for l in range(L)],
                                        torch.from_numpy(zf["x_gt"]).cuda(), torch.from_numpy(zf["valid"]).cuda())
    loss.backward()
    assert int(st.item()) == 0
    nrm = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))
    gz = z.grad.double().cpu().numpy()
    errs = {"z": nrm(z.detach().double().cpu().numpy(), zf["z_f64"]),
            "Minv": max(nrm(Minv[b].detach().cpu().numpy(), zf["Minv_f64"][b].reshape(-1)) for b in range(B)),
            "beta": nrm(beta.detach().cpu().numpy(), zf["beta_f64"]),
            "loss": abs(loss.item() - float(zf["loss_f64"])) / abs(float(zf["loss_f64"])),
            "dL/dz": float((np.abs(gz - zf["gz_f64"]) / zf["gz_abs"]).max())}
    # the branch's backward on the fixed cotangent, a fresh forward
    E2 = torch.from_numpy(E_np).cuda().requires_grad_(True)
    mod.spatial_trans.zero_grad()
    v = torch.from_numpy(cotangent(B, seed + 4)).float().cuda()
    (mod.spatial_trans(E2) * v).sum().backward()
    sd = dict(mod.spatial_trans.named_parameters())
    grads = {"gE_v": E2.grad, **{"g_" + k + "_v": sd[k].grad for k in SAMPLED}}
    for k, g in grads.items():
        got = g.double().cpu().numpy().reshape(-1)[zf[k + "_f64/idx"]]
        errs[k] = nrm(got, zf[k + "_f64/val"])
    with capsys.disabled():
        print("\n%s %s" % (case, " ".join("%s %.1e" % kv for kv in errs.items())))
    assert errs["z"] <= 1e-5 and errs["Minv"] <= 1e-5 and errs["beta"] <= 1e-4 and errs["loss"] <= 1e-5
    assert errs["dL/dz"] <= 1e-4
    for k in grads:
        assert errs[k] <= 1e-4, k


# ---------------------------------------------------------------------------------------------------------------------
# it learns
# ---------------------------------------------------------------------------------------------------------------------
LEARN_B, LEARN_L, LEARN_MASK = 8, 2, 52
BEV_LANES = ((240.0, 0.02, 1.0e-4), (272.0, 0.015, -0.8e-4))      # x' = c + a t + b t^2, t = 255 - y'


def _learn_targets(theta_true, R=256):
    """Ridge maps [B, L, R, 2R] whose lanes are order-2 polynomials in the bird's-eye view of each image's theta_true,
    and the loss targets: each lane's image column at the 56 sample rows, valid where unmasked and inside the image."""
    B, W = theta_true.shape[0], 2 * R
    maps = torch.zeros(B, LEARN_L, R, W, dtype=torch.float64)
    x_gt = torch.zeros(B, LEARN_L, 56, dtype=torch.float64)
    valid = torch.zeros(B, LEARN_L, 56, dtype=torch.float64)
    u = torch.arange(W, dtype=torch.float64)
    ys = (160 + 10 * np.arange(56) - 80) / 2.5
    for b in range(B):
        _, Mi, rowp, yk = hg.warp_host(theta_true[b], R)
        for l, (c, a, q) in enumerate(BEV_LANES):
            t = 255.0 - rowp[:, 2]
            col = (c + a * t + q * t * t - rowp[:, 1]) / rowp[:, 0]           # image column of the lane on each row
            maps[b, l] = torch.exp(-0.5 * ((u[None] - torch.from_numpy(col)[:, None]) / 2.5) ** 2)
            tk = 255.0 - yk
            xp = c + a * tk + q * tk * tk
            xc = (Mi[0, 0] * xp + Mi[0, 1] * yk + Mi[0, 2]) / (Mi[2, 0] * xp + Mi[2, 1] * yk + Mi[2, 2])
            x_gt[b, l] = torch.from_numpy(xc)
            valid[b, l] = torch.from_numpy(((ys >= LEARN_MASK) & (xc >= 0) & (xc < W)).astype(np.float64))
    maps[:, :, :LEARN_MASK] = 0.0
    return maps.float().to(DEV), x_gt.to(DEV), valid.to(DEV)


def _train_warp(corners, maps, x_gt, valid, steps=200, lr=0.01):
    """``steps`` fused-Adam steps on a leaf z through the per-image warp, lsq_warp and the bound loss; (losses, z)."""
    import types
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss, fused_backprojection_loss
    from lanedetection_end2end_b200.optim import FusedOptimizer
    nz = hg.CORNERS[corners][0]
    B, L, R, W = maps.shape
    z = torch.zeros(B, nz, device=DEV, requires_grad=True)
    opt = FusedOptimizer([z], "adam", lr=lr)
    holder = types.SimpleNamespace(current=None)
    extra = ("--predict_homography", "True", "--predict_homography_corners", corners)
    crit = backprojection_loss(_args("--order", "2", "--nclasses", str(L), *extra, L=L, B=B)).bind(
        types.SimpleNamespace(DLT=holder))
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    losses = []
    for _ in range(steps + 1):
        rowp, Minv, yk, M, xtab, yrow, prm = hg._PREDICTED_FUNCTIONS[corners].apply(z, R, LEARN_MASK, 255.0, st)
        holder.current = hg.WarpTables(rowp, Minv, yk, M, xtab, yrow, R, W, delta=prm)
        beta, _ = ops_lsq.lsq_warp(maps, holder.current, 2, LEARN_MASK, "square", 0.0, False, False, st)
        loss, _ = fused_backprojection_loss(crit, [beta[:, l].unsqueeze(-1) for l in range(L)], x_gt, valid)
        losses.append(loss.detach())
        if len(losses) > steps:
            break
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert int(st.item()) == 0
    return torch.stack(losses).cpu().numpy(), z.detach()


def test_the_source_corners_learn_and_the_destination_ones_do_not(capsys):
    """z [8, 5] learns each image's warp from lanes that are order-2 polynomials in the bird's-eye view of known
    offsets: the loss falls at least 2x and theta moves toward the offsets; the destination parametrisation, on the same
    maps and steps, changes the loss at least 100x less (relatively)."""
    g = np.random.default_rng(11)
    theta_true = (g.uniform(-0.5, 0.5, (LEARN_B, 5)) / 64).astype(np.float32)
    maps, x_gt, valid = _learn_targets(theta_true)
    src, z = _train_warp("source", maps, x_gt, valid)
    theta = (torch.tanh(z.double()) / 64).cpu().numpy()
    err0, err1 = np.linalg.norm(theta_true), np.linalg.norm(theta - theta_true)
    dst, _ = _train_warp("destination", maps, x_gt, valid)
    rel_src, rel_dst = abs(src[-1] - src[0]) / src[0], abs(dst[-1] - dst[0]) / dst[0]
    with capsys.disabled():
        print("\nsource: loss %.6g -> %.6g (x%.1f), |theta - true| %.3g -> %.3g; destination: loss %.9g -> %.9g "
              "(relative change %.2e, source %.2e)" % (src[0], src[-1], src[0] / src[-1], err0, err1, dst[0], dst[-1],
                                                       rel_dst, rel_src))
    assert src[-1] * 2 <= src[0]
    # two order-2 lanes do not pin all five offsets (the loss has flat directions at the truth, where it reaches zero):
    # theta moves toward the offsets without reaching them -- a float64 restatement of the same run (torch Adam through
    # an 8x8 solve of each image's warp) ends at 0.82 of the starting distance too
    assert err1 < 0.9 * err0
    assert rel_dst * 100 <= rel_src


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def test_train_epoch_equals_eager_loop(paths):
    """engine.train_epoch with the source corners (train.sh shape, --clas) against the eager loop on the same fused
    functions: parameters including the branch, optimizer state and losses.avg bit for bit; fully_connected2 moves."""
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    args = te.make_args("clas4", paths[0])
    args.predict_homography = True
    args.predict_homography_corners = "source"
    train, _, _ = te.loaders(paths, args)
    batches = list(train)
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    assert ma.DLT.corners == "source"
    mb.load_state_dict(ma.state_dict())
    fc2_before = mb.DLT.spatial_trans.fully_connected2.weight.detach().clone()
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    crits[0].bind(ma)
    want_loss, _, _, skipped = te.eager_train(batches, ma, oa, *crits, args, te.per_lane_loss)
    got_loss, _ = engine.train_epoch(batches, mb, ob, *crits, args, 0)
    assert not skipped and got_loss == want_loss
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    assert not torch.equal(mb.DLT.spatial_trans.fully_connected2.weight, fc2_before)
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)


def test_validate_equals_eager(paths):
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import inference
    args = te.make_args("clas4", paths[0])
    args.predict_homography = True
    args.predict_homography_corners = "source"
    _, valid, _ = te.loaders(paths, args)
    batches = list(valid)
    model = te.make_model(args).eval()
    crits = te.criteria(args)
    crits[0].bind(model)
    want, _ = te.eager_validate(batches, model, *crits, args)
    got = inference.validate(te.Listed(batches), model, *crits, args)
    assert got == want and got[0] != 0


def test_test_model_writes_each_images_host_projection(tmp_path):
    """inference.test_model with the source corners writes what the reference's test loop writes when every image is
    back-projected with its own M^-1 computed on the host (warp_host of the image's theta)."""
    import io
    import json
    from test_tusimple_gpu import _ground_truth
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from oracle import inputs
    N, B = 40, 32
    args = _args("--order", "3", "--clas", "1", *SRC, B=B)
    torch.manual_seed(0)
    model = Net(args).cuda()
    with torch.no_grad():      # a branch away from the fixed warp, different for every image
        model.DLT.spatial_trans.fully_connected2.weight.normal_(0.0, 0.05)
        model.DLT.spatial_trans.fully_connected2.bias.copy_(torch.tensor([0.3, -0.2, 0.4, -0.3, 0.2]))
    model.eval()
    images = torch.from_numpy(inputs.make_images(N, 256, 512, seed=31))
    batches = [images[i:i + B] for i in range(0, N, B)]
    lanes, minvs = [], []
    y_d = (np.arange(160, 720, 10) - 80) / 2.5
    with torch.no_grad():
        for xb in batches:
            out = model(xb.cuda(), torch.zeros(xb.shape[0], 4), True)
            horizon_pred = torch.sigmoid(out[7]).sum(dim=1)
            horizon_pred = (torch.round((inference.resize_coordinates(horizon_pred) + 80) / 10) * 10).int()
            line_pred = torch.round(torch.sigmoid(out[6]))
            beta = torch.stack([t.reshape(xb.shape[0], -1) for t in out[:4]], 1).cpu().numpy()
            theta = model.DLT.current.delta.cpu().numpy()
            assert theta.dtype == np.float32 and theta.shape == (xb.shape[0], 5)
            xcal = np.empty((xb.shape[0], 4, 56))
            for b in range(xb.shape[0]):
                M, Mi, _, _ = hg.warp_host(theta[b], 256)
                minvs.append(Mi)
                yp = (M[1, 1] * y_d + M[1, 2]) / (M[2, 1] * y_d + M[2, 2])
                for l in range(4):
                    xp = np.polyval(beta[b, l], 255.0 - yp)
                    xcal[b, l] = (Mi[0, 0] * xp + Mi[0, 1] * yp + Mi[0, 2]) / (Mi[2, 0] * xp + Mi[2, 1] * yp + Mi[2, 2])
            lanes += inference.lanes_from_predictions(torch.from_numpy(xcal * 2.5), line_pred.cpu(), horizon_pred.cpu())
    assert np.unique(np.round(np.stack(minvs).reshape(N, -1), 9), axis=0).shape[0] == N
    rows = _ground_truth(lanes, 5)
    with open(tmp_path / "test_label.json", "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    want = io.StringIO()
    inference.write_tusimple_predictions(want, rows, lanes, 0)
    args.test_dir = args.save_path = str(tmp_path)
    inference.test_model(batches, model, None, None, None, None, args)
    assert (tmp_path / "test_set_predictions.json").read_text() == want.getvalue()


@pytest.mark.parametrize("mode", ["tf32x3", "fp32", "bf16", "fp8"])
def test_model_with_trapezium_mask_in_every_mode(mode):
    """The source corners with --trapezium_mask through Net.forward in each convolution mode (eval; and one training
    step outside fp8): masked is act(output) * keep, beta is the masked per-image fit of the returned output on the
    model's own warp, and in training the branch receives a finite gradient."""
    from lanedetection_end2end_b200 import Loss_crit, ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    B = 4
    torch.manual_seed(0)
    args = _args("--order", "3", "--clas", "True", "--mask_percentage", "0.2", "--trapezium_mask", "True", *SRC, B=B)
    model = Net(args).cuda()
    with torch.no_grad():
        model.DLT.spatial_trans.fully_connected2.weight.normal_(0.0, 0.05)
    x = torch.rand(B, 3, 256, 512, device=DEV)
    old = ops_net.CONV_MODE
    try:
        ops_net.set_conv_mode(mode)
        model.eval()
        with torch.no_grad():
            out = model(x, torch.zeros(B, 4), True)
            warp = model.DLT.current
            masked, output = out[4], out[5]
            assert torch.equal(masked, (output.float() ** 2) * model.keep.bool())
            beta, _ = ops_lsq.lsq_warp(output, warp, 3, model.zero_rows, "square", keep=model.keep)
        assert torch.equal(torch.stack([b.squeeze(-1) for b in out[:4]], 1), beta)
        assert tuple(warp.delta.shape) == (B, 5)
        assert np.unique(warp.Minv.cpu().numpy(), axis=0).shape[0] == B
        if mode != "fp8":
            model.train()
            crit = Loss_crit.backprojection_loss(args).bind(model)
            out = model(x, torch.zeros(B, 4), True)
            beta_in, x_gt, valid = _loss_inputs(B, 4, 4, 1)
            loss, _ = Loss_crit.fused_backprojection_loss(crit, out[:4], x_gt, valid)
            loss.backward()
            gw = model.DLT.spatial_trans.fully_connected1.weight.grad
            assert torch.isfinite(loss) and gw is not None and bool(torch.isfinite(gw).all())
    finally:
        ops_net.set_conv_mode(old)
