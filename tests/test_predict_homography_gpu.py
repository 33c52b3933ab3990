"""--predict_homography on the GPU: the per-image entry points against the shared-table ones bit for bit, the tables and
their backward against the host hooks, the per-image loss, the model's start from the fixed warp, graphed training
against the eager loop, validation and test_model."""
import numpy as np
import pytest
import torch

from test_epoch_gpu import paths  # noqa: F401  (the synthetic TuSimple directory fixture)

from lanedetection_end2end_b200 import _capi, homography as hg, ops_lsq
from lanedetection_end2end_b200.Networks.utils import define_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
p = _capi.ptr


def _args(*extra, L=4, B=2):
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(L), "--batch_size", str(B),
                                     "--loss_policy", "backproject"] + list(extra))


def _tables(z, R=256, mask_rows=77):
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = hg._PredictedWarpFunction.apply(z, R, mask_rows, 255.0, st)
    return out, st


def _z(B, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 3, generator=g) * scale).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [256, 320])
def test_tables_match_the_host_hooks(R):
    B, mask_rows = 5, int(np.ceil(0.3 * R))
    z = _z(B, 1)
    (rowp, Minv, yk, M, xtab, yrow, delta), st = _tables(z, R, mask_rows)
    assert int(st.item()) == 0
    dt = torch.tanh(z.double()) / 16
    assert (delta - dt).abs().max().item() <= 1e-16
    for b in range(B):
        Mh, Mih, rowph, ykh = hg.predicted_warp_host(delta[b].cpu().numpy(), R)
        # rowp on the unmasked rows only: above the vanishing line the rows' values grow without bound
        for got, ref in ((M[b], Mh), (Minv[b], Mih), (rowp[b, mask_rows:], rowph[mask_rows:]), (yk[b], ykh)):
            got, ref = got.cpu().numpy().reshape(ref.shape), ref
            assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()
        x = (rowp[b, :, 0:1] * torch.arange(2 * R, device=DEV, dtype=torch.float64) + rowp[b, :, 1:2]).float()
        assert torch.equal(xtab[b].view(R, 2 * R), x)
        assert torch.equal(yrow[b], (255.0 - rowp[b, :, 2]).float())
    # one image at a time gives the batch's slices, bit for bit
    for b in range(B):
        one, _ = _tables(z[b:b + 1].contiguous(), R, mask_rows)
        for a, c in zip(one, (rowp, Minv, yk, M, xtab, yrow, delta)):
            assert torch.equal(a[0], c[b])


def test_backward_matches_the_host_hook():
    R, B, mask_rows = 256, 4, 77
    z = _z(B, 2).requires_grad_(True)
    (rowp, Minv, yk, *_), _ = _tables(z, R, mask_rows)
    g = torch.Generator().manual_seed(3)
    g_rowp = torch.randn(B, R, 3, generator=g, dtype=torch.float64).to(DEV)
    g_minv = torch.randn(B, 9, generator=g, dtype=torch.float64).to(DEV) * 1e-3
    g_yk = torch.randn(B, 56, generator=g, dtype=torch.float64).to(DEV) * 1e-2
    (rowp * g_rowp).sum().add((Minv * g_minv).sum()).add((yk * g_yk).sum()).backward()
    for b in range(B):
        zb = z[b].detach().cpu().numpy().astype(np.float32)
        ref = np.zeros(3)
        gr, gm, gy = (t[b].cpu().numpy().copy() for t in (g_rowp, g_minv, g_yk))
        rc = _capi.lib().lf_predicted_homography_bwd_host(zb.ctypes.data, R, mask_rows, gr.ctypes.data, gm.ctypes.data,
                                                          gy.ctypes.data, ref.ctypes.data)
        assert rc == 0
        got = z.grad[b].double().cpu().numpy()
        assert np.abs(got - ref.astype(np.float32)).max() <= 1e-6 * np.abs(ref).max()


def _fwd(o, xtab, yrow, keep, per_image, rowsums, order=3, mask_rows=77, act=_capi.ACT_IDS["square"]):
    B, L, H, W = o.shape
    beta = torch.empty(B, L, order + 1, dtype=torch.float64, device=DEV)
    zinv = torch.empty(B, L, order + 1, order + 1, dtype=torch.float64, device=DEV)
    masked = torch.empty(B, L, H, W, dtype=torch.float32, device=DEV)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    rs = torch.empty(B, L, H, 3, dtype=torch.float32, device=DEV) if rowsums else None
    nb = _capi.lib().lf_lsq_workspace_bytes(B, L, H, W, order)
    ws = torch.zeros(nb, dtype=torch.uint8, device=DEV)
    args = (o.contiguous(), _capi.dtype_id(o))
    if per_image:
        _capi.call("lf_lsq_fwd_per_image", p(args[0]), args[1], p(xtab), p(yrow), p(keep), B, L, H, W, order, mask_rows, act,
                   0.0, 0, p(beta), p(zinv), p(masked), p(st), p(rs), p(ws), nb, _capi.stream_ptr())
    elif rowsums:
        name = "lf_lsq_fwd_rowsums" + ("_keep" if keep is not None else "")
        kp = () if keep is None else (p(keep),)
        _capi.call(name, p(args[0]), args[1], p(xtab), p(yrow), *kp, B, L, H, W, order, mask_rows, act, 0.0, 0,
                   p(beta), p(zinv), p(masked), p(st), p(rs), p(ws), nb, _capi.stream_ptr())
    else:
        name = "lf_lsq_fwd" + ("_keep" if keep is not None else "")
        kp = () if keep is None else (p(keep),)
        _capi.call(name, p(args[0]), args[1], p(xtab), None, p(yrow), *kp, B, L, H, W, order, mask_rows, act, 0.0, 0,
                   p(beta), p(zinv), p(masked), p(st), p(ws), nb, _capi.stream_ptr())
    assert int(st.item()) == 0
    return beta, zinv, masked, rs


def _bwd(o, xtab, yrow, keep, per_image, beta, zinv, gbeta, order=3, mask_rows=77, act=_capi.ACT_IDS["square"]):
    B, L, H, W = o.shape
    d_o = torch.empty_like(o)
    if per_image:
        _capi.call("lf_lsq_bwd_per_image", p(o), _capi.dtype_id(o), p(xtab), p(yrow), p(keep), B, L, H, W, order, mask_rows,
                   act, p(beta), p(zinv), p(gbeta), p(d_o), _capi.stream_ptr())
    else:
        name = "lf_lsq_bwd" + ("_keep" if keep is not None else "")
        kp = () if keep is None else (p(keep),)
        _capi.call(name, p(o), _capi.dtype_id(o), p(xtab), None, p(yrow), *kp, B, L, H, W, order, mask_rows, act, p(beta),
                   p(zinv), p(gbeta), p(d_o), _capi.stream_ptr())
    return d_o


def _grid_grad(rs, yrow, beta, zinv, gbeta, per_image, order=3, mask_rows=77):
    B, L, H, _ = rs.shape
    if per_image:
        g = torch.empty(B, H, 3, dtype=torch.float64, device=DEV)
        _capi.call("lf_lsq_grid_grad_per_image", p(rs), p(yrow), p(beta), p(zinv), p(gbeta), B, L, H, order, mask_rows,
                   p(g), _capi.stream_ptr())
    else:
        g = torch.empty(H, 3, dtype=torch.float64, device=DEV)
        _capi.call("lf_lsq_grid_grad", p(rs), p(yrow), p(beta), p(zinv), p(gbeta), B, L, H, order, mask_rows, p(g),
                   _capi.stream_ptr())
    return g


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("keep", [False, True], ids=["plain", "keep"])
@pytest.mark.parametrize("act", ["square", "relu"])
@pytest.mark.parametrize("L", [2, 4])
def test_per_image_entry_points_are_the_shared_bits(dtype, keep, act, L):
    from lanedetection_end2end_b200.Networks.LSQ_layer import trapezium_keep
    R, H, W, B, mask_rows = 256, 256, 512, 3, 77
    a = _capi.ACT_IDS[act]
    torch.manual_seed(L)
    o = (torch.randn(B, L, H, W, device=DEV) * 0.5 + 0.7).to(dtype)
    km = trapezium_keep(R, mask_rows).to(DEV) if keep else None
    z = _z(B, 5, 0.5)
    (rowp, Minv, yk, M, xtab, yrow, delta), _ = _tables(z, R, mask_rows)
    gbeta = torch.randn(B, L, 4, dtype=torch.float64, device=DEV)
    kw = dict(act=a, mask_rows=mask_rows)

    def same(x, y):
        # the run-time activation kernels (act != square) may contract the per-pixel products differently in the
        # per-image instantiation, as the keep kernels do against the plain ones: fp32 rounding, bounded at 1e-6
        if act == "square":
            return torch.equal(x, y)
        return (x.double() - y.double()).abs().max().item() <= 1e-6 * y.double().abs().max().item()
    # distinct tables: image b is a single-image shared-table call on b's tables.  Row sums, masked maps, d_o and the
    # grid gradient are per row and equal bit for bit (given the same beta, Z^-1); beta and Z^-1 sum the rows' fp64
    # moments over chunks whose count lf_lsq_plan picks from B (it fills the SMs' waves), so a B-image and a one-image
    # call group the same terms differently; the order-3 normal matrix's conditioning (y up to 255) amplifies that
    # reassociation, so the bound is 1e-6 norm-wise per image and lane (measured up to 8e-9 on the constant term)
    for rowsums in (False, True):
        got = _fwd(o, xtab, yrow, km, True, rowsums, **kw)
        d_got = _bwd(o, xtab, yrow, km, True, got[0], got[1], gbeta, **kw)
        g_got = _grid_grad(got[3], yrow, got[0], got[1], gbeta, True, mask_rows=mask_rows) if rowsums else None
        for b in range(B):
            ob = o[b:b + 1].contiguous()
            want = _fwd(ob, xtab[b], yrow[b], km, False, rowsums, **kw)
            for x, y in zip(got[:2], want[:2]):
                x, y = x[b:b + 1].reshape(L, -1), y.reshape(L, -1)
                assert ((x - y).norm(dim=1) / y.norm(dim=1)).max().item() <= 1e-6
            assert same(got[2][b:b + 1], want[2])
            if rowsums:
                assert same(got[3][b:b + 1, :, mask_rows:], want[3][:, :, mask_rows:])
            bb, zb, gb = (t[b:b + 1].contiguous() for t in (got[0], got[1], gbeta))
            d_want = _bwd(ob, xtab[b], yrow[b], km, False, bb, zb, gb, **kw)
            assert same(d_got[b:b + 1], d_want)
            if rowsums:
                g_want = _grid_grad(got[3][b:b + 1].contiguous(), yrow[b], bb, zb, gb, False, mask_rows=mask_rows)
                assert torch.equal(g_got[b], g_want)       # the same row sums in: the same per-row code
    # every image given the same tables: the shared-table entry points' bits
    xs, ys = xtab[:1].expand(B, -1).contiguous(), yrow[:1].expand(B, -1).contiguous()
    for rowsums in (False, True):
        got = _fwd(o, xs, ys, km, True, rowsums, **kw)
        want = _fwd(o, xtab[0], yrow[0], km, False, rowsums, **kw)
        for x, y in zip(got[:3], want[:3]):
            assert same(x, y)
        if rowsums:      # rows above mask_rows are not written
            assert same(got[3][:, :, mask_rows:], want[3][:, :, mask_rows:])
        assert same(_bwd(o, xs, ys, km, True, got[0], got[1], gbeta, **kw),
                    _bwd(o, xtab[0], yrow[0], km, False, want[0], want[1], gbeta, **kw))
        if rowsums:
            # the shared kernel sums the B images inside one fp64 accumulator per row; the per-image kernel keeps them
            # apart, so their sum over images is a reassociation of the same terms
            gs = _grid_grad(got[3], ys, got[0], got[1], gbeta, True, mask_rows=mask_rows).sum(0)
            gw = _grid_grad(want[3], yrow[0], want[0], want[1], gbeta, False, mask_rows=mask_rows)
            tol = 1e-12 if act == "square" else 1e-6      # the row sums themselves agree to 1e-6 otherwise (above)
            assert (gs - gw).abs().max().item() <= tol * gw.abs().max().item()


def _loss_per_image(Minv, yk, beta, x_gt, valid):
    B, L, n = beta.shape
    f64 = dict(dtype=torch.float64, device=DEV)
    lane, loss, dbeta, xcal = torch.empty(L, **f64), torch.empty(1, **f64), torch.empty_like(beta), torch.empty(B, L, 56, **f64)
    scratch = torch.empty(int(_capi.lib().lf_backproj_loss_per_image_scratch(B, L)), **f64)
    g = torch.empty(B, 65, **f64)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    _capi.call("lf_backproj_loss_per_image", p(yk.contiguous()), p(Minv.contiguous()), p(beta), p(x_gt), p(valid), B, L, n,
               p(lane), p(loss), p(dbeta), p(xcal), p(scratch), p(g), p(ticket), _capi.stream_ptr())
    return loss, dbeta, xcal, g


def _loss_inputs(B, L, n, seed):
    g = torch.Generator().manual_seed(seed)
    beta = (torch.randn(B, L, n, generator=g, dtype=torch.float64) * torch.tensor([1e-5, 1e-3, 1e-1, 1.0])[-n:]
            + torch.tensor([0.0] * (n - 1) + [256.0])).to(DEV)
    x_gt = (torch.rand(B, L, 56, generator=g, dtype=torch.float64) * 1280).to(DEV)
    valid = (torch.rand(B, L, 56, generator=g) > 0.3).double().to(DEV)
    return beta, x_gt, valid


def test_loss_per_image():
    from lanedetection_end2end_b200 import Loss_crit
    B, L, n = 4, 4, 4
    beta, x_gt, valid = _loss_inputs(B, L, n, 0)
    z = _z(B, 7, 0.5)
    (rowp, Minv, yk, *_), _ = _tables(z)
    # every image given the same warp: lf_backproj_loss_dev's loss, dbeta and xcal bits
    Ms, ys = Minv[:1].expand(B, -1).contiguous(), yk[:1].expand(B, -1).contiguous()
    loss, dbeta, xcal, g = _loss_per_image(Ms, ys, beta, x_gt, valid)
    f64 = dict(dtype=torch.float64, device=DEV)
    lane, loss_s, dbeta_s, xcal_s = torch.empty(L, **f64), torch.empty(1, **f64), torch.empty_like(beta), torch.empty(B, L, 56, **f64)
    gp, gc = torch.empty(L, 65, **f64), torch.empty(65, **f64)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    _capi.call("lf_backproj_loss_dev", p(yk[0].contiguous()), p(Minv[0].contiguous()), p(beta), p(x_gt), p(valid), B, L, n,
               p(lane), p(loss_s), p(dbeta_s), p(xcal_s), p(gp), p(gc), p(ticket), _capi.stream_ptr())
    assert torch.equal(loss, loss_s) and torch.equal(dbeta, dbeta_s) and torch.equal(xcal, xcal_s)
    # the shared kernel sums the images per sample before the lane sum; per image the same terms are summed after it
    assert (g.sum(0) - gc).abs().max().item() <= 1e-12 * gc.abs().max().item()
    # distinct warps: the torch restatement with per-image constants (backprojection_loss.forward_lanes) and autograd
    loss, dbeta, xcal, g = _loss_per_image(Minv, yk, beta, x_gt, valid)
    Mi_t, yk_t, beta_t = Minv.clone().requires_grad_(True), yk.clone().requires_grad_(True), beta.clone().requires_grad_(True)

    class W:
        per_image = True
        Minv, yk = Mi_t, yk_t
    crit = Loss_crit.backprojection_loss(_args("--order", "3"))
    crit.learn_homography = True
    crit.__dict__["_warp"] = type("H", (), {"current": W})()
    ref, xref = crit.forward_lanes([beta_t[:, l, :, None] for l in range(L)], x_gt, valid)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-12 * abs(ref.item())
    assert (xcal - xref).abs().max().item() <= 1e-9
    for got, want in ((dbeta, beta_t.grad), (g[:, :9], Mi_t.grad), (g[:, 9:], yk_t.grad)):
        assert (got - want).abs().max().item() <= 1e-10 * want.abs().max().item()


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def test_starts_from_the_fixed_warp_and_trains_the_branch():
    from lanedetection_end2end_b200 import Loss_crit
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    B = 4
    torch.manual_seed(0)
    fixed = Net(_args("--order", "3", "--clas", "True", B=B)).cuda()
    define_init_weights(fixed, "kaiming")
    pred = Net(_args("--order", "3", "--clas", "True", "--predict_homography", "True", B=B)).cuda()
    define_init_weights(pred, "kaiming")
    res = pred.load_state_dict(fixed.state_dict(), strict=False)
    assert all(k.startswith("DLT.") for k in res.missing_keys) and not res.unexpected_keys
    x = torch.rand(B, 3, 256, 512, device=DEV)
    fixed.eval(), pred.eval()
    with torch.no_grad():
        a = torch.stack([t.squeeze(-1) for t in fixed(x, torch.zeros(B, 4), True)[:4]], 1)
        b = torch.stack([t.squeeze(-1) for t in pred(x, torch.zeros(B, 4), True)[:4]], 1)
    # the fixed warp's tables come from the reference's fp32 grid, the predicted ones from the closed form: 1-ulp table
    # differences, gated norm-wise per image and lane
    assert ((a - b).norm(dim=-1) / a.norm(dim=-1)).max().item() <= 1e-5
    # train mode: the loss reaches fully_connected2 (and through it the rest of the branch); conv5 gets nothing
    pred.train()
    crit = Loss_crit.backprojection_loss(_args("--order", "3", "--predict_homography", "True", B=B)).bind(pred)
    out = pred(x, torch.zeros(B, 4), True)
    beta_in, x_gt, valid = _loss_inputs(B, 4, 4, 1)
    loss, _ = Loss_crit.fused_backprojection_loss(crit, out[:4], x_gt, valid)
    loss.backward()
    st = pred.DLT.spatial_trans
    assert st.fully_connected2.weight.grad.abs().sum() > 0 and st.conv5.weight.grad is None


def test_train_epoch_equals_eager_loop(paths):
    """engine.train_epoch with --predict_homography (train.sh shape, --clas) against the eager loop on the same fused
    functions: parameters including the branch, optimizer state and losses.avg bit for bit."""
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    args = te.make_args("clas4", paths[0])
    args.predict_homography = True
    train, _, _ = te.loaders(paths, args)
    batches = list(train)
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    assert hasattr(ma, "DLT")
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    crits[0].bind(ma)
    want_loss, _, _, skipped = te.eager_train(batches, ma, oa, *crits, args, te.per_lane_loss)
    got_loss, _ = engine.train_epoch(batches, mb, ob, *crits, args, 0)
    assert not skipped and got_loss == want_loss
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    assert ma.DLT.spatial_trans.fully_connected2.weight.abs().sum() > 0
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)


def test_validate_equals_eager(paths):
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import inference
    args = te.make_args("clas4", paths[0])
    args.predict_homography = True
    _, valid, _ = te.loaders(paths, args)
    batches = list(valid)
    model = te.make_model(args).eval()
    crits = te.criteria(args)
    crits[0].bind(model)
    want, _ = te.eager_validate(batches, model, *crits, args)
    got = inference.validate(te.Listed(batches), model, *crits, args)
    assert got == want and got[0] != 0


def test_test_model_writes_each_images_host_projection(tmp_path):
    """inference.test_model with --predict_homography writes what the reference's test loop writes when every image is
    back-projected with its own M^-1 computed on the host (predicted_warp_host of the image's delta)."""
    import io
    import json
    from test_tusimple_gpu import _ground_truth
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from oracle import inputs
    N, B = 40, 32
    args = _args("--order", "3", "--clas", "1", "--predict_homography", "True", B=B)
    torch.manual_seed(0)
    model = Net(args).cuda()
    with torch.no_grad():      # a branch away from the fixed warp, different for every image
        model.DLT.spatial_trans.fully_connected2.weight.normal_(0.0, 0.05)
        model.DLT.spatial_trans.fully_connected2.bias.copy_(torch.tensor([0.3, -0.2, 0.4]))
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
            delta = model.DLT.current.delta.cpu().numpy()
            xcal = np.empty((xb.shape[0], 4, 56))
            for b in range(xb.shape[0]):
                M, Mi, _, _ = hg.predicted_warp_host(delta[b], 256)
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
    """The flag with --trapezium_mask through Net.forward in each convolution mode (eval; and one training step outside
    fp8): masked is act(output) * keep, beta is the masked per-image fit of the returned output on the model's own warp,
    and in training the branch receives a finite gradient."""
    from lanedetection_end2end_b200 import Loss_crit, ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    B = 4
    torch.manual_seed(0)
    args = _args("--order", "3", "--clas", "True", "--mask_percentage", "0.2", "--trapezium_mask", "True",
                 "--predict_homography", "True", B=B)
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


GOLDEN_CASES = ["predict_homography_l2_d2", "predict_homography_l2_d2_trapezium", "predict_homography_l4_d3",
                "predict_homography_l4_d3_trapezium"]


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_golden_reference_modules(case, capsys):
    """The branch, the per-image warps, the fit and the loss against the reference modules' float64 golden
    (oracle/make_predict_homography_golden.py), in the default tf32x3 mode: z and each image's M^-1 within 1e-5, beta
    within 1e-4 and the loss within 1e-5 (norm-wise); dL/dz per entry within 1e-4 of the sum of its absolute chain-rule
    terms (the loss does not depend on z in exact arithmetic, so the total is rounding on both sides); and the branch's
    backward on a fixed cotangent -- sampled gradients of the encoder map and of the branch's weights -- within 1e-4."""
    import json
    import os
    import types
    from math import ceil
    from conftest import GOLDEN
    from oracle import inputs
    from oracle.make_predict_homography_golden import SAMPLED, branch_weights, cotangent, encoder_map
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
    mod = hg.PredictedHomography(H, mask).cuda().train()
    mod.spatial_trans.load_state_dict({k: torch.from_numpy(v) for k, v in branch_weights(seed + 3).items()}, strict=False)
    E = torch.from_numpy(E_np).cuda().requires_grad_(True)
    st = torch.zeros(1, dtype=torch.int32, device=DEV)
    z = mod.spatial_trans(E)
    z.retain_grad()
    rowp, Minv, yk, M, xtab, yrow, delta = hg._PredictedWarpFunction.apply(z, H, mask, 255.0, st)
    warp = hg.WarpTables(rowp, Minv, yk, M, xtab, yrow, H, W, delta=delta)
    mod.current = warp
    crit = backprojection_loss(_args("--order", str(order), "--nclasses", str(L), "--predict_homography", "True", L=L))
    crit.bind(types.SimpleNamespace(DLT=mod))
    o = torch.from_numpy(o_np).cuda()
    beta, _ = ops_lsq.lsq_warp(o, warp, order, mask, "square", 0.0, False, False, st, keep)
    loss, _ = fused_backprojection_loss(crit, [beta[:, l].unsqueeze(-1) for l in range(L)],
                                        torch.from_numpy(zf["x_gt"]).cuda(), torch.from_numpy(zf["valid"]).cuda())
    loss.backward()
    assert int(st.item()) == 0
    nrm = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))
    errs = {"z": nrm(z.detach().double().cpu().numpy(), zf["z_f64"]),
            "Minv": max(nrm(Minv[b].detach().cpu().numpy(), zf["Minv_f64"][b].reshape(-1)) for b in range(B)),
            "beta": nrm(beta.detach().cpu().numpy(), zf["beta_f64"]),
            "loss": abs(loss.item() - float(zf["loss_f64"])) / abs(float(zf["loss_f64"])),
            "dL/dz": float((np.abs(z.grad.double().cpu().numpy() - zf["gz_f64"]) / zf["gz_abs"]).max())}
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
