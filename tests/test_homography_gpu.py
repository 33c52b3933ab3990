"""Learned bird's-eye-view homography (--learn_homography) on the H100: the least-squares layer on the warp's device
tables against float64 autograd, theta = 0 against the fixed warp, a graphed training step that moves theta, and the
vanishing-line guard."""
import json
import os
import types
import zlib

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_epoch_gpu import paths  # noqa: F401  (the synthetic TuSimple directory fixture)
from oracle import inputs
from oracle.make_homography_golden import CASES as GOLDEN_CASES, warp_fp64

from lanedetection_end2end_b200 import _capi, homography as hg, ops_lsq
from lanedetection_end2end_b200.Networks.utils import define_args

pytestmark = pytest.mark.gpu


def _warp_fp64(theta, R):
    """rowp (alpha, gamma, y') [R, 3] of theta through a differentiable float64 8x8 solve."""
    from test_homography_cpu import _torch_warp
    M, _ = _torch_warp(theta, R)
    v = torch.arange(R, dtype=torch.float64, device=M.device)
    den = M[2, 1] * v + M[2, 2]
    return torch.stack([M[0, 0] / den, (M[0, 1] * v + M[0, 2]) / den, (M[1, 1] * v + M[1, 2]) / den], 1)


def _lsq_fp64(o, rowp, order, mask, act, reg, chol):
    R, W = o.shape[2], o.shape[3]
    u = torch.arange(W, dtype=torch.float64)
    a = {"square": o ** 2, "none": o, "relu": torch.relu(o)}[act]
    w = a ** 2
    w = torch.cat([torch.zeros_like(w[:, :, :mask]), w[:, :, mask:]], 2)
    x = rowp[:, 0:1] * u + rowp[:, 1:2]
    y = (255.0 - rowp[:, 2])[:, None].expand(R, W)
    phi = torch.stack([y ** (order - i) for i in range(order + 1)], -1)
    Z = torch.einsum("blhw,hwi,hwj->blij", w, phi, phi) + reg * torch.eye(order + 1, dtype=torch.float64)
    X = torch.einsum("blhw,hwi,hw->bli", w, phi, x)
    if chol:
        return torch.cholesky_solve(X.unsqueeze(-1), torch.linalg.cholesky(Z)).squeeze(-1)
    return torch.linalg.solve(Z, X)


@pytest.mark.parametrize("order,act,reg,chol", [(2, "square", 0.0, False), (3, "square", 0.0, True),
                                                (1, "relu", 0.1, False)])
def test_lsq_on_learned_warp_against_fp64(order, act, reg, chol):
    R, B, L, mask = 256, 4, 4, 52
    gen = torch.Generator().manual_seed(order)
    o = torch.randn(B, L, R, 2 * R, generator=gen) * 0.5 + torch.linspace(-1, 1, 2 * R)
    theta = torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01])
    gb = torch.randn(B, L, order + 1, generator=gen, dtype=torch.float64)

    mod = hg.LearnedHomography(R, mask).cuda()
    with torch.no_grad():
        mod.offsets.copy_(theta)
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    oc = o.cuda().requires_grad_(True)
    warp = mod(st)
    beta, _ = ops_lsq.lsq_warp(oc, warp, order, mask, act, reg, chol, False, st)
    (beta * gb.cuda()).sum().backward()
    assert int(st.item()) == 0

    th = theta.double().requires_grad_(True)
    o64 = o.double().requires_grad_(True)
    ref = _lsq_fp64(o64, _warp_fp64(th, R), order, mask, act, reg, chol)
    (ref * gb).sum().backward()
    rel = lambda a, b: float((a.double().cpu() - b).norm() / b.norm())
    assert rel(beta, ref.detach()) < 1e-5
    assert rel(oc.grad, o64.grad) < 1e-4
    err = rel(mod.offsets.grad, th.grad)
    print("theta.grad rel err %.2e" % err)
    assert err < 1e-4


def test_theta_zero_matches_fixed_warp():
    from lanedetection_end2end_b200.Networks.LSQ_layer import ProjectiveGridGenerator
    from lanedetection_end2end_b200.Networks.utils import get_homography
    R, B, L, mask, order = 256, 2, 4, 52, 2
    o = torch.randn(B, L, R, 2 * R, generator=torch.Generator().manual_seed(3)).cuda()
    M, _ = get_homography(R)
    grid = ProjectiveGridGenerator((B, L, R, 2 * R), torch.from_numpy(M).unsqueeze(0).float(), False)
    b_fixed, _ = ops_lsq.lsq(o, grid, order, 255.0, mask, "square")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    warp = hg.LearnedHomography(R, mask).cuda()(st)
    b_warp, _ = ops_lsq.lsq_warp(o, warp, order, mask, "square", status_out=st)
    assert int(st.item()) == 0
    assert float((b_warp - b_fixed).norm() / b_fixed.norm()) < 1e-5
    # d_o: the same upstream gradient through both
    gb = torch.randn(B, L, order + 1, generator=torch.Generator().manual_seed(4), dtype=torch.float64).cuda()
    of, ow = o.clone().requires_grad_(True), o.clone().requires_grad_(True)
    (ops_lsq.lsq(of, grid, order, 255.0, mask, "square")[0] * gb).sum().backward()
    st.zero_()
    warp = hg.LearnedHomography(R, mask).cuda()(st)
    (ops_lsq.lsq_warp(ow, warp, order, mask, "square", status_out=st)[0] * gb).sum().backward()
    assert float((ow.grad - of.grad).norm() / of.grad.norm()) < 1e-5


def _args(*extra):
    return define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--loss_policy", "backproject", "--batch_size",
                                     "2", "--resize", "256", "--nclasses", "4", "--order", "3", "--learn_homography", "True"]
                                    + list(extra))


def _step():
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    torch.manual_seed(0)
    args = _args()
    model = Net(args).cuda()
    crit = backprojection_loss(args).bind(model)
    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    x = torch.rand(2, 3, 256, 512, device="cuda")
    xgt = torch.rand(2, 4, 56, device="cuda", dtype=torch.float64) * 400 + 50
    valid = torch.ones(2, 4, 56, device="cuda", dtype=torch.float64)
    step = GraphedTrainStep(model, crit, 4, x, xgt, valid, optimizer=opt)
    return model, step


def test_graphed_step_moves_theta():
    model, step = _step()
    before = model.homography.offsets.detach().clone()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    assert int(step.status.item()) == 0
    assert torch.isfinite(model.homography.offsets.grad).all()
    assert not torch.equal(model.homography.offsets.detach(), before)


def test_vanishing_line_guard_skips_update():
    # theta drifts in training: theta_4 = 0.25 lowers the top corners by 64 rows, and the vanishing line moves from row
    # 27.2 to row 98.8, below the 52 masked rows.  The replay flags the batch and updates nothing.
    model, step = _step()
    with torch.no_grad():
        model.homography.offsets[4] = 0.25
    params = [p.detach().clone() for p in model.parameters()]
    step()
    torch.cuda.synchronize()
    assert int(step.status.item()) & _capi.STATUS_NONFINITE
    for p, q in zip(model.parameters(), params):
        assert torch.equal(p.detach(), q)


def _bound_crit(args, mod):
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    return backprojection_loss(args).bind(types.SimpleNamespace(homography=mod))


@pytest.mark.parametrize("case", [c[0] for c in GOLDEN_CASES])
def test_golden_reference_modules(case, capsys):
    """The learned warp's LSQ layer and loss on the reference modules' float64 golden (oracle/make_homography_golden.py):
    beta within 1e-5, d_o within 1e-4, and theta.grad per entry within 1e-4 of the sum of the absolute chain-rule terms
    -- the totals cancel by about six orders of magnitude on these well-fitted lane maps, so a norm-wise gate on the
    total would measure the cancellation, not the kernels."""
    z = np.load(os.path.join(GOLDEN, case + ".npz"))
    meta = json.loads(str(z["meta"]))
    B, L, H, W, order = meta["B"], meta["L"], meta["H"], meta["W"], meta["order"]
    o_np = inputs.make_lane_maps(B, L, H, W, seed=meta["seed"]).astype(np.float32)
    if meta["act"] == "relu":
        o_np = ((o_np - 0.3) * 4.0).astype(np.float32)
    assert inputs.sha256_of(o_np, z["x_gt"], z["valid"]) == str(z["input_sha"])
    from math import ceil
    mask = ceil(H * meta["mask_pct"])
    args = _args("--order", str(order), "--nclasses", str(L))
    mod = hg.LearnedHomography(H, mask).cuda()
    with torch.no_grad():
        mod.offsets.copy_(torch.from_numpy(z["theta"]))
    crit = _bound_crit(args, mod)
    from lanedetection_end2end_b200.Loss_crit import fused_backprojection_loss
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    o = torch.from_numpy(o_np).cuda().requires_grad_(True)
    warp = mod(st)
    beta, _ = ops_lsq.lsq_warp(o, warp, order, mask, meta["act"], meta["reg_ls"], meta["cholesky"], False, st)
    betas = [beta[:, l].unsqueeze(-1) for l in range(L)]
    loss, _ = fused_backprojection_loss(crit, betas, torch.from_numpy(z["x_gt"]).cuda(), torch.from_numpy(z["valid"]).cuda())
    loss.backward()
    assert int(st.item()) == 0
    ref_beta = torch.from_numpy(z["beta_f64"])
    assert float((beta.cpu() - ref_beta).norm() / ref_beta.norm()) < 1e-5
    assert abs(loss.item() - float(z["loss_f64"])) <= 1e-5 * abs(float(z["loss_f64"]))
    d_o = o.grad.double().cpu().numpy().reshape(-1)[z["grad_f64/idx"]]
    ref_do = z["grad_f64/val"]
    assert np.linalg.norm(d_o - ref_do) <= 1e-4 * np.linalg.norm(ref_do)
    got = mod.offsets.grad.double().cpu().numpy()
    err = np.abs(got - z["gtheta_f64"])
    ratio = float((err / z["gtheta_abs"]).max())
    with capsys.disabled():
        print("\n%s theta.grad: worst |err| / sum|terms| %.2e, |err| / |total| %.2e"
              % (case, ratio, float(np.linalg.norm(err) / np.linalg.norm(z["gtheta_f64"]))))
    assert ratio <= 1e-4


def test_backproj_loss_dev_matches_host_twin():
    """lf_backproj_loss_dev on the device (all three passes, the per-lane partials and the last-CTA reduction) against its
    host twin, and _FusedBackprojLossWarp's lane_scale branch against per-lane host calls."""
    from lanedetection_end2end_b200.Loss_crit import _FusedBackprojLossWarp
    B, L, n = 5, 4, 4
    rng = np.random.default_rng(11)
    _, Mi, _, yk = hg.warp_host(np.array([0.003, -0.002, 0.004, 0.001, -0.006]), 256)
    Mi = np.ascontiguousarray(Mi.reshape(-1))
    beta = rng.standard_normal((B, L, n)) * np.array([1e-6, 1e-3, 1e-1, 1.0]) + np.array([0, 0, 0, 250.0])
    xgt = rng.uniform(100, 500, (B, L, 56))
    valid = (rng.uniform(size=(B, L, 56)) > 0.25).astype(np.float64)
    valid[:, 3] = 0.0                                    # a lane with nothing valid
    h = _capi.lib()

    def host(b, x, v, nl):
        lane, lo, db, xc, g = np.zeros(nl), np.zeros(1), np.zeros_like(b), np.zeros_like(x), np.zeros(65)
        _capi.check(h.lf_backproj_loss_dev_host(yk.ctypes.data, Mi.ctypes.data, b.ctypes.data, x.ctypes.data, v.ctypes.data,
                                                B, nl, n, lane.ctypes.data, lo.ctypes.data, db.ctypes.data, xc.ctypes.data,
                                                g.ctypes.data), "lf_backproj_loss_dev_host")
        return lane, lo[0], db, xc, g

    lane_h, loss_h, db_h, xc_h, g_h = host(beta, xgt, valid, L)
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dev = {k: torch.empty(*s, dtype=torch.float64, device="cuda") for k, s in
           (("lane", (L,)), ("loss", (1,)), ("db", (B, L, n)), ("xc", (B, L, 56)), ("gp", (L, 65)), ("g", (65,)))}
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    p = _capi.ptr
    bt, xt, vt, yt, mt = c(beta), c(xgt), c(valid), c(yk), c(Mi)
    for _ in range(2):                                   # the ticket resets itself: a second launch gives the same result
        _capi.call("lf_backproj_loss_dev", p(yt), p(mt), p(bt), p(xt), p(vt), B, L, n, p(dev["lane"]), p(dev["loss"]),
                   p(dev["db"]), p(dev["xc"]), p(dev["gp"]), p(dev["g"]), p(ticket), _capi.stream_ptr())
    close = lambda a, b: np.abs(a.cpu().numpy() - b).max() <= 1e-12 * max(np.abs(b).max(), 1e-300)
    assert close(dev["lane"], lane_h) and close(dev["loss"], np.array([loss_h]))
    assert close(dev["db"], db_h) and close(dev["xc"], xc_h) and close(dev["g"], g_h)
    assert np.all(g_h[3:6] == 0) and np.abs(g_h).max() > 0

    # lane_scale: loss = mean_l(ls_l lane_l); the constants' gradient = sum_l ls_l g_l / L
    ls = torch.tensor([0.5, 2.0, 1.5, 3.0], dtype=torch.float64, device="cuda")
    Minv_t = mt.clone().requires_grad_(True)
    yk_t = yt.clone().requires_grad_(True)
    crit = types.SimpleNamespace(_fused_ticket=lambda d: ticket)
    loss, _ = _FusedBackprojLossWarp.apply(bt, xt, vt, Minv_t, yk_t, crit, ls)
    loss.backward()
    want = sum(ls[l].item() * host(np.ascontiguousarray(beta[:, l:l + 1]), np.ascontiguousarray(xgt[:, l:l + 1]),
                                    np.ascontiguousarray(valid[:, l:l + 1]), 1)[4] for l in range(L)) / L
    want_loss = sum(ls[l].item() * lane_h[l] for l in range(L)) / L
    assert abs(loss.item() - want_loss) <= 1e-12 * abs(want_loss)
    assert close(Minv_t.grad, want[:9]) and close(yk_t.grad, want[9:])


def test_projections_learned_warp_equals_host_constants():
    """Projections.compute_all on a learned warp (lf_backproj_loss_dev) against the host-constant path (lf_backproj_loss)
    given the same M^-1, y' and Y56: the same bits."""
    from lanedetection_end2end_b200.inference import Projections
    R, mask, B, L, n = 256, 52, 3, 4, 4
    mod = hg.LearnedHomography(R, mask).cuda()
    with torch.no_grad():
        mod.offsets.copy_(torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01]))
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        warp = mod(st)
    args = _args("--clas", "True")
    learned = Projections(args).bind(types.SimpleNamespace(homography=mod))
    rng = np.random.default_rng(2)
    betas = [torch.from_numpy(rng.standard_normal((B, n, 1)) * np.array([[1e-6], [1e-3], [1e-1], [1.0]])
                              + np.array([[0], [0], [0], [250.0]])).cuda() for _ in range(L)]
    got = learned.compute_all(betas)

    fixed = Projections(_args("--clas", "True", "--learn_homography", "False"))
    crit = fixed._crit
    yp = warp.yk.detach().cpu()
    y = 255 - yp
    crit.y_prime = yp.clone()
    crit.Y = torch.stack([(y * y) * y, y * y, y, torch.ones_like(y)], 1)      # the kernel's product order
    crit.M_inv = warp.Minv.detach().cpu().view(3, 3).clone()
    want = fixed.compute_all(betas)
    assert torch.equal(got, want)


def test_trainsh_step_theta_grad_against_fp64():
    """A train.sh-shaped step (4 lanes, order 3, --clas, tf32x3): theta.grad of the whole step against the float64 chain
    (8x8-solve warp -> least squares -> back-projection loss) on the step's own decoder maps, per entry within 1e-4 of
    the sum of the absolute per-row and per-constant terms."""
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss, fused_backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    assert ops_net.CONV_MODE == "tf32x3"
    torch.manual_seed(0)
    args = _args("--clas", "True", "--mask_percentage", "0.2")
    B, R, L, order = 2, 256, 4, 3
    model = Net(args).cuda()
    with torch.no_grad():
        model.homography.offsets.copy_(torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01]))
    crit = backprojection_loss(args).bind(model)
    x = torch.rand(B, 3, R, 2 * R, device="cuda")
    rng = np.random.default_rng(3)
    xgt = torch.from_numpy(rng.uniform(150, 350, (B, L, 56))).cuda()
    valid = torch.ones(B, L, 56, dtype=torch.float64, device="cuda")
    out = model(x, torch.zeros(B, 4), True)
    loss, _ = fused_backprojection_loss(crit, out[:L], xgt, valid)
    line = torch.nn.functional.binary_cross_entropy_with_logits(out[6], torch.ones_like(out[6]))
    (loss + line.double()).backward()
    got = model.homography.offsets.grad.double().cpu()

    maps = out[5].detach().double().cpu()
    mask = model.zero_rows
    th = torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01], dtype=torch.float32).double().requires_grad_(True)

    def rows(t):
        M, Mi = warp_fp64(t, R)
        v = torch.arange(R, dtype=torch.float64)
        den = M[2, 1] * v + M[2, 2]
        y_d = (torch.arange(160, 720, 10) - 80).double() / 2.5
        yk = (M[1, 1] * y_d + M[1, 2]) / (M[2, 1] * y_d + M[2, 2])
        return torch.stack([M[0, 0] / den, (M[0, 1] * v + M[0, 2]) / den, (M[1, 1] * v + M[1, 2]) / den], 1), yk, Mi

    rowp, yk, Mi = rows(th)
    rowp_l, yk_l, Mi_l = (t.detach().clone().requires_grad_(True) for t in (rowp, yk, Mi))
    bet = _lsq_fp64(maps, rowp_l, order, mask, "square", 0.0, False)
    Y = torch.stack([(255 - yk_l) ** (order - i) for i in range(order + 1)], 1)
    xp = bet @ Y.t()
    xcal = (Mi_l[0, 0] * xp + Mi_l[0, 1] * yk_l + Mi_l[0, 2]) / (Mi_l[2, 0] * xp + Mi_l[2, 1] * yk_l + Mi_l[2, 2])
    vv = valid.cpu()
    lref = (((xgt.cpu() - xcal) * vv) ** 2).sum((0, 2)) / vv.sum((0, 2))
    lref.mean().backward()
    ref = torch.autograd.grad((rowp * rowp_l.grad).sum() + (yk * yk_l.grad).sum() + (Mi * Mi_l.grad).sum(), th)[0]
    absterm = torch.zeros(5, dtype=torch.float64)
    for j in range(5):
        e = torch.zeros(5, dtype=torch.float64)
        e[j] = 1.0
        _, (jr, jy, jm) = torch.func.jvp(rows, (th.detach(),), (e,))
        absterm[j] = (rowp_l.grad * jr).abs().sum() + (yk_l.grad * jy).abs().sum() + (Mi_l.grad * jm).abs().sum()
    ratio = float(((got - ref).abs() / absterm).max())
    print("train.sh step theta.grad: worst |err| / sum|terms| %.2e" % ratio)
    assert ratio <= 1e-4


def test_train_epoch_equals_eager_loop(paths):
    """engine.train_epoch with --learn_homography against the eager loop on the same fused functions: parameters (the
    warp's offsets among them), optimizer state and losses.avg bit for bit, and the offsets move."""
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    args = te.make_args("clas4", paths[0])
    args.learn_homography = True
    train, _, _ = te.loaders(paths, args)
    batches = list(train)
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    crits[0].bind(ma)
    want_loss, _, _, skipped = te.eager_train(batches, ma, oa, *crits, args, te.per_lane_loss)
    got_loss, _ = engine.train_epoch(batches, mb, ob, *crits, args, 0)
    assert not skipped and got_loss == want_loss
    assert ma.homography.offsets.abs().sum() > 0
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
