"""Learned bird's-eye-view homography (--learn_homography) on the CPU: the closed-form warp against an exact rational
solve and cv2, the least-squares layer's table gradient against autograd, the loss's constant gradient chained to
theta against autograd, and the model's refusals and state_dict keys."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from lanedetection_end2end_b200 import _capi, homography as hg
from lanedetection_end2end_b200.Networks.utils import define_args, get_homography


def _corners(theta, R):
    w = 2 * R
    f = lambda v: float(np.float32(v))
    src = [[f(0.45 * w), f(0.20 * R)], [f(0.55 * w), f(0.20 * R)], [f(0.02 * w), f(R - 1)], [f(0.97 * w), f(R - 1)]]
    dst = [[f(0.45 * w), f(0.20 * R)], [f(0.55 * w), f(0.20 * R)], [f(0.45 * w), f(R - 1)], [f(0.55 * w), f(R - 1)]]
    th = np.asarray(theta, dtype=np.float32).astype(np.float64)
    for i in range(4):
        src[i][0] += th[i] * w
    src[0][1] += th[4] * R
    src[1][1] += th[4] * R
    return src, dst


def _exact(src, dst):
    """The 8x8 perspective system solved in rational arithmetic (m22 = 1)."""
    A, b = [], []
    for (x, y), (X, Y) in zip(src, dst):
        x, y, X, Y = (Fraction(v) for v in (x, y, X, Y))
        A.append([x, y, 1, 0, 0, 0, -X * x, -X * y]); b.append(X)
        A.append([0, 0, 0, x, y, 1, -Y * x, -Y * y]); b.append(Y)
    n = 8
    M = [row[:] + [bb] for row, bb in zip(A, b)]
    for c in range(n):
        p = next(r for r in range(c, n) if M[r][c] != 0)
        M[c], M[p] = M[p], M[c]
        for r in range(n):
            if r != c and M[r][c] != 0:
                f = M[r][c] / M[c][c]
                M[r] = [a - f * q for a, q in zip(M[r], M[c])]
    sol = [M[i][n] / M[i][i] for i in range(n)]
    return np.array([float(v) for v in sol] + [1.0]).reshape(3, 3)


THETAS = [np.zeros(5)] + [np.random.default_rng(s).uniform(-0.02, 0.02, 5) for s in range(3)]


@pytest.mark.parametrize("R", [256, 320])
@pytest.mark.parametrize("k", range(len(THETAS)))
def test_closed_form_matches_exact_solve(R, k):
    theta = THETAS[k]
    M, Mi, _, _ = hg.warp_host(theta, R)
    src, dst = _corners(theta, R)
    for got, ref in ((M, _exact(src, dst)), (Mi, _exact(dst, src))):
        assert np.abs(got - ref).max() / np.abs(ref).max() <= 1e-13
        assert got[1, 0] == 0.0 and got[2, 0] == 0.0


@pytest.mark.parametrize("R", [256, 320])
def test_theta_zero_matches_cv2(R):
    M, Mi, _, _ = hg.warp_host(np.zeros(5), R)
    Mc, Mic = get_homography(R)
    # cv2's unnormalised LU leaves 8.6e-7 at --resize 256: a tolerance, not the bits
    assert np.abs(M - Mc).max() / np.abs(Mc).max() < 1e-6
    assert np.abs(Mi - Mic).max() / np.abs(Mic).max() < 1e-6


def _torch_warp(theta, R):
    """M(theta), M^-1(theta) by a differentiable float64 8x8 solve (independent of the closed form)."""
    w = 2 * R
    f = lambda v: float(np.float32(v))
    t = theta.double()
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


def _act(o, kind):
    return {"none": o, "square": o ** 2, "abs": o.abs(), "relu": torch.relu(o), "sigmoid": torch.sigmoid(o),
            "softplus": torch.nn.functional.softplus(o)}[kind]


@pytest.mark.parametrize("order,chol,reg,act", [(0, False, 0.0, "none"), (1, False, 0.0, "square"), (2, True, 0.0, "abs"),
                                                (3, False, 0.0, "relu"), (2, False, 0.5, "sigmoid"),
                                                (3, True, 0.1, "softplus")])
def test_table_gradient_formulas(order, chol, reg, act):
    """The per-row formulas of lf_lsq_grid_grad, restated in NumPy from row sums, against torch autograd of the weighted
    least squares on the tables x = alpha_v u + gamma_v, y = 255 - y'_v (float64)."""
    rng = np.random.default_rng(order * 7 + int(chol))
    B, L, H, W, mask = 2, 2, 24, 16, 5
    o = torch.tensor(rng.standard_normal((B, L, H, W)))
    alpha = torch.tensor(rng.uniform(0.5, 2.0, H), requires_grad=True)
    gamma = torch.tensor(rng.uniform(-20, 20, H), requires_grad=True)
    yp = torch.tensor(np.sort(rng.uniform(0, 250, H)), requires_grad=True)
    gb = torch.tensor(rng.standard_normal((B, L, order + 1)))
    u = torch.arange(W, dtype=torch.float64)
    wts = _act(o, act) ** 2
    wts = torch.cat([torch.zeros_like(wts[:, :, :mask]), wts[:, :, mask:]], 2)
    x = alpha[:, None] * u + gamma[:, None]
    y = (255 - yp)[:, None].expand(H, W) / 255.0 * 255.0
    phi = torch.stack([y ** (order - i) for i in range(order + 1)], -1)              # [H, W, n]
    Z = torch.einsum("blhw,hwi,hwj->blij", wts, phi, phi) + reg * torch.eye(order + 1, dtype=torch.float64)
    X = torch.einsum("blhw,hwi,hw->bli", wts, phi, x)
    if chol:
        beta = torch.cholesky_solve(X.unsqueeze(-1), torch.linalg.cholesky(Z)).squeeze(-1)
    else:
        beta = (torch.linalg.inv(Z) @ X.unsqueeze(-1)).squeeze(-1)
    (beta * gb).sum().backward()

    wn = wts.detach().numpy()
    A, Bs, C = wn.sum(-1), (wn * x.detach().numpy()).sum(-1), (wn * np.arange(W)).sum(-1)       # [B, L, H]
    yv = 255 - yp.detach().numpy()
    ph = np.stack([yv ** (order - i) for i in range(order + 1)], -1)
    dph = np.stack([(order - i) * yv ** max(order - i - 1, 0) for i in range(order + 1)], -1)
    z = np.einsum("blij,blj->bli", np.linalg.inv(Z.detach().numpy()), gb.numpy())
    bt = beta.detach().numpy()
    pz, dz = np.einsum("hi,bli->blh", ph, z), np.einsum("hi,bli->blh", dph, z)
    pb, db = np.einsum("hi,bli->blh", ph, bt), np.einsum("hi,bli->blh", dph, bt)
    g_gamma = (pz * A).sum((0, 1))
    g_alpha = (pz * C).sum((0, 1))
    g_yp = -(dz * (Bs - pb * A) - pz * db * A).sum((0, 1))
    for got, ref in ((g_alpha, alpha.grad), (g_gamma, gamma.grad), (g_yp, yp.grad)):
        ref = ref.numpy()
        assert np.abs(got - ref).max() <= 1e-9 * np.abs(ref).max()


@pytest.mark.parametrize("order", [1, 2, 3])
def test_loss_constant_gradient_reaches_theta(order):
    """lf_backproj_loss_dev_host's dloss/d(M^-1, y'_k), chained by lf_homography_bwd_host, against autograd of the
    reference loss formula on M(theta) from a float64 8x8 solve."""
    R, B, L = 256, 3, 2
    n = order + 1
    rng = np.random.default_rng(order)
    theta = torch.tensor(rng.uniform(-0.01, 0.01, 5), dtype=torch.float32)
    beta = rng.standard_normal((B, L, n)) * np.array([1e-5, 1e-3, 1e-1, 1.0])[-n:] + np.r_[np.zeros(n - 1), 200.0]
    xgt = rng.uniform(100, 1100, (B, L, 56)) / 2.5
    valid = (rng.uniform(size=(B, L, 56)) > 0.3).astype(np.float64)

    th = theta.double().requires_grad_(True)
    M, Mi = _torch_warp(th, R)
    yd = (torch.arange(160, 720, 10) - 80).double() / 2.5
    yk = (M[1, 1] * yd + M[1, 2]) / (M[2, 1] * yd + M[2, 2])
    Y = torch.stack([(255 - yk) ** (order - i) for i in range(n)], 1)
    xp = torch.tensor(beta) @ Y.t()
    xcal = (Mi[0, 0] * xp + Mi[0, 1] * yk + Mi[0, 2]) / (Mi[2, 0] * xp + Mi[2, 1] * yk + Mi[2, 2])
    err = (torch.tensor(xgt) - xcal) * torch.tensor(valid)
    loss = ((err ** 2).sum((0, 2)) / torch.tensor(valid).sum((0, 2))).mean()
    loss.backward()

    _, Mi_h, _, yk_h = hg.warp_host(theta.numpy(), R)
    h = _capi.lib()
    c = lambda a: np.ascontiguousarray(a, dtype=np.float64)
    beta_c, xgt_c, valid_c, Mi_c, yk_c = c(beta), c(xgt), c(valid), c(Mi_h.reshape(-1)), c(yk_h)
    lane, lo, db, g = np.zeros(L), np.zeros(1), np.zeros((B, L, n)), np.zeros(65)
    _capi.check(h.lf_backproj_loss_dev_host(yk_c.ctypes.data, Mi_c.ctypes.data, beta_c.ctypes.data, xgt_c.ctypes.data,
                                            valid_c.ctypes.data, B, L, n, lane.ctypes.data, lo.ctypes.data, db.ctypes.data,
                                            None, g.ctypes.data), "lf_backproj_loss_dev_host")
    assert abs(lo[0] - loss.item()) <= 1e-12 * abs(loss.item())
    th_c = np.ascontiguousarray(theta.numpy())
    gt = np.zeros(5)
    _capi.check(h.lf_homography_bwd_host(th_c.ctypes.data, R, 0, None, g[:9].ctypes.data, g[9:].ctypes.data, gt.ctypes.data),
                "lf_homography_bwd_host")
    ref = th.grad.double().numpy()
    assert np.abs(gt - ref).max() <= 1e-12 * np.abs(ref).max() + 1e-300


def test_row_gradient_reaches_theta():
    """lf_homography_bwd_host on dL/d(alpha, gamma, y') against autograd through the 8x8 solve."""
    R, mask = 256, 52
    rng = np.random.default_rng(5)
    theta = torch.tensor(rng.uniform(-0.01, 0.01, 5), dtype=torch.float32)
    g_rowp = rng.standard_normal((R, 3))
    g_rowp[:mask] = 0.0
    th = theta.double().requires_grad_(True)
    M, _ = _torch_warp(th, R)
    v = torch.arange(R, dtype=torch.float64)
    den = M[2, 1] * v + M[2, 2]
    rowp = torch.stack([M[0, 0] / den, (M[0, 1] * v + M[0, 2]) / den, (M[1, 1] * v + M[1, 2]) / den], 1)
    (rowp * torch.tensor(g_rowp)).sum().backward()
    gt = np.zeros(5)
    th_c, g_c = np.ascontiguousarray(theta.numpy()), np.ascontiguousarray(g_rowp)
    _capi.check(_capi.lib().lf_homography_bwd_host(th_c.ctypes.data, R, mask, g_c.ctypes.data, None, None, gt.ctypes.data),
                "lf_homography_bwd_host")
    ref = th.grad.double().numpy()
    assert np.abs(gt - ref).max() <= 1e-10 * np.abs(ref).max()


def _args(*extra):
    return define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--no_cuda", "--loss_policy", "backproject", "--batch_size", "2",
                                     "--resize", "256", "--nclasses", "2"] + list(extra))


def test_refusals_and_state_dict_keys():
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    fixed = Net(_args())
    learned = Net(_args("--learn_homography", "True"))
    assert set(learned.state_dict()) - set(fixed.state_dict()) == {"homography.offsets"}
    assert set(fixed.state_dict()) <= set(learned.state_dict())
    assert not any("homography" in k for k in fixed.state_dict())
    assert learned.homography.offsets.dtype == torch.float32 and not learned.homography.offsets.any()
    # a fixed-warp checkpoint starts the fine-tuning at offsets = 0
    missing, unexpected = learned.load_state_dict(fixed.state_dict(), strict=False)
    assert missing == ["homography.offsets"] and not unexpected
    with pytest.raises(ValueError):
        Net(_args("--learn_homography", "True", "--no_mapping", "True"))
    with pytest.raises(ValueError):
        Net(_args("--learn_homography", "True", "--loss_policy", "area"))
    crit = backprojection_loss(_args("--learn_homography", "True"))
    with pytest.raises(RuntimeError):
        crit(torch.zeros(2, 3, 1, dtype=torch.float64), torch.zeros(2, 56), torch.ones(2, 56))
    with pytest.raises(ValueError):
        crit.bind(fixed)
    assert backprojection_loss(_args()).warp() is None
