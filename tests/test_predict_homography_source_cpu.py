"""--predict_homography_corners source without a GPU: the per-image source-corner warp's closed form against an exact
rational 8x8 solve, its fixed-warp start, the backward against central differences and lf_homography_bwd's sum, the
vanishing-line margin over the tanh box, the refusals, the branch's shape and the header; and, in a float64 restatement
of the fit and the back-projection loss, that the loss sees the source corners and not the destination ones."""
from math import ceil

import numpy as np
import pytest
import torch

from test_homography_cpu import _corners, _exact

from lanedetection_end2end_b200 import _capi, homography as hg
from lanedetection_end2end_b200.Networks.utils import define_args, get_homography

BOX = 1.0 / 64          # |theta| < 1/64: tanh(z) / 64
ZS = [np.zeros(5, np.float32)] + [np.random.default_rng(s).uniform(-2.0, 2.0, 5).astype(np.float32) for s in range(4)] \
    + [np.array([30, -30, 30, -30, 30], np.float32), np.array([-30, 30, -30, 30, -30], np.float32)]   # the box's corners


@pytest.mark.parametrize("R", [256, 320])
@pytest.mark.parametrize("k", range(len(ZS)))
def test_closed_form_matches_exact_dlt_solve(R, k):
    theta, M, Mi, _, _ = hg.predicted_source_warp_host(ZS[k], R)
    assert theta.dtype == np.float32
    np.testing.assert_array_equal(theta, (np.tanh(ZS[k].astype(np.float64)) / 64).astype(np.float32))
    src, dst = _corners(theta, R)
    for got, ref in ((M, _exact(src, dst)), (Mi, _exact(dst, src))):
        assert np.abs(got - ref).max() / np.abs(ref).max() <= 1e-13
        assert got[1, 0] == 0.0 and got[2, 0] == 0.0 and got[2, 2] == 1.0


@pytest.mark.parametrize("R", [256, 320])
def test_zero_is_the_fixed_warp(R):
    theta, M, Mi, rowp, yk = hg.predicted_source_warp_host(np.zeros(5), R)
    Mc, Mic = get_homography(R)
    assert not theta.any()
    assert np.abs(M - Mc).max() / np.abs(Mc).max() < 1e-6
    assert np.abs(Mi - Mic).max() / np.abs(Mic).max() < 1e-6
    for a, b in zip((M, Mi, rowp, yk), hg.warp_host(np.zeros(5), R)):
        np.testing.assert_array_equal(a, b)


def _warp_f64(src, dst):
    """M (m22 = 1) of four point pairs by a float64 8x8 solve."""
    A, b = [], []
    for (x, y), (X, Y) in zip(src, dst):
        A.append([x, y, 1, 0, 0, 0, -X * x, -X * y])
        b.append(X)
        A.append([0, 0, 0, x, y, 1, -Y * x, -Y * y])
        b.append(Y)
    return np.append(np.linalg.solve(np.array(A), np.array(b)), 1.0).reshape(3, 3)


def _base(R):
    return _corners(np.zeros(5), R)


def source_warp(theta, R):
    """M of get_homography's corners with the source corners moved by theta [5] (float64, not rounded)."""
    src, dst = _base(R)
    w = 2 * R
    for i in range(4):
        src[i][0] += theta[i] * w
    src[0][1] += theta[4] * R
    src[1][1] += theta[4] * R
    return _warp_f64(src, dst)


def destination_warp(delta, R):
    """M with the destination corners moved as the reference DLT does: left / right column by delta_0 / delta_1 * 2R,
    top row by delta_2 * R."""
    src, dst = _base(R)
    w = 2 * R
    for i, j in ((0, 0), (2, 0), (1, 1), (3, 1)):
        dst[i][0] += delta[j] * w
    dst[0][1] += delta[2] * R
    dst[1][1] += delta[2] * R
    return _warp_f64(src, dst)


def _tables_f64(M, R):
    Mi = np.linalg.inv(M)
    Mi = Mi / Mi[2, 2]
    v = np.arange(R, dtype=np.float64)
    den = M[2, 1] * v + M[2, 2]
    rowp = np.stack([M[0, 0] / den, (M[0, 1] * v + M[0, 2]) / den, (M[1, 1] * v + M[1, 2]) / den], 1)
    ys = (160 + 10 * np.arange(56) - 80) / 2.5
    yk = (M[1, 1] * ys + M[1, 2]) / (M[2, 1] * ys + M[2, 2])
    return Mi, rowp, yk


def _objective(M, R, mask_rows, g_rowp, g_minv, g_yk):
    Mi, rowp, yk = _tables_f64(M, R)
    return (g_rowp[mask_rows:] * rowp[mask_rows:]).sum() + (g_minv * Mi.reshape(-1)).sum() + (g_yk * yk).sum()


def _bwd_host(name, x, R, mask_rows, g_rowp, g_minv, g_yk, extra=True):
    out = np.zeros(5)
    g_theta = np.zeros(5)
    p = lambda a: np.ascontiguousarray(a).ctypes.data
    args = (p(x), R, mask_rows, p(g_rowp), p(g_minv), p(g_yk), p(out)) + ((p(g_theta),) if extra else ())
    assert getattr(_capi.lib(), name)(*args) == 0
    return out, g_theta


@pytest.mark.parametrize("R", [256, 320])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_dual_backward_matches_central_differences(R, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(-1.5, 1.5, 5).astype(np.float32)
    mask_rows = ceil(0.3 * R)
    g_rowp = rng.standard_normal((R, 3)) * np.array([10.0, 0.01, 0.01])
    g_minv = rng.standard_normal(9) * 1e-3
    g_yk = rng.standard_normal(56) * 1e-2
    g_z, g_theta = _bwd_host("lf_predicted_homography_source_bwd_host", z, R, mask_rows, g_rowp, g_minv, g_yk)
    zd = z.astype(np.float64)
    for j in range(5):
        h = 1e-5
        zp, zm = zd.copy(), zd.copy()
        zp[j] += h
        zm[j] -= h
        fd = (_objective(source_warp(np.tanh(zp) / 64, R), R, mask_rows, g_rowp, g_minv, g_yk)
              - _objective(source_warp(np.tanh(zm) / 64, R), R, mask_rows, g_rowp, g_minv, g_yk)) / (2 * h)
        assert abs(g_z[j] - fd) <= 1e-6 * max(abs(fd), np.abs(g_z).max())
    # g_theta is dL/dtheta at the rounded theta, summed as lf_homography_bwd sums it: the learned warp's own bits
    theta, *_ = hg.predicted_source_warp_host(z, R)
    g_ref, _ = _bwd_host("lf_homography_bwd_host", theta, R, mask_rows, g_rowp, g_minv, g_yk, extra=False)
    np.testing.assert_array_equal(g_theta, g_ref)
    t = np.tanh(zd)
    np.testing.assert_allclose(g_z, g_theta * (1 - t * t) / 64, rtol=1e-14, atol=0)


def _vanishing_rows(R):
    """The vanishing-line row of every theta on a 9^5 grid of the box (corners included), by the kernel's closed form
    on the host (lf_homography_host)."""
    grid = np.linspace(-BOX, BOX, 9)
    th = np.stack(np.meshgrid(*[grid] * 5, indexing="ij"), -1).reshape(-1, 5).astype(np.float32)
    Mpair = np.zeros(18)
    lib = _capi.lib()
    rows = np.empty(len(th))
    for i, t in enumerate(th):
        t = np.ascontiguousarray(t)
        assert lib.lf_homography_host(t.ctypes.data, R, Mpair.ctypes.data, None, None) == 0
        # den_v = m21 v + 1 vanishes at v = -1 / m21; with m21 > 0 the line lies above the image
        rows[i] = -1.0 / Mpair[7] if Mpair[7] < 0 else -np.inf
    return rows


@pytest.mark.parametrize("R", [256, 320])
def test_vanishing_line_stays_above_the_mask(R):
    """The lowest vanishing-line row over the source box against mask_rows at --mask_percentage 0.2 (train.sh) and 0.3
    (the default): the guard of the tables kernel cannot fire inside the box (DESIGN.md 4f)."""
    lowest = _vanishing_rows(R).max()
    print("R=%d lowest vanishing row %.2f" % (R, lowest))
    for pct in (0.2, 0.3):
        assert lowest < ceil(pct * R), (pct, lowest)
    assert lowest == pytest.approx({256: 40.1, 320: 50.2}[R], abs=0.1)


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def _args(*extra):
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--nclasses", "4",
                                     "--batch_size", "2", "--loss_policy", "backproject"] + list(extra))


def test_flag_defaults_to_destination():
    assert _args().predict_homography_corners == "destination"
    with pytest.raises(SystemExit):
        _args("--predict_homography_corners", "both")


def test_source_needs_predict_homography():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    with pytest.raises(ValueError, match="--predict_homography_corners"):
        Net(_args("--predict_homography_corners", "source"))


@pytest.mark.parametrize("extra", [["--learn_homography", "True"], ["--no_mapping", "True"], ["--loss_policy", "area"],
                                   ["--end_to_end", "False"], ["--pretrained", "True"], ["--resize", "258"]],
                         ids=["learn_homography", "no_mapping", "loss_policy", "end_to_end", "pretrained", "resize"])
def test_source_keeps_every_refusal(extra):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    with pytest.raises(ValueError, match="--predict_homography"):
        Net(_args("--predict_homography", "True", "--predict_homography_corners", "source", *extra))


def test_bev_net_refuses():
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net as BevNet
    from lanedetection_end2end_b200.bev.Networks.utils import define_args as bev_args
    a = bev_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--batch_size", "2"])
    a.predict_homography_corners = "source"
    with pytest.raises(ValueError, match="--predict_homography"):
        BevNet(a)


def test_branch_shape_keys_and_destination_checkpoint():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    torch.manual_seed(0)
    dst = Net(_args("--predict_homography", "True"))
    torch.manual_seed(0)
    src = Net(_args("--predict_homography", "True", "--predict_homography_corners", "source"))
    assert dst.DLT.corners == "destination" and src.DLT.corners == "source"
    assert list(src.state_dict()) == list(dst.state_dict())
    fc2 = src.DLT.spatial_trans.fully_connected2
    assert tuple(fc2.weight.shape) == (5, 128) and tuple(fc2.bias.shape) == (5,)
    assert tuple(dst.DLT.spatial_trans.fully_connected2.weight.shape) == (3, 128)
    define_init_weights(src, "kaiming")
    assert not fc2.weight.any() and not fc2.bias.any()
    # a destination-mode checkpoint does not fill the 5-output layer; without its keys it loads with strict=False
    sd = dst.state_dict()
    with pytest.raises(RuntimeError, match="size mismatch"):
        src.load_state_dict(sd)
    fc2_keys = [k for k in sd if k.startswith("DLT.spatial_trans.fully_connected2.")]
    res = src.load_state_dict({k: v for k, v in sd.items() if k not in fc2_keys}, strict=False)
    assert sorted(res.missing_keys) == sorted(fc2_keys) and not res.unexpected_keys


def test_header_declares_the_entry_points():
    import os
    import re
    from conftest import ROOT
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_predicted_homography_source_tables", "lf_predicted_homography_source_bwd",
                 "lf_predicted_homography_source_host", "lf_predicted_homography_source_bwd_host"):
        assert re.search(r"\bint %s\(" % name, hdr), name
        assert name in open(os.path.join(ROOT, "INTEGRATION.md")).read(), name


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement: which corners does the loss see?
# ---------------------------------------------------------------------------------------------------------------------
H, W, MASK = 256, 512, 77
BOTTOM_X = (150.0, 230.0, 290.0, 370.0)


def lane_x(l, v):
    """Image column of synthetic lane l at image row v: straight toward a vanishing point near (256, 40), bent."""
    s = (v - 40.0) / (H - 1 - 40.0)
    return 256.0 + (BOTTOM_X[l] - 256.0) * s + 12.0 * s * s * (1 - s) * (1 if l % 2 else -1)


def ridge_maps(L=4, width=3.0):
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    return np.stack([np.exp(-0.5 * ((u - lane_x(l, v)) / width) ** 2) for l in range(L)])


def restated_loss(M, maps, order=2):
    """The weighted least-squares fit of each lane in the bird's-eye view of M (square activation, MASK masked rows)
    and the back-projection loss at the 56 sample rows, in float64."""
    L = maps.shape[0]
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    den = M[2, 0] * u + M[2, 1] * v + M[2, 2]
    xb = (M[0, 0] * u + M[0, 1] * v + M[0, 2]) / den
    yb = (M[1, 0] * u + M[1, 1] * v + M[1, 2]) / den
    Y = np.stack([(255.0 - yb) ** k for k in range(order, 0, -1)] + [np.ones_like(yb)], -1)
    Mi, _, yk = _tables_f64(M, H)
    ys = (160 + 10 * np.arange(56) - 80) / 2.5
    valid = ys >= MASK
    loss = 0.0
    for l in range(L):
        w = maps[l] ** 2
        w[:MASK] = 0.0
        beta = np.linalg.solve(np.einsum("hwi,hwj,hw->ij", Y, Y, w), np.einsum("hwi,hw,hw->i", Y, w, xb))
        xp = np.polyval(beta, 255.0 - yk)
        x_cal = (Mi[0, 0] * xp + Mi[0, 1] * yk + Mi[0, 2]) / (Mi[2, 0] * xp + Mi[2, 1] * yk + Mi[2, 2])
        loss += ((x_cal - lane_x(l, ys)) ** 2)[valid].mean()
    return loss / L


def relative_slopes(warp, n, maps, h=1e-4):
    """|dL/dp_j| / L per unit offset p_j, by central differences at p = 0."""
    L0 = restated_loss(warp(np.zeros(n), H), maps)
    out = []
    for j in range(n):
        e = np.zeros(n)
        e[j] = h
        out.append(abs(restated_loss(warp(e, H), maps) - restated_loss(warp(-e, H), maps)) / (2 * h) / L0)
    return np.array(out)


def test_loss_sees_the_source_corners_not_the_destination_ones():
    maps = ridge_maps()
    src = relative_slopes(source_warp, 5, maps)
    dst = relative_slopes(destination_warp, 3, maps)
    print("relative dL/dtheta source", src, "destination", dst)
    assert src.min() >= 1e4 * dst.max()
