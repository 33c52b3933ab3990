"""--predict_homography without a GPU: the per-image warp's closed form against an exact rational solve of the
reference DLT's 6x6 equations, its fixed-warp start against get_homography, the dual-number backward against central
differences, the vanishing-line margin over the tanh box, and the flag's refusals and state_dict keys."""
from fractions import Fraction
from math import ceil

import numpy as np
import pytest
import torch

from lanedetection_end2end_b200 import _capi, homography as hg
from lanedetection_end2end_b200.Networks.utils import define_args, get_homography

BOX = 1.0 / 16          # |delta| < 1/16: tanh(z) / 16


def _pix(R):
    f = lambda v: Fraction(float(np.float32(v)))
    w = 2 * R
    return dict(w=w, sx=[f(0.45 * w), f(0.55 * w), f(0.02 * w), f(0.97 * w)], top=f(0.20 * R), bot=f(R - 1),
                dl=f(0.45 * w), dr=f(0.55 * w))


def _exact_dlt(delta, R):
    """M of the reference DLT (Least_squares_net.DLT.forward) on the back-projection corners in pixel units, its 6x6
    system solved in rational arithmetic; M^-1 its exact inverse normalised to m22 = 1."""
    c = _pix(R)
    d0, d1, d2 = (Fraction(float(v)) for v in delta)
    w, R_ = Fraction(c["w"]), Fraction(R)
    xd_l, xd_r, yd_t, yd_b = c["dl"] + d0 * w, c["dr"] + d1 * w, c["top"] + d2 * R_, c["bot"]
    ys_b, ys_t = c["bot"], c["top"]
    A = [[0, 0, 0, -ys_b, -1, ys_b * yd_b],
         [c["sx"][2], ys_b, 1, 0, 0, -ys_b * xd_l],
         [c["sx"][3], ys_b, 1, 0, 0, -ys_b * xd_r],
         [0, 0, 0, -ys_t, -1, ys_t * yd_t],
         [c["sx"][0], ys_t, 1, 0, 0, -ys_t * xd_l],
         [c["sx"][1], ys_t, 1, 0, 0, -ys_t * xd_r]]
    b = [-yd_b, xd_l, xd_r, -yd_t, xd_l, xd_r]
    n = 6
    Mx = [[Fraction(v) for v in row] + [Fraction(bb)] for row, bb in zip(A, b)]
    for col in range(n):
        p = next(r for r in range(col, n) if Mx[r][col] != 0)
        Mx[col], Mx[p] = Mx[p], Mx[col]
        for r in range(n):
            if r != col and Mx[r][col] != 0:
                f = Mx[r][col] / Mx[col][col]
                Mx[r] = [a - f * q for a, q in zip(Mx[r], Mx[col])]
    h = [Mx[i][n] / Mx[i][i] for i in range(n)]
    M = [[h[0], h[1], h[2]], [Fraction(0), h[3], h[4]], [Fraction(0), h[5], Fraction(1)]]
    # adjugate inverse, normalised so that [2][2] = 1
    cof = lambda i, j: (M[(i + 1) % 3][(j + 1) % 3] * M[(i + 2) % 3][(j + 2) % 3]
                        - M[(i + 1) % 3][(j + 2) % 3] * M[(i + 2) % 3][(j + 1) % 3])
    adj = [[cof(j, i) for j in range(3)] for i in range(3)]
    Mi = [[v / adj[2][2] for v in row] for row in adj]
    to = lambda m: np.array([[float(v) for v in row] for row in m])
    return to(M), to(Mi)


def _deltas():
    rng = np.random.default_rng(7)
    corners = [np.array([sx, sy, sz]) * BOX for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]
    return [np.zeros(3)] + [rng.uniform(-BOX, BOX, 3) for _ in range(4)] + corners


DELTAS = _deltas()


@pytest.mark.parametrize("R", [256, 320])
@pytest.mark.parametrize("k", range(len(DELTAS)))
def test_closed_form_matches_exact_dlt_solve(R, k):
    M, Mi, _, _ = hg.predicted_warp_host(DELTAS[k], R)
    Me, Mie = _exact_dlt(DELTAS[k], R)
    for got, ref in ((M, Me), (Mi, Mie)):
        assert np.abs(got - ref).max() / np.abs(ref).max() <= 1e-13
        assert got[1, 0] == 0.0 and got[2, 0] == 0.0 and got[2, 2] == 1.0


@pytest.mark.parametrize("R", [256, 320])
def test_zero_offsets_are_the_fixed_warp(R):
    M, Mi, rowp, yk = hg.predicted_warp_host(np.zeros(3), R)
    Mc, Mic = get_homography(R)
    # the tolerance DESIGN.md "Learned homography" states against cv2's unnormalised LU
    assert np.abs(M - Mc).max() / np.abs(Mc).max() < 1e-6
    assert np.abs(Mi - Mic).max() / np.abs(Mic).max() < 1e-6
    # and the learned warp's closed form at theta = 0, bit for bit
    Ml, Mil, rowpl, ykl = hg.warp_host(np.zeros(5), R)
    for a, b in ((M, Ml), (Mi, Mil), (rowp, rowpl), (yk, ykl)):
        np.testing.assert_array_equal(a, b)


def _objective(delta, R, mask_rows, g_rowp, g_minv, g_yk):
    _, Mi, rowp, yk = hg.predicted_warp_host(delta, R)
    return (g_rowp[mask_rows:] * rowp[mask_rows:]).sum() + (g_minv * Mi.reshape(-1)).sum() + (g_yk * yk).sum()


@pytest.mark.parametrize("R", [256, 320])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_dual_backward_matches_central_differences(R, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(-1.5, 1.5, 3).astype(np.float32)
    mask_rows = ceil(0.3 * R)
    g_rowp = rng.standard_normal((R, 3)) * np.array([10.0, 0.01, 0.01])
    g_minv = rng.standard_normal(9) * 1e-3
    g_yk = rng.standard_normal(56) * 1e-2
    g_z = np.zeros(3)
    p = lambda a: np.ascontiguousarray(a).ctypes.data
    rc = _capi.lib().lf_predicted_homography_bwd_host(p(z), R, mask_rows, p(g_rowp), p(g_minv), p(g_yk), p(g_z))
    assert rc == 0
    zd = z.astype(np.float64)
    for j in range(3):
        h = 1e-5
        zp, zm = zd.copy(), zd.copy()
        zp[j] += h
        zm[j] -= h
        fp = _objective(np.tanh(zp) / 16, R, mask_rows, g_rowp, g_minv, g_yk)
        fm = _objective(np.tanh(zm) / 16, R, mask_rows, g_rowp, g_minv, g_yk)
        fd = (fp - fm) / (2 * h)
        assert abs(g_z[j] - fd) <= 1e-6 * max(abs(fd), abs(g_z).max())


def _vanishing_row(delta, R):
    M, _, _, _ = hg.predicted_warp_host(delta, R)
    # den_v = m21 v + 1 vanishes at v = -1 / m21 (above the image when m21 > 0)
    return -1.0 / M[2, 1] if M[2, 1] < 0 else -np.inf


@pytest.mark.parametrize("R", [256, 320])
def test_vanishing_line_stays_above_the_mask(R):
    """The lowest vanishing-line row over the tanh box (a 9x9x9 grid including its corners) against mask_rows at the
    default --mask_percentage 0.3: the guard of lf_predicted_homography_tables cannot fire there (NOTES.md)."""
    grid = np.linspace(-BOX, BOX, 9)
    lowest = max(_vanishing_row(np.array([a, b, c]), R) for a in grid for b in grid for c in grid)
    mask_rows = ceil(0.3 * R)
    print("R=%d lowest vanishing row %.2f, mask_rows %d" % (R, lowest, mask_rows))
    assert lowest < mask_rows


def _args(*extra):
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--nclasses", "4",
                                     "--batch_size", "2", "--loss_policy", "backproject"] + list(extra))


REFERENCE_DLT_KEYS = [
    "spatial_trans.conv1.weight", "spatial_trans.conv1.bias",
    "spatial_trans.conv1_bn.weight", "spatial_trans.conv1_bn.bias", "spatial_trans.conv1_bn.running_mean",
    "spatial_trans.conv1_bn.running_var", "spatial_trans.conv1_bn.num_batches_tracked",
    "spatial_trans.conv2.weight", "spatial_trans.conv2.bias",
    "spatial_trans.conv2_bn.weight", "spatial_trans.conv2_bn.bias", "spatial_trans.conv2_bn.running_mean",
    "spatial_trans.conv2_bn.running_var", "spatial_trans.conv2_bn.num_batches_tracked",
    "spatial_trans.conv3.weight", "spatial_trans.conv3.bias",
    "spatial_trans.conv3_bn.weight", "spatial_trans.conv3_bn.bias", "spatial_trans.conv3_bn.running_mean",
    "spatial_trans.conv3_bn.running_var", "spatial_trans.conv3_bn.num_batches_tracked",
    "spatial_trans.conv4.weight", "spatial_trans.conv4.bias",
    "spatial_trans.conv4_bn.weight", "spatial_trans.conv4_bn.bias", "spatial_trans.conv4_bn.running_mean",
    "spatial_trans.conv4_bn.running_var", "spatial_trans.conv4_bn.num_batches_tracked",
    "spatial_trans.conv5.weight", "spatial_trans.conv5.bias",
    "spatial_trans.fully_connected1.weight", "spatial_trans.fully_connected1.bias",
    "spatial_trans.fully_connected2.weight", "spatial_trans.fully_connected2.bias",
]


def test_flag_defaults_to_off_and_adds_only_the_branch():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    assert _args().predict_homography is False
    torch.manual_seed(0)
    off = Net(_args())
    torch.manual_seed(0)
    on = Net(_args("--predict_homography", "True"))
    assert not hasattr(off, "DLT")
    dlt = ["DLT." + k for k in REFERENCE_DLT_KEYS]
    assert [k for k in on.state_dict() if k.startswith("DLT.")] == dlt
    assert [k for k in on.state_dict() if not k.startswith("DLT.")] == list(off.state_dict())
    st = on.DLT.spatial_trans
    assert tuple(st.fully_connected1.weight.shape) == (128, 64 * 32 * 64 // 4)
    assert tuple(st.conv5.weight.shape) == (64, 64, 3, 3)
    define_init_weights(on, "kaiming")
    assert not st.fully_connected2.weight.any() and not st.fully_connected2.bias.any()
    assert st.fully_connected1.weight.abs().sum() > 0
    # a fixed-warp checkpoint loads with strict=False and leaves exactly the branch missing (BatchNorm does not report a
    # missing num_batches_tracked)
    res = on.load_state_dict(off.state_dict(), strict=False)
    assert sorted(res.missing_keys) == sorted(k for k in dlt if "num_batches_tracked" not in k)
    assert not res.unexpected_keys


@pytest.mark.parametrize("extra", [["--learn_homography", "True"], ["--no_mapping", "True"], ["--loss_policy", "area"],
                                   ["--end_to_end", "False"], ["--pretrained", "True"], ["--resize", "258"]],
                         ids=["learn_homography", "no_mapping", "loss_policy", "end_to_end", "pretrained", "resize"])
def test_refusals_name_the_flag(extra):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    with pytest.raises(ValueError, match="--predict_homography"):
        Net(_args("--predict_homography", "True", *extra))


def test_bev_net_refuses():
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net as BevNet
    from lanedetection_end2end_b200.bev.Networks.utils import define_args as bev_args
    a = bev_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--batch_size", "2"])
    a.predict_homography = True
    with pytest.raises(ValueError, match="--predict_homography"):
        BevNet(a)


def test_header_declares_the_entry_points():
    import os
    import re
    from conftest import ROOT
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_predicted_homography_tables", "lf_predicted_homography_bwd", "lf_predicted_homography_host",
                 "lf_predicted_homography_bwd_host", "lf_lsq_fwd_per_image", "lf_lsq_bwd_per_image",
                 "lf_lsq_grid_grad_per_image", "lf_backproj_loss_per_image", "lf_backproj_loss_per_image_scratch"):
        assert re.search(r"\b%s\(" % name, hdr), name
