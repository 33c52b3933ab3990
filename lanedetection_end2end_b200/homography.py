"""Learned bird's-eye-view homography (``--learn_homography``) and the predicted per-image homography
(``--predict_homography``, ``PredictedHomography`` below).

``--learn_homography``: the warp of ``get_homography(resize)`` with its source
corners shifted by a learnable ``offsets`` [5] (float32, initialised to zero), so that the back-projection ``Net`` can
fine-tune the fixed transformation together with the network.

  offsets[0..3]  x of the four source corners, in units of the image width 2*resize
  offsets[4]     row of the two top source corners, in units of resize

The destination corners and the bottom row stay fixed, so the warp stays row-preserving (M[1,0] = M[2,0] = 0) and the
row-separable least-squares kernels and the loss's sample rows stay exact.  Every forward builds M, M^-1 and the
least-squares tables on the device (lf_homography_tables); the backward reduces the gradients of the least-squares
layer (lf_lsq_grid_grad) and of the loss (lf_backproj_loss_dev) to ``offsets.grad`` (lf_homography_bwd).  DESIGN.md
section "Learned homography" has the maths.
"""
import torch
import torch.nn as nn

from . import _capi

N_SAMPLES = 56


class WarpTables:
    """One forward's warp: ``rowp`` [R, 3] f64 (alpha_v, gamma_v, y'_v, differentiable), ``Minv`` [9] and ``yk`` [56]
    f64 (differentiable), ``M`` [9] f64, and the least-squares tables ``xtab`` [R*2R] / ``yrow`` [R] f32."""

    ytab = None
    rowsep = True

    def __init__(self, rowp, Minv, yk, M, xtab, yrow, H, W, delta=None):
        self.rowp, self.Minv, self.yk, self.M = rowp, Minv, yk, M
        self.xtab, self.yrow, self.H, self.W = xtab, yrow, H, W
        # per image (PredictedHomography): every field gains a leading batch dimension -- rowp [B, R, 3], Minv / M
        # [B, 9], yk [B, 56], xtab [B, R*2R], yrow [B, R] -- and delta holds the per-image parameters: [B, 3] f64
        # tanh(z) / 16 for the destination corners, [B, 5] f32 theta = tanh(z) / 64 for the source corners
        self.delta = delta
        self.per_image = delta is not None


class _WarpFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, theta, resize, mask_rows, y_const, status):
        _capi.require_cuda(theta, status)
        dev = theta.device
        R, W = resize, 2 * resize
        M = torch.empty(9, dtype=torch.float64, device=dev)
        Minv = torch.empty(9, dtype=torch.float64, device=dev)
        rowp = torch.empty(R, 3, dtype=torch.float64, device=dev)
        yk = torch.empty(N_SAMPLES, dtype=torch.float64, device=dev)
        xtab = torch.empty(R * W, dtype=torch.float32, device=dev)
        yrow = torch.empty(R, dtype=torch.float32, device=dev)
        theta = theta.detach().contiguous()
        _capi.call("lf_homography_tables", _capi.ptr(theta), R, mask_rows, float(y_const), _capi.ptr(M), _capi.ptr(Minv), _capi.ptr(rowp),
                   _capi.ptr(xtab), _capi.ptr(yrow), _capi.ptr(yk), _capi.ptr(status), _capi.stream_ptr(),
                   nbytes=4 * R * W)
        ctx.save_for_backward(theta)
        ctx.cfg = (R, mask_rows)
        ctx.mark_non_differentiable(M, xtab, yrow)
        return rowp, Minv, yk, M, xtab, yrow

    @staticmethod
    def backward(ctx, g_rowp, g_minv, g_yk, _gm, _gx, _gy):
        (theta,) = ctx.saved_tensors
        R, mask_rows = ctx.cfg
        prep = lambda g: None if g is None else g.to(torch.float64).contiguous()
        g_theta = torch.empty(5, dtype=torch.float32, device=theta.device)
        _capi.call("lf_homography_bwd", _capi.ptr(theta), R, mask_rows, _capi.ptr(prep(g_rowp)), _capi.ptr(prep(g_minv)),
                   _capi.ptr(prep(g_yk)), _capi.ptr(g_theta), _capi.stream_ptr())
        return g_theta, None, None, None, None


class LearnedHomography(nn.Module):
    """``offsets`` [5] and the per-forward warp.  ``forward(status)`` builds the warp (ORing LF_STATUS_NONFINITE into the
    device int32 ``status`` when an unmasked row reaches the vanishing line), keeps it as ``self.current`` for the loss
    bound to the model (``backprojection_loss.bind``) and returns it."""

    def __init__(self, resize, mask_rows, y_const=255.0):
        super().__init__()
        self.resize, self.mask_rows, self.y_const = resize, mask_rows, y_const
        self.offsets = nn.Parameter(torch.zeros(5, dtype=torch.float32))
        self.current = None

    def forward(self, status):
        out = _WarpFunction.apply(self.offsets, self.resize, self.mask_rows, self.y_const, status)
        rowp, Minv, yk, M, xtab, yrow = out
        self.current = WarpTables(rowp, Minv, yk, M, xtab, yrow, self.resize, 2 * self.resize)
        return self.current


def warp_host(theta, resize):
    """(M [3,3], M^-1 [3,3], rowp [R,3], yk [56]) of ``theta`` as float64 numpy arrays, computed on the host by the
    kernel's own closed form (lf_homography_host)."""
    import numpy as np
    th = np.ascontiguousarray(np.asarray(theta, dtype=np.float32).reshape(5))
    Mpair = np.zeros(18)
    rowp = np.zeros((resize, 3))
    yk = np.zeros(N_SAMPLES)
    _capi.check(_capi.lib().lf_homography_host(th.ctypes.data, resize, Mpair.ctypes.data, rowp.ctypes.data, yk.ctypes.data),
                "lf_homography_host")
    return Mpair[:9].reshape(3, 3), Mpair[9:].reshape(3, 3), rowp, yk


# the two parametrisations of the branch's output z (--predict_homography_corners): entries of z per image, dtype of
# the per-image parameters the tables entry point writes (delta / theta), and the tables and backward entry points
CORNERS = {"destination": (3, torch.float64, "lf_predicted_homography_tables", "lf_predicted_homography_bwd"),
           "source": (5, torch.float32, "lf_predicted_homography_source_tables", "lf_predicted_homography_source_bwd")}


def _predicted_forward(ctx, corners, z, resize, mask_rows, y_const, status):
    _capi.require_cuda(z, status)
    nz, param_dtype, tables, _ = CORNERS[corners]
    z = z.detach().float().contiguous()
    B, dev = z.shape[0], z.device
    if tuple(z.shape) != (B, nz):
        raise ValueError("%s corners need z [B, %d], got %s" % (corners, nz, tuple(z.shape)))
    R, W = resize, 2 * resize
    f64 = dict(dtype=torch.float64, device=dev)
    param = torch.empty(B, nz, dtype=param_dtype, device=dev)
    M = torch.empty(B, 9, **f64)
    Minv = torch.empty(B, 9, **f64)
    rowp = torch.empty(B, R, 3, **f64)
    yk = torch.empty(B, N_SAMPLES, **f64)
    xtab = torch.empty(B, R * W, dtype=torch.float32, device=dev)
    yrow = torch.empty(B, R, dtype=torch.float32, device=dev)
    p = _capi.ptr
    _capi.call(tables, p(z), B, R, mask_rows, float(y_const), p(param), p(M), p(Minv), p(rowp), p(xtab), p(yrow), p(yk),
               p(status), _capi.stream_ptr(), nbytes=4 * B * R * W)
    ctx.save_for_backward(z)
    ctx.cfg = (corners, R, mask_rows)
    ctx.mark_non_differentiable(M, xtab, yrow, param)
    return rowp, Minv, yk, M, xtab, yrow, param


def _predicted_backward(ctx, g_rowp, g_minv, g_yk):
    (z,) = ctx.saved_tensors
    corners, R, mask_rows = ctx.cfg
    bwd = CORNERS[corners][3]
    prep = lambda g: None if g is None else g.to(torch.float64).contiguous()
    g_z = torch.empty_like(z)
    extra = (None,) if corners == "source" else ()         # dL/dtheta in f64: not needed here
    _capi.call(bwd, _capi.ptr(z), z.shape[0], R, mask_rows, _capi.ptr(prep(g_rowp)), _capi.ptr(prep(g_minv)),
               _capi.ptr(prep(g_yk)), _capi.ptr(g_z), *extra, _capi.stream_ptr())
    return g_z, None, None, None, None


class _PredictedWarpFunction(torch.autograd.Function):
    """z [B, 3] -> the destination-corner warps: (rowp, Minv, yk, M, xtab, yrow, delta [B, 3] f64)."""

    @staticmethod
    def forward(ctx, z, resize, mask_rows, y_const, status):
        return _predicted_forward(ctx, "destination", z, resize, mask_rows, y_const, status)

    @staticmethod
    def backward(ctx, g_rowp, g_minv, g_yk, _gm, _gx, _gy, _gd):
        return _predicted_backward(ctx, g_rowp, g_minv, g_yk)


class _PredictedSourceWarpFunction(torch.autograd.Function):
    """z [B, 5] -> the source-corner warps: (rowp, Minv, yk, M, xtab, yrow, theta [B, 5] f32), image b's tables those of
    --learn_homography's warp at theta_b = tanh(z_b) / 64."""

    @staticmethod
    def forward(ctx, z, resize, mask_rows, y_const, status):
        return _predicted_forward(ctx, "source", z, resize, mask_rows, y_const, status)

    @staticmethod
    def backward(ctx, g_rowp, g_minv, g_yk, _gm, _gx, _gy, _gt):
        return _predicted_backward(ctx, g_rowp, g_minv, g_yk)


_PREDICTED_FUNCTIONS = {"destination": _PredictedWarpFunction, "source": _PredictedSourceWarpFunction}


class SpatialTransformer(nn.Module):
    """The reference's ``Spatial_transformer_net`` (Backprojection_Loss/Networks/Least_squares_net.py) on the encoder
    map [B, 128, rows, cols]: conv 1x1 / 3x3 / 3x3 with BatchNorm + ReLU, max-pool 2x2, conv 3x3 + BatchNorm + ReLU,
    Linear + ReLU, Linear(128, nz) -> z [B, nz] (nz = 3, the reference's; 5 for the source corners).  The modules only
    hold the parameters under the reference's names; forward runs on the library's kernels as the Classification heads
    do (ops_heads).  As in the reference, ``conv5`` is built and never used (it receives no gradient) and ``conv4_bn`` is
    registered once, where its first assignment put it.
    ``fully_connected2`` starts at zero (``zero_init``: define_init_weights leaves it there), so a new model starts from
    the fixed warp."""

    def __init__(self, size, channels_in, nz=3):
        super().__init__()
        self.conv1 = nn.Conv2d(channels_in, 128, 1)
        self.conv1_bn = nn.BatchNorm2d(128)
        self.conv2 = nn.Conv2d(128, 128, 3, padding=1)
        self.conv2_bn = nn.BatchNorm2d(128)
        self.conv3 = nn.Conv2d(128, 64, 3, padding=1)
        self.conv3_bn = nn.BatchNorm2d(64)
        self.conv4 = nn.Conv2d(64, 64, 3, padding=1)
        self.conv4_bn = nn.BatchNorm2d(64)
        rows, cols = size
        self.size = (rows, cols)
        self.maxpool = nn.MaxPool2d((2, 2), stride=2)
        self.conv5 = nn.Conv2d(64, 64, 3, padding=1)
        self.fully_connected1 = nn.Linear(64 * rows * cols // 4, 128)
        self.fully_connected2 = nn.Linear(128, nz)
        self.fully_connected2.zero_init = True
        with torch.no_grad():
            self.fully_connected2.weight.zero_()
            self.fully_connected2.bias.zero_()

    def forward(self, x):
        from . import ops_heads, ops_net
        from .Networks.ERFNet import _track
        h = ops_net.as_nhwc(x)
        _capi.require_cuda(h)
        if tuple(h.shape[1:3]) != self.size:
            raise ValueError("spatial transformer built for a %dx%d encoder map, got %dx%d" % (self.size + tuple(h.shape[1:3])))
        for conv, bn in ((self.conv1, self.conv1_bn), (self.conv2, self.conv2_bn), (self.conv3, self.conv3_bn)):
            h = ops_heads.conv_bn_relu(h, conv, bn, self.training, _track)
        h = ops_heads.MaxPool2Function.apply(h)
        h = ops_heads.conv_bn_relu(h, self.conv4, self.conv4_bn, self.training, _track)
        f = ops_heads.NchwFlatFunction.apply(h)
        f = ops_heads.LinearFunction.apply(f, self.fully_connected1.weight, self.fully_connected1.bias, True)
        return ops_heads.LinearFunction.apply(f, self.fully_connected2.weight, self.fully_connected2.bias, False)


class PredictedHomography(nn.Module):
    """``--predict_homography``: the reference's ``DLT`` module -- the spatial-transformer branch (``spatial_trans``)
    and one row-preserving warp per image built on the device from its output z.  ``corners`` picks the parametrisation
    (``--predict_homography_corners``): ``"destination"``, the reference's (z [B, 3], delta = tanh(z) / 16 moves the
    destination corners; lf_predicted_homography_tables), or ``"source"`` (z [B, 5], theta = tanh(z) / 64 moves the
    source corners as ``LearnedHomography.offsets`` does; lf_predicted_homography_source_tables).  Only the source
    corners change what the loss sees (NOTES.md "Predicted homography").  ``forward(encoder_map, status)`` keeps the
    batched WarpTables (``delta`` holding delta or theta) as ``self.current`` for the loss bound to the model and
    returns it; ORs LF_STATUS_NONFINITE into ``status`` when any image's unmasked row reaches its vanishing line."""

    def __init__(self, resize, mask_rows, size=(32, 64), channels_in=128, y_const=255.0, corners="destination"):
        super().__init__()
        if corners not in CORNERS:
            raise ValueError("corners must be one of %s, got %r" % (sorted(CORNERS), corners))
        self.resize, self.mask_rows, self.y_const, self.corners = resize, mask_rows, y_const, corners
        self.spatial_trans = SpatialTransformer(size, channels_in, nz=CORNERS[corners][0])
        self.current = None

    def forward(self, encoder_map, status):
        z = self.spatial_trans(encoder_map)
        rowp, Minv, yk, M, xtab, yrow, param = _PREDICTED_FUNCTIONS[self.corners].apply(z, self.resize, self.mask_rows,
                                                                                       self.y_const, status)
        self.current = WarpTables(rowp, Minv, yk, M, xtab, yrow, self.resize, 2 * self.resize, delta=param)
        return self.current


def predicted_warp_host(delta, resize):
    """(M [3,3], M^-1 [3,3], rowp [R,3], yk [56]) of one image's delta [3] (inside [-1/16, 1/16]^3) as float64 numpy
    arrays, by the kernel's own closed form on the host (lf_predicted_homography_host)."""
    import numpy as np
    d = np.ascontiguousarray(np.asarray(delta, dtype=np.float64).reshape(3))
    Mpair = np.zeros(18)
    rowp = np.zeros((resize, 3))
    yk = np.zeros(N_SAMPLES)
    _capi.check(_capi.lib().lf_predicted_homography_host(d.ctypes.data, resize, Mpair.ctypes.data, rowp.ctypes.data,
                                                           yk.ctypes.data), "lf_predicted_homography_host")
    return Mpair[:9].reshape(3, 3), Mpair[9:].reshape(3, 3), rowp, yk


def predicted_source_warp_host(z, resize):
    """(theta [5] f32, M [3,3], M^-1 [3,3], rowp [R,3], yk [56]) of one image's z [5] in the source-corner
    parametrisation, as numpy arrays, by the kernel's own code on the host (lf_predicted_homography_source_host)."""
    import numpy as np
    zz = np.ascontiguousarray(np.asarray(z, dtype=np.float32).reshape(5))
    theta = np.zeros(5, np.float32)
    Mpair = np.zeros(18)
    rowp = np.zeros((resize, 3))
    yk = np.zeros(N_SAMPLES)
    _capi.check(_capi.lib().lf_predicted_homography_source_host(zz.ctypes.data, resize, theta.ctypes.data, Mpair.ctypes.data,
                                                                  rowp.ctypes.data, yk.ctypes.data),
                "lf_predicted_homography_source_host")
    return theta, Mpair[:9].reshape(3, 3), Mpair[9:].reshape(3, 3), rowp, yk
