"""Learned bird's-eye-view homography (``--learn_homography``): the warp of ``get_homography(resize)`` with its source
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

    def __init__(self, rowp, Minv, yk, M, xtab, yrow, H, W):
        self.rowp, self.Minv, self.yk, self.M = rowp, Minv, yk, M
        self.xtab, self.yrow, self.H, self.W = xtab, yrow, H, W


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
