"""Host side of the fused weighted least-squares layer: grid tables, workspace
and the ``torch.autograd.Function`` that calls ``lf_lsq_fwd`` / ``lf_lsq_bwd``
(include/lanefit_b200.h), or their ``*_keep`` variants when a per-pixel keep map is given, and their ``*_lanes`` forms
when only the first ``lanes`` maps are fitted (a lane curriculum).  Torch is plumbing here (device memory, streams,
autograd graph); all arithmetic on the maps happens in csrc/lsq.cu.
"""
import torch

from . import _capi

_TABLE_CACHE = {}
_WS_CACHE = {}


class GridTables:
    """De-interleaved, batch-invariant view of the reference's ``grid`` [N, H*W, 2]
    (BP/Networks/LSQ_layer.py:50-68):  xtab = grid[0,:,0],  ytab = const - grid[0,:,1]
    (:93-94, fp32 like the reference), and yrow [H] when ytab is constant along rows
    (true for every homography ``get_homography`` builds) -> row-separable fast kernel.
    """

    def __init__(self, grid, H, W, const):
        g = grid[0] if grid.dim() == 3 else grid
        if g.shape[0] != H * W or g.shape[1] != 2:
            raise ValueError("grid must be [N, H*W, 2]; got %s for H=%d W=%d" % (tuple(grid.shape), H, W))
        g = g.detach().to(torch.float32)
        self.xtab = g[:, 0].contiguous()
        self.ytab = (const - g[:, 1]).contiguous()
        y2 = self.ytab.view(H, W)
        # Row-separable?  Mathematically y' depends on the row only for every homography the reference
        # builds (M[1,0], M[2,0] are round-off zeros), but its fp32 bmm leaves 1-ulp differences inside a
        # few rows (10 of 256 at --resize 256).  Rows whose spread is <= 4 ulp are snapped to their median
        # (effect on beta ~1e-7 relative, far below the reference's own fp32 noise; DESIGN.md section 2).
        # Non-finite rows (the vanishing line at --resize 320, SURVEY.md 7.2 #10) count as constant: they
        # must be masked anyway.
        finite = torch.isfinite(y2)
        ysafe = torch.where(finite, y2, torch.zeros_like(y2))
        spread = ysafe.max(dim=1).values - ysafe.min(dim=1).values
        # ulp of the quantity the reference rounded: max(|y'|, |const - y'|) per row
        yp = torch.where(finite, g[:, 1].view(H, W), torch.zeros_like(y2))
        scale = torch.maximum(ysafe.abs().max(dim=1).values, yp.abs().max(dim=1).values).clamp_min(1e-30)
        row_ok = (spread <= 4 * 1.1920929e-07 * scale) | (~finite).any(dim=1)
        self.rowsep = bool(row_ok.all().item()) and (W % 4 == 0)
        self.yrow = y2.median(dim=1).values.contiguous() if self.rowsep else None
        self.H, self.W, self.const = H, W, const


def grid_tables(grid, H, W, const):
    key = (grid.data_ptr(), grid._version, tuple(grid.shape), str(grid.device), H, W, float(const))
    t = _TABLE_CACHE.get(key)
    if t is None:
        if len(_TABLE_CACHE) > 16:
            _TABLE_CACHE.clear()
        t = GridTables(grid, H, W, const)
        _TABLE_CACHE[key] = t
    return t


def _workspace(device, nbytes):
    key = (str(device), torch.cuda.current_stream(device).cuda_stream)
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.zeros(max(nbytes, 1 << 16), dtype=torch.uint8, device=device)
        _WS_CACHE[key] = ws
    return ws


def keep_map(keep, H, W, device):
    """A per-pixel keep map as the ``*_keep`` kernels read it: uint8 [H, W], contiguous, on ``device``; any nonzero
    byte keeps the pixel.  Accepts a bool or uint8 [H, W] tensor on that device (a bool map is viewed, not copied);
    None stays None (no map: the plain entry points)."""
    if keep is None:
        return None
    if not isinstance(keep, torch.Tensor) or keep.dtype not in (torch.bool, torch.uint8) or tuple(keep.shape) != (H, W):
        raise ValueError("keep must be a bool or uint8 tensor of shape [%d, %d]; got %s" % (
            H, W, "%s %s" % (tuple(keep.shape), keep.dtype) if isinstance(keep, torch.Tensor) else type(keep).__name__))
    if keep.device != torch.device(device):
        raise ValueError("keep is on %s but the maps are on %s" % (keep.device, device))
    if keep.dtype == torch.bool:
        keep = keep.view(torch.uint8)
    return keep.contiguous()


def status_message(st):
    parts = []
    if st & _capi.STATUS_SINGULAR:
        parts.append("singular normal matrix (torch.inverse would raise)")
    if st & _capi.STATUS_NOT_POSDEF:
        parts.append("normal matrix not positive definite (torch.cholesky would raise)")
    if st & _capi.STATUS_NONFINITE:
        parts.append("non-finite moments or coefficients")
    return "weighted least squares: " + "; ".join(parts)


class LsqFunction(torch.autograd.Function):
    """beta, masked = LSQ(o).  o: [B,Lmap,H,W] f32/bf16 raw (or pre-activated) maps, of which the first ``lanes`` (default
    all) are fitted: beta [B, lanes, order+1], masked [B, lanes, H, W], and the gradient of the other maps is zero."""

    @staticmethod
    def forward(ctx, o, tables, order, mask_rows, act, reg_ls, solver, want_masked, status_out, rowp=None, keep=None,
                lanes=None):
        # rowp: a learned warp's (alpha, gamma, y') per row (homography.WarpTables.rowp); the forward then also keeps the
        # row sums and the backward returns dL/drowp.  keep: uint8 [H, W] from keep_map, or None
        _capi.require_cuda(o)
        if order < 0 or order > _capi.MAX_ORDER:
            raise NotImplementedError("Requested order {} for polynomial fit is not implemented".format(order))
        o = o.contiguous()
        B, Lmap, H, W = o.shape
        assert (H, W) == (tables.H, tables.W)
        L = Lmap if lanes is None else lanes
        # a prefix fit: the *_lanes entry points take the maps' channel count after L
        Ls, lsfx = ((L,), "") if L == Lmap else ((L, Lmap), "_lanes")
        n = order + 1
        h = _capi.lib()
        dev = o.device
        beta = torch.empty(B, L, n, dtype=torch.float64, device=dev)
        zinv = torch.empty(B, L, n, n, dtype=torch.float64, device=dev)
        masked = torch.empty(B, L, H, W, dtype=torch.float32, device=dev) if want_masked else None
        status = status_out if status_out is not None else torch.zeros(1, dtype=torch.int32, device=dev)
        nbytes = h.lf_lsq_workspace_bytes(B, L, H, W, order)
        ws = _workspace(dev, nbytes)
        esz = o.element_size()
        rowsums = None
        # with a keep map the *_keep entry points take it right after the tables
        kp = () if keep is None else (_capi.ptr(keep),)
        sfx = "" if keep is None else "_keep"
        per_image = getattr(tables, "per_image", False)
        if per_image:
            # a predicted homography: image b's tables are xtab[b] / yrow[b]; row sums only when rowp needs a gradient
            if rowp is not None and ctx.needs_input_grad[9]:
                rowsums = torch.empty(B, L, H, 3, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _capi.call("lf_lsq_fwd_per_image" + lsfx, _capi.ptr(o), _capi.dtype_id(o), _capi.ptr(tables.xtab),
                           _capi.ptr(tables.yrow), _capi.ptr(keep), B, *Ls, H, W, order, mask_rows, act, float(reg_ls), solver,
                           _capi.ptr(beta), _capi.ptr(zinv), _capi.ptr(masked), _capi.ptr(status), _capi.ptr(rowsums),
                           _capi.ptr(ws), ws.numel(), _capi.stream_ptr(),
                           nbytes=B * L * H * W * (esz + (4 if want_masked else 0)) + 4 * B * H * W)
        elif rowp is not None and ctx.needs_input_grad[9]:
            rowsums = torch.empty(B, L, H, 3, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _capi.call("lf_lsq_fwd_rowsums" + sfx + lsfx, _capi.ptr(o), _capi.dtype_id(o), _capi.ptr(tables.xtab),
                           _capi.ptr(tables.yrow), *kp, B, *Ls, H, W, order, mask_rows, act, float(reg_ls), solver,
                           _capi.ptr(beta), _capi.ptr(zinv), _capi.ptr(masked), _capi.ptr(status), _capi.ptr(rowsums),
                           _capi.ptr(ws), ws.numel(), _capi.stream_ptr(),
                           nbytes=B * L * H * W * (esz + (4 if want_masked else 0)))
        else:
            # the fixed warp, or a learned warp without a gradient (validation, test scoring): no row sums
            with torch.cuda.device(dev):
                _capi.call("lf_lsq_fwd" + sfx + lsfx, _capi.ptr(o), _capi.dtype_id(o), _capi.ptr(tables.xtab),
                           _capi.ptr(tables.ytab), _capi.ptr(tables.yrow), *kp, B, *Ls, H, W, order, mask_rows, act, float(reg_ls), solver,
                           _capi.ptr(beta), _capi.ptr(zinv), _capi.ptr(masked), _capi.ptr(status),
                           _capi.ptr(ws), ws.numel(), _capi.stream_ptr(),
                           nbytes=B * L * H * W * (esz + (4 if want_masked else 0)))
        if status_out is None:
            # same implicit sync + RuntimeError as torch.inverse in the reference
            # (BP/Networks/LSQ_layer.py:114, caught at BP/main.py:289-292)
            st = int(status.item())
            if st:
                raise RuntimeError(status_message(st))
        ctx.save_for_backward(o, beta, zinv, rowsums, keep)
        ctx.tables = tables
        ctx.cfg = (order, mask_rows, act, L)
        if masked is not None:
            ctx.mark_non_differentiable(masked)
            return beta, masked
        return beta, None

    @staticmethod
    def backward(ctx, gbeta, _gmasked):
        o, beta, zinv, rowsums, keep = ctx.saved_tensors
        order, mask_rows, act, L = ctx.cfg
        t = ctx.tables
        B, Lmap, H, W = o.shape
        Ls, lsfx = ((L,), "") if L == Lmap else ((L, Lmap), "_lanes")
        gbeta = gbeta.to(torch.float64).contiguous()
        d_o = torch.empty_like(o)
        if getattr(t, "per_image", False):
            with torch.cuda.device(o.device):
                _capi.call("lf_lsq_bwd_per_image" + lsfx, _capi.ptr(o), _capi.dtype_id(o), _capi.ptr(t.xtab),
                           _capi.ptr(t.yrow), _capi.ptr(keep), B, *Ls, H, W, order, mask_rows, act, _capi.ptr(beta), _capi.ptr(zinv),
                           _capi.ptr(gbeta), _capi.ptr(d_o), _capi.stream_ptr(),
                           nbytes=B * (L + Lmap) * H * W * o.element_size() + 4 * B * H * W)
                g_rowp = None
                if rowsums is not None:
                    g_rowp = torch.empty(B, H, 3, dtype=torch.float64, device=o.device)
                    _capi.call("lf_lsq_grid_grad_per_image", _capi.ptr(rowsums), _capi.ptr(t.yrow), _capi.ptr(beta),
                               _capi.ptr(zinv), _capi.ptr(gbeta), B, L, H, order, mask_rows, _capi.ptr(g_rowp),
                               _capi.stream_ptr())
            return d_o, None, None, None, None, None, None, None, None, g_rowp, None, None
        with torch.cuda.device(o.device):
            _capi.call("lf_lsq_bwd" + ("" if keep is None else "_keep") + lsfx, _capi.ptr(o), _capi.dtype_id(o),
                       _capi.ptr(t.xtab), _capi.ptr(t.ytab), _capi.ptr(t.yrow),
                       *(() if keep is None else (_capi.ptr(keep),)), B, *Ls, H, W, order, mask_rows, act, _capi.ptr(beta), _capi.ptr(zinv),
                       _capi.ptr(gbeta), _capi.ptr(d_o), _capi.stream_ptr(),
                       nbytes=B * (L + Lmap) * H * W * o.element_size())
        g_rowp = None
        if rowsums is not None:
            g_rowp = torch.empty(H, 3, dtype=torch.float64, device=o.device)
            _capi.call("lf_lsq_grid_grad", _capi.ptr(rowsums), _capi.ptr(t.yrow), _capi.ptr(beta), _capi.ptr(zinv),
                       _capi.ptr(gbeta), B, L, H, order, mask_rows, _capi.ptr(g_rowp), _capi.stream_ptr())
        return d_o, None, None, None, None, None, None, None, None, g_rowp, None, None


def check_lanes(lanes, L):
    """The number of lanes to fit of L maps: None means all; otherwise an int in [1, L] (ValueError else)."""
    if lanes is None:
        return None
    if isinstance(lanes, bool) or not isinstance(lanes, int) or not 1 <= lanes <= L:
        raise ValueError("lanes must be an int in [1, %d] (the maps' lane count) or None, got %r" % (L, lanes))
    return lanes


def lsq(o, grid, order, const=255.0, mask_rows=0, act="none", reg_ls=0.0, use_cholesky=False,
        want_masked=False, status_out=None, keep=None, lanes=None):
    """Functional entry: returns (beta [B,L,order+1] f64, masked or None).  keep: optional bool / uint8 [H, W] map
    shared by every image and lane; act(o) is zeroed where it is 0 (masked holds the zeros, d_o is 0 there).
    lanes: fit the first ``lanes`` maps only (default all): beta [B, lanes, order+1], masked [B, lanes, H, W], a zero
    gradient for the other maps, and their systems never reach ``status_out``."""
    B, L, H, W = o.shape
    lanes = check_lanes(lanes, L)
    tables = grid_tables(grid, H, W, const)
    if act not in _capi.ACT_IDS:
        raise NotImplementedError("Activation type: {} is not implemented".format(act))
    solver = _capi.SOLVER_CHOLESKY if use_cholesky else _capi.SOLVER_INVERSE
    return LsqFunction.apply(o, tables, order, mask_rows, _capi.ACT_IDS[act], reg_ls, solver, want_masked,
                             status_out, None, keep_map(keep, H, W, o.device), lanes)


def lsq_warp(o, warp, order, mask_rows=0, act="none", reg_ls=0.0, use_cholesky=False, want_masked=False, status_out=None,
             keep=None, lanes=None):
    """``lsq`` on a learned warp's tables (homography.WarpTables): beta has a gradient with respect to ``warp.rowp``
    as well as ``o``; the row sums behind it cover the kept pixels only.  A per-image warp (``warp.per_image``, a
    predicted homography) fits image b on its own tables and gives rowp [B, R, 3] its per-image gradient.  lanes as in
    ``lsq``."""
    if getattr(warp, "per_image", False) and warp.xtab.shape[0] != o.shape[0]:
        raise ValueError("per-image warp tables for %d images, maps for %d" % (warp.xtab.shape[0], o.shape[0]))
    if act not in _capi.ACT_IDS:
        raise NotImplementedError("Activation type: {} is not implemented".format(act))
    lanes = check_lanes(lanes, o.shape[1])
    solver = _capi.SOLVER_CHOLESKY if use_cholesky else _capi.SOLVER_INVERSE
    return LsqFunction.apply(o, warp, order, mask_rows, _capi.ACT_IDS[act], reg_ls, solver, want_masked, status_out,
                             warp.rowp, keep_map(keep, o.shape[2], o.shape[3], o.device), lanes)
