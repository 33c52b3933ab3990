"""Losses that consume the curve coefficients beta -- host-side mirror of the
reference's ``Loss_crit.py`` (BP/Loss_crit.py; BEV: Birds_Eye_View_Loss/Loss_crit.py).

  define_loss_crit      BP/Loss_crit.py:47-67
  backprojection_loss   :161-218   (float64; supplies dL/dbeta to the fused LSQ backward)
  Area_Loss             :87-143    (closed-form weighted area between curves)
  MSE_Loss              :146-159
  polynomial            Birds_Eye_View_Loss/Loss_crit.py:12-35 (the exact-area metric's trapezium rule, CPU)
  fused_area_loss       Area_Loss over all lanes + the exact-area metric in one launch (lf_area_loss)
The arithmetic here is O(B*56) float64 -- launch-latency, not bandwidth; fusing it into
the LSQ kernels' epilogue/prologue is SURVEY.md 8f rank 1 ("next").
"""
import torch
import torch.nn as nn

if __package__:                        # imported as lanedetection_end2end_b200.Loss_crit
    from .Networks.utils import get_homography
    from . import _capi
else:                                  # imported as top-level `Loss_crit` by the reference's main.py
    from Networks.utils import get_homography
    import _capi


def define_loss_crit(options):
    if options.loss_policy == "mse":
        loss_crit = MSE_Loss(options)
    elif options.loss_policy == "backproject":
        loss_crit = backprojection_loss(options)
    elif options.loss_policy == "area":
        loss_crit = Area_Loss(options.order, options.weight_funct)
    elif options.loss_policy == "homography_mse":
        # referenced but never defined by the reference (BP/Loss_crit.py:56-57 -> NameError)
        raise NameError("name 'Homography_MSE_Loss' is not defined")
    else:
        return NotImplementedError("The requested loss criterion is not implemented")
    weights = torch.Tensor([1] + [options.weight_seg] * options.nclasses)
    if not getattr(options, "no_cuda", False) and torch.cuda.is_available():
        weights = weights.cuda()       # the reference moves them unconditionally (:64); honour --no_cuda on a GPU box
    return loss_crit, CrossEntropyLoss2d(weights)


class _CE2dFunction(torch.autograd.Function):
    """Weighted pixel-wise cross entropy on planar [B,C,H,W] logits: lf_ce2d_fwd / lf_ce2d_bwd (csrc/seg.cu)."""

    @staticmethod
    def forward(ctx, x, target, weight):
        _capi.require_cuda(x, target)
        x = x.contiguous().float()
        target = target.contiguous()
        B, C, H, W = x.shape
        h = _capi.lib()
        scratch = torch.empty(2 * int(h.lf_ce2d_blocks(B, H, W)) + 3, dtype=torch.float64, device=x.device)
        sums, loss = scratch[-3:-1], scratch[-1:]
        _capi.call("lf_ce2d_fwd", _capi.ptr(x), _capi.ptr(target), _capi.ptr(weight), B, C, H, W, _capi.ptr(scratch), _capi.ptr(sums),
                   _capi.ptr(loss), _capi.stream_ptr(), nbytes=4 * x.numel() + 8 * target.numel())
        ctx.save_for_backward(x, target, weight if weight is not None else x.new_empty(0), sums)
        ctx.has_weight = weight is not None
        return loss.reshape(()).float()

    @staticmethod
    def backward(ctx, g):
        x, target, weight, sums = ctx.saved_tensors
        B, C, H, W = x.shape
        dx = torch.empty_like(x)
        _capi.call("lf_ce2d_bwd", _capi.ptr(x), _capi.ptr(target), _capi.ptr(weight if ctx.has_weight else None), B, C, H, W,
                   _capi.ptr(sums), _capi.ptr(g.double().contiguous()), _capi.ptr(dx), _capi.stream_ptr(), nbytes=8 * x.numel())
        return dx, None, None


class CrossEntropyLoss2d(nn.Module):
    """The segmentation criterion `define_loss_crit` returns (nn.CrossEntropyLoss(weights) in the reference,
    BP/Loss_crit.py:64-65; used at BP/main.py:258,307 on the decoder's [B, L+1, H, W] logits and the [B, H, W] label map):
    same value and gradient, one fused kernel each way on CUDA tensors (no log-softmax / nll intermediates)."""

    def __init__(self, weight=None):
        super().__init__()
        self.register_buffer("weight", weight)

    def forward(self, output, target):
        if target.dim() == 4:                       # the loader hands [B,1,H,W] (main.py squeezes it)
            target = target[:, 0]
        w = self.weight
        if w is not None and w.device != output.device:
            w = self.weight = w.to(output.device)
        return _CE2dFunction.apply(output, target.long(), None if w is None else w.float().contiguous())


def seg_proxy_loss(loss_fit, criterion_seg, output_seg, gt, weight):
    """The --seg_proxy joint loss: (loss_fit + weight * ce, ce) with ce = criterion_seg(output_seg, gt), the sum formed in
    float64 in that order, so an eager loop and a graph replay form the same bits.  ``loss_fit`` is the end-to-end loss
    (with --clas, ``loss * weight_fit + (line + horizon) * weight_class``).  Targets outside [0, L] add to neither the
    loss nor the weight sum (lf_ce2d); the reference's nn.CrossEntropyLoss would device-assert on them."""
    ce = criterion_seg(output_seg, gt)
    return loss_fit.double() + weight * ce.double(), ce


def seg_confusion(logits, target, counts, status=None):
    """counts[t * C + pred] += 1 over the pixels of ``logits`` [B, C, H, W] float32 whose ``target`` [B, H, W] int64 t is
    in [0, C); pred is the segmentation branch's argmax (the first maximum wins).  ``counts`` [C * C] int64 is
    accumulated; a nonzero ``status`` (device int32, the LSQ status word) makes the launch count nothing.  One
    capturable launch of lf_seg_confusion (csrc/seg.cu), no synchronisation."""
    _capi.require_cuda(logits, target, counts, status)
    if logits.dtype != torch.float32 or target.dtype != torch.int64 or counts.dtype != torch.int64:
        raise ValueError("seg_confusion takes float32 logits, int64 target and int64 counts, got %s, %s, %s"
                         % (logits.dtype, target.dtype, counts.dtype))
    if target.dim() == 4:                           # the loader hands [B,1,H,W]
        target = target[:, 0]
    B, C, H, W = logits.shape
    if tuple(target.shape) != (B, H, W) or counts.numel() != C * C or not counts.is_contiguous():
        raise ValueError("seg_confusion: target %s and counts of %d for logits %s" % (tuple(target.shape), counts.numel(),
                                                                                      tuple(logits.shape)))
    if status is not None and status.dtype != torch.int32:
        raise ValueError("seg_confusion: the status word is int32, got %s" % status.dtype)
    logits, target = logits.contiguous(), target.contiguous()
    _capi.call("lf_seg_confusion", _capi.ptr(logits), _capi.ptr(target), B, C, H, W, _capi.ptr(status), _capi.ptr(counts),
               _capi.stream_ptr(), nbytes=4 * logits.numel() + 8 * target.numel())
    return counts


def seg_metrics_from_confusion(counts):
    """Pixel accuracy, per-class IoU n_cc / (row_c + col_c - n_cc) (NaN where the denominator is 0) and their mean over
    the classes with a nonzero denominator, from a [C, C] (target, prediction) count matrix on the host."""
    n = torch.as_tensor(counts, dtype=torch.int64).cpu()
    diag, rows, cols = n.diagonal(), n.sum(1), n.sum(0)
    total = int(n.sum())
    den = rows + cols - diag
    iou = [float(d) / float(u) if u else float("nan") for d, u in zip(diag.tolist(), den.tolist())]
    seen = [v for v, u in zip(iou, den.tolist()) if u]
    return {"pixel_acc": float(diag.sum()) / total if total else float("nan"), "iou": iou,
            "miou": sum(seen) / len(seen) if seen else float("nan"), "confusion": n.tolist()}


def _design(y, order):
    return torch.stack([y ** k for k in range(order, 0, -1)] + [torch.ones_like(y)], 1)


class backprojection_loss(nn.Module):
    """Sample the fitted curve at the 56 TuSimple rows in BEV space, project the samples
    back into the image with M^-1 and take the masked mean squared x-error (float64).

    forward(params [B,order+1,1] f64, x_gt [B,56] f64, valid [B,56] f64) -> (loss, x_cal*valid)
    """

    def __init__(self, options):
        super().__init__()
        if options.order > 3:
            raise NotImplementedError(
                "Requested order {} for polynomial fit is not implemented".format(options.order))
        M, M_inv = get_homography(options.resize, options.no_mapping)
        self.M, self.M_inv = torch.from_numpy(M).double(), torch.from_numpy(M_inv).double()
        y_d = (torch.arange(160, 720, 10) - 80).double() / 2.5          # image rows of the h_samples (:173)
        self.y_prime = (self.M[1, 1] * y_d + self.M[1, 2]) / (self.M[2, 1] * y_d + self.M[2, 2])
        self.Y = _design(255 - self.y_prime, options.order)            # [56, order+1]  (:176-188)
        self._dev = None
        # --learn_homography: the warp is the model's (bind), read every call from its last forward
        self.learn_homography = bool(getattr(options, "learn_homography", False))
        self.__dict__["_warp"] = None

    def bind(self, model):
        """Use ``model``'s learned warp (Net.homography, --learn_homography): every call then reads M^-1 and y' of the
        model's last forward, and the loss's gradient reaches the warp.  A criterion built with --learn_homography raises
        until it is bound, so it never silently uses the fixed warp."""
        warp = getattr(model, "homography", None)
        if warp is None:
            raise ValueError("bind() needs a model built with --learn_homography (it has no learned warp)")
        self.__dict__["_warp"] = warp
        return self

    def warp(self):
        """The bound model's current warp (homography.WarpTables), or None with a fixed warp."""
        if not self.learn_homography:
            return None
        w = self.__dict__["_warp"]
        if w is None:
            raise RuntimeError("backprojection_loss was built with --learn_homography: call criterion.bind(model) first")
        if w.current is None:
            raise RuntimeError("backprojection_loss: the bound model has not run a forward yet")
        return w.current

    def _warp_constants(self, device):
        """(M^-1 [3,3], Y [56, n], c_num, c_den) of the bound warp, differentiable (the torch path of forward*)."""
        w = self.warp()
        Mi, yp = w.Minv.view(3, 3), w.yk
        Y = _design(255 - yp, self.Y.shape[1] - 1)
        return Mi, Y, Mi[0, 1] * yp + Mi[0, 2], Mi[2, 1] * yp + Mi[2, 2]

    def _to(self, device):
        if self._dev != device:
            self.M, self.M_inv = self.M.to(device), self.M_inv.to(device)
            self.y_prime, self.Y = self.y_prime.to(device), self.Y.to(device)
            Mi, yp = self.M_inv, self.y_prime
            # the parts of M^-1 [x', y', 1]^T that do not depend on the curve: computed once, not per call
            self._c_num = Mi[0, 1] * yp + Mi[0, 2]
            self._c_den = Mi[2, 1] * yp + Mi[2, 2]
            self._dev = device

    def forward_lanes(self, betas, x_gt, valid_samples, lane_scale=None):
        """``mean_l forward(betas[l], x_gt[:, l], valid[:, l])[0]`` -- the lane loop of BP/main.py:297-305 -- evaluated for
        all lanes at once (same float64 arithmetic per element, a third of the launches).  betas: L tensors
        [B, order+1, 1]; x_gt, valid_samples: [B, >=L, 56].  Returns (loss, x_cal * valid [B, L, 56]).
        lane_scale ([L], optional): per-lane factors, e.g. ddp.lane_valid_scale (batch-global normaliser under data
        parallelism)."""
        L = len(betas)
        self._to(betas[0].device)
        p = torch.stack([b.reshape(b.size(0), -1) for b in betas], 1).double()     # [B, L, n]
        if self.learn_homography:
            Mi, Y, c_num, c_den = self._warp_constants(betas[0].device)
        else:
            Mi, Y, c_num, c_den = self.M_inv, self.Y, self._c_num, self._c_den
        x_prime = p @ Y.t()                                                         # [B, L, 56]
        x_cal = (Mi[0, 0] * x_prime + c_num) / (Mi[2, 0] * x_prime + c_den)
        v = valid_samples[:, :L]
        x_err = (x_gt[:, :L] - x_cal) * v
        nvalid = v.sum(dim=(0, 2))                                                  # per lane, like the per-lane calls
        sq = (x_err ** 2).sum(dim=(0, 2))
        lane = sq / torch.where(nvalid == 0, torch.ones_like(nvalid), nvalid)
        if lane_scale is not None:
            lane = lane * lane_scale.to(lane.dtype)
        return lane.mean(), x_cal * v

    def _fused_host_constants(self):
        """(Y56 [56, n], y' [56], M^-1 [9]) as contiguous float64 numpy arrays for lf_backproj_loss."""
        if self.learn_homography:
            raise RuntimeError("backprojection_loss with --learn_homography reads its warp on the device "
                               "(lf_backproj_loss_dev); the fixed warp's host constants do not describe it")
        # keyed on the identity and in-place version of the tensors it was built from: reassigning or editing
        # M_inv / Y / y_prime (e.g. a finetuned homography) rebuilds the host copies
        key = tuple((id(t), t._version) for t in (self.Y, self.y_prime, self.M_inv))
        c = self.__dict__.get("_fused_consts")
        if c is None or c[0] != key:
            c = self.__dict__["_fused_consts"] = (key, (
                self.Y.detach().cpu().double().contiguous().numpy().copy(),
                self.y_prime.detach().cpu().double().contiguous().numpy().copy(),
                self.M_inv.detach().cpu().double().contiguous().numpy().reshape(-1).copy()))
        return c[1]

    def _fused_ticket(self, device):
        t = self.__dict__.setdefault("_fused_tickets", {})
        if device not in t:
            t[device] = torch.zeros(1, dtype=torch.int32, device=device)
        return t[device]

    def forward(self, params, x_gt, valid_samples):
        self._to(params.device)
        p = params.reshape(params.size(0), -1).double()
        if self.learn_homography:
            Mi, Y, c_num, c_den = self._warp_constants(params.device)
        else:
            Mi, Y, c_num, c_den = self.M_inv, self.Y, self._c_num, self._c_den
        x_prime = p @ Y.t()                                             # [B,56]   (:205)
        num = Mi[0, 0] * x_prime + c_num                                # M^-1 [x', y', 1]^T  (:208-210)
        den = Mi[2, 0] * x_prime + c_den
        x_cal = num / den
        x_err = (x_gt - x_cal) * valid_samples                          # (:214)
        nvalid = valid_samples.sum()
        # loss = sum(err^2) / nvalid, and 0 when nothing is valid (:215-217) -- written without the
        # reference's host-side `if nvalid == 0` so the step has no sync and can live in a CUDA graph
        loss = torch.sum(x_err ** 2) / torch.where(nvalid == 0, torch.ones_like(nvalid), nvalid)
        return loss, x_cal * valid_samples


class _FusedBackprojLoss(torch.autograd.Function):
    """mean over lanes of backprojection_loss, forward + gradient in ONE launch (csrc/loss.cu: lf_backproj_loss)."""

    @staticmethod
    def forward(ctx, beta, x_gt, valid, crit, lane_scale=None):
        import ctypes
        if __package__:
            from . import _capi
        else:
            import _capi
        B, L, n = beta.shape
        dev = beta.device
        lane = torch.empty(L, dtype=torch.float64, device=dev)
        loss = torch.empty(1, dtype=torch.float64, device=dev)
        dbeta = torch.empty_like(beta)
        xcal = torch.empty(B, L, 56, dtype=torch.float64, device=dev)
        ticket = crit._fused_ticket(dev)
        host = crit._fused_host_constants()
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        _capi.call("lf_backproj_loss", host[0].ctypes.data, host[1].ctypes.data, host[2].ctypes.data, p(beta), p(x_gt), p(valid),
                   B, L, n, p(lane), p(loss), p(dbeta), p(xcal), p(ticket), _capi.stream_ptr())
        if lane_scale is not None:      # per-lane factors (ddp.lane_valid_scale): the kernel's outputs are linear in them
            ls = lane_scale.to(torch.float64)
            loss = (lane * ls).mean().reshape(1)
            dbeta = dbeta * ls.view(1, L, 1)
        ctx.save_for_backward(dbeta)
        ctx.mark_non_differentiable(xcal)
        return loss.reshape(()), xcal

    @staticmethod
    def backward(ctx, g, _g_xcal):
        (dbeta,) = ctx.saved_tensors
        return dbeta * g, None, None, None, None


class _FusedBackprojLossWarp(torch.autograd.Function):
    """_FusedBackprojLoss on a learned warp's device constants (lf_backproj_loss_dev): also the gradient with respect to
    M^-1 and y' of the sample rows."""

    @staticmethod
    def forward(ctx, beta, x_gt, valid, Minv, yk, crit, lane_scale=None):
        B, L, n = beta.shape
        dev = beta.device
        lane = torch.empty(L, dtype=torch.float64, device=dev)
        loss = torch.empty(1, dtype=torch.float64, device=dev)
        dbeta = torch.empty_like(beta)
        xcal = torch.empty(B, L, 56, dtype=torch.float64, device=dev)
        g_part = torch.empty(L, 65, dtype=torch.float64, device=dev)
        g_const = torch.empty(65, dtype=torch.float64, device=dev)
        p = _capi.ptr
        _capi.call("lf_backproj_loss_dev", p(yk.detach().contiguous()), p(Minv.detach().contiguous()), p(beta), p(x_gt),
                   p(valid), B, L, n, p(lane), p(loss), p(dbeta), p(xcal), p(g_part), p(g_const), p(crit._fused_ticket(dev)),
                   _capi.stream_ptr())
        if lane_scale is not None:      # the kernel's outputs are linear in per-lane factors
            ls = lane_scale.to(torch.float64)
            loss = (lane * ls).mean().reshape(1)
            dbeta = dbeta * ls.view(1, L, 1)
            g_const = (g_part * ls.view(L, 1)).sum(0)
        ctx.save_for_backward(dbeta, g_const)
        ctx.mark_non_differentiable(xcal)
        return loss.reshape(()), xcal

    @staticmethod
    def backward(ctx, g, _g_xcal):
        dbeta, g_const = ctx.saved_tensors
        return dbeta * g, None, None, g_const[:9] * g, g_const[9:] * g, None, None


def fused_backprojection_loss(crit, betas, x_gt, valid, lane_scale=None):
    """``mean_l crit(betas[l], x_gt[:, l], valid[:, l])[0]`` (what BP/main.py:297-305 computes) in one launch.
    betas: sequence of L tensors [B, order+1, 1] float64 (Net.forward's beta0..3); x_gt, valid: [B, >=L, 56] float64.
    Returns (loss scalar, x_cal*valid [B, L, 56])."""
    L = len(betas)
    beta = torch.stack([b.reshape(b.shape[0], -1) for b in betas], 1).double().contiguous()      # [B, L, n]
    warp = crit.warp() if hasattr(crit, "warp") else None
    if warp is not None:
        return _FusedBackprojLossWarp.apply(beta, x_gt[:, :L].double().contiguous(), valid[:, :L].double().contiguous(),
                                            warp.Minv, warp.yk, crit, lane_scale)
    return _FusedBackprojLoss.apply(beta, x_gt[:, :L].double().contiguous(), valid[:, :L].double().contiguous(), crit, lane_scale)


class Area_Loss(nn.Module):
    """int_0^0.7 W(y) (delta_a y^2 + delta_b y + delta_c)^2 dy with W in {1, 1-y, 1-sqrt(y)},
    averaged over the lanes whose ground-truth parameters are all non-zero (:98-143)."""

    def __init__(self, order, weight_funct):
        super().__init__()
        self.order = order
        self.weight_funct = weight_funct

    def forward(self, params, gt_params, compute=True):
        diff = params.squeeze(-1) - gt_params
        a, b = diff[:, 0], diff[:, 1]
        t = 0.7
        if self.order == 2:
            c = diff[:, 2]
            if self.weight_funct == "none":
                loss_fit = a * a * t ** 5 / 5 + a * b * t ** 4 / 2 + (b * b + 2 * a * c) * t ** 3 / 3 \
                    + b * c * t ** 2 + c * c * t
            elif self.weight_funct == "linear":
                loss_fit = c * c * t - t ** 5 * (2 * a * b / 5 - a * a / 5) + t ** 2 * (b * c - c * c / 2) \
                    - a * a * t ** 6 / 6 - t ** 4 * (b * b / 4 - a * b / 2 + a * c / 2) \
                    + t ** 3 * (b * b / 3 - 2 * c * b / 3 + 2 * a * c / 3)
            elif self.weight_funct == "quadratic":
                loss_fit = t ** 3 * (b * b / 3 + 2 * a * c / 3) - t ** 3.5 * (2 * b * b / 7 + 4 * a * c / 7) \
                    + c * c * t + 0.2 * a * a * t ** 5 - 2 / 11 * a * a * t ** 5.5 - 2 / 3 * c * c * t ** 1.5 \
                    + 0.5 * a * b * t ** 4 - 4 / 9 * a * b * t ** 4.5 + b * c * t ** 2 - 0.8 * b * c * t ** 2.5
            else:
                return NotImplementedError("The requested weight function is not implemented")
        elif self.order == 1:
            loss_fit = b * b * t + a * b * t ** 2 + a * a * t ** 3 / 3
        else:
            return NotImplementedError("The requested order is not implemented")
        present = (gt_params != 0).all(1)        # bool restatement of the .byte() mask (:140-141)
        sel = loss_fit[present]
        return sel.mean(0) if sel.numel() != 0 else 0


class MSE_Loss(nn.Module):
    def __init__(self, options):
        super().__init__()
        self.loss_crit = nn.MSELoss()

    def forward(self, params, gt_params, compute=True):
        return self.loss_crit(params.squeeze(-1), gt_params)


class polynomial:
    """x(y) = a y^2 + b y + c per image, integrated with the trapezium rule (Birds_Eye_View_Loss/Loss_crit.py:12-35).
    ``coeffs``: [B, 3] or [B, 3, 1]; ``trapezoidal(other)`` is the area between the two curves on [a, b] in n steps, in
    the coefficients' dtype -- on float32 CPU tensors the reference's bits (lf_area_loss's exact output restates it)."""

    def __init__(self, coeffs, a=0, b=0.7, n=100):
        self.a1, self.b1, self.c1 = (t.squeeze() for t in torch.chunk(coeffs, 3, 1))
        self.a, self.b, self.n = a, b, n

    def calc_pol(self, x):
        return self.a1 * x ** 2 + self.b1 * x + self.c1

    def trapezoidal(self, other):
        h = float(self.b - self.a) / self.n
        s = 0.0 + abs(self.calc_pol(self.a) / 2.0 - other.calc_pol(other.a) / 2.0)
        for i in range(1, self.n):
            x = self.a + i * h
            s += abs(self.calc_pol(x) - other.calc_pol(x))
        s += abs(self.calc_pol(self.b) / 2.0 - other.calc_pol(self.b) / 2.0)
        return s * h


AREA_WEIGHTS = {"none": 0, "linear": 1, "quadratic": 2}     # lf_area_loss's weight argument


class _FusedAreaLoss(torch.autograd.Function):
    """sum over lanes of Area_Loss (order 2) and the exact-area batch mean, ONE launch (csrc/loss.cu: lf_area_loss)."""

    @staticmethod
    def forward(ctx, beta, params, weight, exact):
        _capi.require_cuda(beta, params)
        B, L, _ = beta.shape
        out = torch.empty(2 + B * L * 3, dtype=torch.float32, device=beta.device)
        loss, exact_mean, dbeta = out[0:1], out[1:2], out[2:].view(B, L, 3)
        p = _capi.ptr
        _capi.call("lf_area_loss", p(beta), p(params), B, L, weight, p(loss), p(dbeta), None, p(exact_mean) if exact else None,
                   _capi.stream_ptr())
        ctx.save_for_backward(dbeta)
        ctx.mark_non_differentiable(exact_mean)
        return loss.reshape(()), exact_mean.reshape(())

    @staticmethod
    def backward(ctx, g, _g_exact):
        (dbeta,) = ctx.saved_tensors
        return dbeta * g, None, None, None


def fused_area_loss(betas, params, weight_funct, exact=False):
    """``sum_l Area_Loss(2, weight_funct)(betas[l], params[:, l])`` -- BEV/main.py:223,237 -- and, with ``exact``, the
    exact-area metric ``((trap_left + trap_right) / 2).mean()`` of BEV/main.py:273-280, in one launch on the device.
    betas: sequence of L (2 or 4) float32 tensors [B, 3, 1] (Net.forward's beta0..3); params: the loader's [B, 4, 3].
    Returns (loss, exact_mean or None), float32 0-d tensors; only the loss has a gradient.

    The loss sums float64 terms in a fixed order and rounds once, so it is the reference's value to float32 rounding (not
    its float32 bits).  A lane that no image has contributes 0, also when none has any lane (where Area_Loss returns the
    Python 0).  The 4-lane masks of main.py:226-234 multiply by 1 exactly the images Area_Loss selects, so they change
    neither the value nor the gradient and are not applied.  The per-image metric is the reference's float32 bits; the
    mean differs from torch's .mean() by summation order only."""
    if weight_funct not in AREA_WEIGHTS:
        raise ValueError("unknown weight_funct %r (none, linear or quadratic)" % (weight_funct,))
    if len(betas) not in (2, 4):
        raise ValueError("fused_area_loss takes 2 or 4 lanes, got %d" % len(betas))
    B = params.shape[0]
    for b in betas:
        if b.numel() != B * 3:
            raise ValueError("order 2 only: every beta must be [B, 3, 1], got %s" % (tuple(b.shape),))
    if tuple(params.shape) != (B, 4, 3):
        raise ValueError("params must be [B, 4, 3], got %s" % (tuple(params.shape),))
    beta = torch.stack([b.reshape(B, 3) for b in betas], 1).float().contiguous()
    loss, exact_mean = _FusedAreaLoss.apply(beta, params.float().contiguous(), AREA_WEIGHTS[weight_funct], bool(exact))
    return loss, (exact_mean if exact else None)
