"""Host-side mirror of the reference's ``Networks/LSQ_layer.py`` (BP variant; the BEV
variant is ``LSQ_layer_bev.py``): same public names, constructor arguments, forward
signatures, return arities/dtypes and error behaviour, with the device work done by
the fused sm_90a kernels in csrc/lsq.cu through the C ABI.

  activation_layer        BP/Networks/LSQ_layer.py:27-47
  ProjectiveGridGenerator :50-68
  Weighted_least_squares  :72-154
  Classification          :157-207   (SURVEY.md 8f-2: on the library's kernels through ops_heads.py)
  Net                     :210-315
  trapezium_keep          :236-246 (the column / corner masks the reference builds and leaves unused)
"""
from math import ceil

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from ._pkg import submodule
from .utils import get_homography

_ops = submodule("ops_lsq")
_capi = submodule("_capi")
_ops_net = submodule("ops_net")


def square_tensor(x):
    return x ** 2


def return_tensor(x):
    return x


class _Activation:
    """Callable with the semantics of the reference's activation objects; carries the
    name so ``Net`` can hand the activation to the fused kernel instead of running it."""

    def __init__(self, kind):
        self.kind = kind

    def __call__(self, x):
        k = self.kind
        if k == "square":
            return x ** 2
        if k == "abs":
            return torch.abs(x)
        if k == "relu":
            return F.relu(x)
        if k == "sigmoid":
            return torch.sigmoid(x)
        if k == "softplus":
            return F.softplus(x)
        return x

    def cuda(self):
        return self


def activation_layer(activation="square", no_cuda=False):
    if activation not in _capi.ACT_IDS:
        raise NotImplementedError("Activation type: {} is not implemented".format(activation))
    return _Activation(activation)


def ProjectiveGridGenerator(size, theta, no_cuda):
    """grid [N, H*W, 2]: pixel (x, y, 1) mapped through ``theta`` [N,3,3] and perspective-
    divided.  Built for one image with the same fp32 torch ops as the reference (so the
    values are the reference's) and expanded (not copied) over the batch."""
    N, C, H, W = size
    t0 = theta[0:1].detach().cpu()
    ys, xs = torch.meshgrid(torch.linspace(0, H - 1, H), torch.linspace(0, W - 1, W), indexing="ij")
    base = torch.stack((xs, ys, torch.ones_like(xs)), dim=-1).to(t0.dtype).view(1, H * W, 3)
    g = torch.bmm(base, t0.transpose(1, 2))
    g = torch.div(g[:, :, 0:2], g[:, :, 2:])
    if not no_cuda:
        g = g.cuda()
    return g.expand(N, H * W, 2)


def trapezium_keep(resize, zero_rows):
    """--trapezium_mask: keep [resize, 2*resize] uint8, 0 on the rows < zero_rows, on the columns idx_col1 / idx_col2
    and where idx_mask is nonzero, 1 elsewhere.  idx_col1 / idx_col2 / idx_mask are built with the reference
    constructor's own expressions (BP/Networks/LSQ_layer.py:236-246, Birds_Eye_View_Loss/...:257-266), including the
    truncation of linspace(1, 13, 14).long() to [1, 1, 2, .., 13]."""
    n_row = 13
    idx_col1 = torch.linspace(1, n_row, n_row + 1).long()
    idx_col2 = torch.linspace(0, n_row, n_row + 1).long() + 2 * resize - (n_row + 1)
    idx_mask = (np.arange(resize)[:, None] < np.arange(2 * resize) - (resize + 10)) * 1
    idx_mask = np.flip(idx_mask, 1).copy() + idx_mask
    keep = torch.ones(resize, 2 * resize, dtype=torch.uint8)
    keep[:zero_rows] = 0
    keep[:, idx_col1] = 0
    keep[:, idx_col2] = 0
    keep[torch.from_numpy(idx_mask) != 0] = 0
    return keep


class Weighted_least_squares(nn.Module):
    """beta_k = argmin sum_p (W_k,p (x_p - phi(y_p)^T beta))^2 per image and lane.

    forward(W, grid) -> (beta0, beta1, beta2, beta3), each [B, order+1, 1] float64,
    beta2/beta3 None unless nclasses > 3 (reference :130-154).  ``W`` is the activated,
    masked map; the weight enters squared exactly as in the reference (:111-115).
    Extensions beyond the reference API: ``forward_all`` returns the stacked
    [B, L, order+1] tensor for any L and order <= 4 (BASELINE config 5).
    """

    def __init__(self, size, nclasses, order, no_cuda, reg_ls=0, use_cholesky=False, y_const=255.0,
                 out_dtype=torch.float64):
        super().__init__()
        N, C, self.H, W = size
        self.W = W
        self.nclasses = nclasses
        self.order = order
        self.reg_ls_value = float(reg_ls)
        self.reg_ls = reg_ls * torch.eye(order + 1)          # plain attribute like the reference (:79)
        self.use_cholesky = use_cholesky
        self.y_const = y_const          # the reference hard-codes 255 (:94) whatever --resize is
        self.out_dtype = out_dtype

    def forward_all(self, W, grid, mask_rows=0, act="none", want_masked=False, status_out=None, max_order=4, keep=None,
                    lanes=None):
        """keep: optional bool / uint8 [H, W] map; act(W) is zeroed where it is 0 before the fit (ops_lsq.lsq).
        lanes: fit the first ``lanes`` maps only (default all; ops_lsq.lsq)."""
        if self.order > max_order:
            raise NotImplementedError(
                "Requested order {} for polynomial fit is not implemented".format(self.order))
        Wm = W.reshape(-1, self.nclasses, self.H, self.W)
        beta, masked = _ops.lsq(Wm, grid, self.order, self.y_const, mask_rows, act, self.reg_ls_value,
                                self.use_cholesky, want_masked, status_out, keep, lanes)
        return beta, masked

    def _split(self, beta):
        b = beta.to(self.out_dtype).unsqueeze(-1)            # [B, L, d+1, 1]; fewer lanes after a prefix fit
        K = b.shape[1]
        beta0, beta1 = b[:, 0], b[:, 1] if K > 1 else None
        beta2 = beta3 = None
        if self.nclasses > 3:
            beta2, beta3 = (b[:, 2] if K > 2 else None), (b[:, 3] if K > 3 else None)
        return beta0, beta1, beta2, beta3

    def forward(self, W, grid):
        beta, _ = self.forward_all(W, grid, max_order=3)     # order > 3 raises like :105-107
        return self._split(beta)


class Classification(nn.Module):
    """Line-type / horizon heads on the encoder output (BP/Networks/LSQ_layer.py:157-207; SURVEY.md 8f rank 2).
    The torch modules below only hold the parameters / buffers under the reference's names (``--clas 1`` checkpoints
    round-trip); ``forward`` runs every stage on the library's kernels through ``ops_heads`` (tensor-core gather-GEMM
    convolutions, the ERFNet BatchNorm kernels with eps 1e-5, max / row-mean pooling, HBM-bound fully connected
    layers) -- forward and backward, no torch operator on a feature map."""

    def __init__(self, class_type, size, channels_in, resize):
        super().__init__()
        self.class_type = class_type
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
        self.avgpool = nn.AvgPool2d((1, cols))
        self.maxpool = nn.MaxPool2d((2, 2), stride=2)
        if class_type == "line":
            self.fully_connected1 = nn.Linear(64 * rows * cols // 4, 128)
            self.fully_connected_line1 = nn.Linear(128, 4)
        else:
            self.fully_connected_horizon = nn.Linear(64 * rows, resize)

    def stages(self, x):
        """The four conv -> BatchNorm -> ReLU stages on the encoder map x: NHWC [B, rows, cols, 64]."""
        _heads, _net = submodule("ops_heads"), _ops_net
        from .ERFNet import _track
        h = _net.as_nhwc(x)
        _capi.require_cuda(h)
        if tuple(h.shape[1:3]) != self.size:
            raise ValueError("Classification head built for a %dx%d encoder map, got %dx%d" % (self.size + tuple(h.shape[1:3])))
        for conv, bn in ((self.conv1, self.conv1_bn), (self.conv2, self.conv2_bn),
                         (self.conv3, self.conv3_bn), (self.conv4, self.conv4_bn)):
            h = _heads.conv_bn_relu(h, conv, bn, self.training, _track)
        return h

    def forward(self, x):
        _heads = submodule("ops_heads")
        h = self.stages(x)
        if self.class_type == "line":
            f = _heads.MaxPool2FlatFunction.apply(h)
            f = _heads.LinearFunction.apply(f, self.fully_connected1.weight, self.fully_connected1.bias, True)
            return _heads.LinearFunction.apply(f, self.fully_connected_line1.weight, self.fully_connected_line1.bias, False)
        f = _heads.RowMeanFlatFunction.apply(h)
        return _heads.LinearFunction.apply(f, self.fully_connected_horizon.weight, self.fully_connected_horizon.bias, False)


class Net(nn.Module):
    """ERFNet -> activation -> row mask -> weighted least squares (reference :210-315).

    forward(input, gt_line, end_to_end, early_return=False, gt=None) ->
        (beta0, beta1, beta2, beta3, masked, output, line, horizon, output_seg)
    A singular / non-finite normal matrix raises RuntimeError (main.py:289-292 skips the
    batch).  Set ``self.defer_status_check = True`` to skip the per-step host sync; the
    OR-ed status word is then left in ``self.lsq_status`` (device int32) for the caller.
    ``self.fit_lanes = K`` makes a training forward end to end fit lanes [0, K) only (beta_K .. beta3 are None, masked
    has K maps, the other systems never reach the status word); eval forwards fit every lane.
    """

    def __init__(self, args):
        super().__init__()
        from . import define_model
        self.nclasses = args.nclasses
        resize = args.resize
        size = torch.Size([args.batch_size, args.nclasses, resize, 2 * resize])
        M, _ = get_homography(resize, args.no_mapping)
        M = torch.from_numpy(M).unsqueeze_(0).expand([args.batch_size, 3, 3]).float()

        # --seg_proxy: the decoder's second branch (net.decoder.layers1, the reference's dormant `do_segmentation`
        # decoder) on the shared encoder, trained with a cross-entropy proxy term next to the fit (engine.train_epoch);
        # its logits [B, L + 1, H, W] are output_seg.  A checkpoint without the branch loads with strict=False, the
        # branch then keeps its define_init_weights start.
        self.seg_proxy = bool(getattr(args, "seg_proxy", False))
        if self.seg_proxy and not args.end_to_end:
            raise ValueError("--seg_proxy needs --end_to_end True: the segmentation branch already trains the decoder "
                             "output with cross-entropy")
        if self.seg_proxy and args.pretrained:
            raise ValueError("--seg_proxy cannot be combined with --pretrained: its phases change the trained parameter "
                             "sets")
        out_channels = args.nclasses + int(not args.end_to_end)
        kw = {"do_segmentation": True} if self.seg_proxy else {}
        self.net = define_model(mod=args.mod, layers=args.layers, in_channels=args.channels_in,
                                out_channels=out_channels, pretrained=args.pretrained, pool=args.pool, **kw)
        self.activation = activation_layer(args.activation_layer, args.no_cuda)
        self.grid = ProjectiveGridGenerator(size, M, args.no_cuda)
        self.ls_layer = Weighted_least_squares(size, args.nclasses, args.order, args.no_cuda,
                                               args.reg_ls, args.use_cholesky)
        self.zero_rows = ceil(resize * args.mask_percentage)
        self.idx_row = torch.linspace(0, self.zero_rows - 1, self.zero_rows).long()

        self.end_to_end = args.end_to_end
        self.pretrained = args.pretrained
        self.classification_branch = args.clas
        if self.classification_branch:
            self.line_classification = Classification("line", size=(32, 64), channels_in=128, resize=resize)
            self.horizon_estimation = Classification("horizon", size=(32, 64), channels_in=128, resize=resize)
            # the heads' conv weights are re-packed by the ERFNet module's one-launch weight packer (plain dict entry:
            # not a second registration of the submodules)
            self.net.__dict__["_pack_extra"] = (self.line_classification, self.horizon_estimation)
        # --learn_homography: the warp is a parameter (homography.LearnedHomography, state_dict key
        # homography.offsets) whose tables are built on the device every forward; a fixed-warp checkpoint loads with
        # strict=False and starts the fine-tuning from the fixed warp (offsets = 0)
        self.learn_homography = bool(getattr(args, "learn_homography", False))
        if self.learn_homography:
            if args.no_mapping:
                raise ValueError("--learn_homography learns the bird's-eye-view warp; it cannot be combined with --no_mapping")
            if getattr(args, "loss_policy", "backproject") != "backproject":
                raise ValueError("--learn_homography needs --loss_policy backproject (the loss that sees the warp), got %r"
                                 % (args.loss_policy,))
            self.homography = submodule("homography").LearnedHomography(resize, self.zero_rows)
        # --predict_homography: one warp per image from the spatial-transformer branch on the encoder map (the
        # reference's DLT module, state_dict keys DLT.spatial_trans.*); a checkpoint without the branch loads with
        # strict=False and starts from the fixed warp (fully_connected2 = 0)
        self.predict_homography = bool(getattr(args, "predict_homography", False))
        # --predict_homography_corners source: the branch predicts --learn_homography's five source-corner offsets per
        # image (the reference's destination corners give the loss nothing to learn from: NOTES.md); a destination-mode
        # checkpoint loads with DLT.spatial_trans.fully_connected2.* dropped and strict=False
        corners = getattr(args, "predict_homography_corners", "destination")
        if corners != "destination" and not self.predict_homography:
            raise ValueError("--predict_homography_corners %s needs --predict_homography True" % corners)
        if self.predict_homography:
            if self.learn_homography:
                raise ValueError("--predict_homography cannot be combined with --learn_homography: pick one warp model")
            if args.no_mapping:
                raise ValueError("--predict_homography predicts the bird's-eye-view warp; it cannot be combined with "
                                 "--no_mapping")
            if getattr(args, "loss_policy", "backproject") != "backproject":
                raise ValueError("--predict_homography needs --loss_policy backproject (the loss that sees the warp), got "
                                 "%r" % (args.loss_policy,))
            if not args.end_to_end or args.pretrained:
                raise ValueError("--predict_homography needs --end_to_end True and no --pretrained: the branch is trained "
                                 "by the fit's loss only")
            if resize % 4:
                # the per-image least-squares kernels are the row-separable ones only, whose 16-byte loads need
                # 2 * resize to be a multiple of 8 (bf16 maps)
                raise ValueError("--predict_homography needs --resize a multiple of 4, got %d" % resize)
            self.DLT = submodule("homography").PredictedHomography(resize, self.zero_rows, size=(32, 64), channels_in=128,
                                                                   corners=corners)
            self.net.__dict__["_pack_extra"] = tuple(self.net.__dict__.get("_pack_extra", ())) + (self.DLT,)
        # --trapezium_mask: the per-pixel keep map of the end-to-end fit (NOTES.md "Trapezium mask"); a plain attribute
        # like idx_row, not a buffer, so checkpoints stay the reference's
        self.keep = trapezium_keep(resize, self.zero_rows) if getattr(args, "trapezium_mask", False) else None
        if not args.no_cuda:
            self.idx_row = self.idx_row.cuda()
            if self.keep is not None:
                self.keep = self.keep.cuda()
        self.defer_status_check = False
        self.lsq_status = None
        # a lane curriculum (engine.train_epoch, --lane_curriculum): a training forward end to end fits lanes
        # [0, fit_lanes) only and returns None for the other betas; None fits every lane, and so does every eval forward
        self.fit_lanes = None

    def forward(self, input, gt_line, end_to_end, early_return=False, gt=None):
        line, horizon = None, None
        shared_encoder, output, output_seg = self.net(input, end_to_end * self.pretrained)
        if early_return:
            return output

        status = None
        if self.defer_status_check:
            if self.lsq_status is None or self.lsq_status.device != output.device:
                self.lsq_status = torch.zeros(1, dtype=torch.int32, device=output.device)
            status = self.lsq_status
        warp = None
        if self.learn_homography:
            st = status if status is not None else torch.zeros(1, dtype=torch.int32, device=output.device)
            warp = self.homography(st)
        elif self.predict_homography:
            st = status if status is not None else torch.zeros(1, dtype=torch.int32, device=output.device)
            warp = self.DLT(shared_encoder, st)
        grid = self.grid
        if grid.device != output.device:
            grid = self.grid = grid.to(output.device)
        grid = grid[:output.size(0)]
        keep = self.keep
        if keep is not None and keep.device != output.device:
            keep = self.keep = keep.to(output.device)

        if not end_to_end:
            # segmentation pre-training branch (:279-293): argmax -> per-lane label maps,
            # detached; fitted without gradient
            nl = 2 if self.nclasses < 3 else 4
            _capi.require_cuda(output)
            # argmax + per-lane label maps + row mask + the gt_line substitution of :308-311 in one launch
            # (csrc/seg.cu: lf_seg_lane_maps_line), with no host read of a device gt_line
            od = output.detach().contiguous().float()
            B = od.shape[0]
            masked = torch.empty(B, nl, od.shape[2], od.shape[3], dtype=torch.float32, device=od.device)
            gl = gt_line
            if not gl.is_cuda and not bool(gl.ne(0).any()):             # a host gt_line is checked on the host
                gl = None
            if gl is not None and tuple(gl.shape) != (B, nl):
                # not one flag per map: the reference broadcasts its mask when gt_line is nonzero, and raises where it
                # cannot (4 line flags for 2 lanes); this needs the host read the [B, nl] case avoids
                gl = gl[:, :, None, None].expand_as(masked)[:, :, 0, 0] if gl.sum() != 0 else None
            if gl is not None:
                gl = gl.to(od.device, torch.float32, non_blocking=True).contiguous()
            _capi.call("lf_seg_lane_maps_line", _capi.ptr(od), B, od.shape[1], od.shape[2], od.shape[3], nl,
                       self.zero_rows, _capi.ptr(gl), _capi.ptr(masked), _capi.stream_ptr())
            with torch.no_grad():
                if warp is not None:
                    beta, _ = self._lsq_warp(masked, warp, 0, "none", False, st, status is None)
                else:
                    beta, _ = self.ls_layer.forward_all(masked, grid, status_out=status, max_order=3)
        else:
            if self.classification_branch:
                line = self.line_classification(shared_encoder)
                horizon = self.horizon_estimation(shared_encoder)
            # activation (:295) + row mask (:301) [+ the trapezium keep map] + least squares (:314) in one launch;
            # `masked` is materialised only because the API returns it (:315)
            lanes = self.fit_lanes if self.training else None
            if warp is not None:
                beta, masked = self._lsq_warp(output, warp, self.zero_rows, self.activation.kind, True, st, status is None,
                                              keep, lanes)
            else:
                beta, masked = self.ls_layer.forward_all(output, grid, mask_rows=self.zero_rows,
                                                         act=self.activation.kind, want_masked=True,
                                                         status_out=status, max_order=3, keep=keep, lanes=lanes)
        beta0, beta1, beta2, beta3 = self.ls_layer._split(beta)
        return beta0, beta1, beta2, beta3, masked, output, line, horizon, output_seg

    def _lsq_warp(self, W, warp, mask_rows, act, want_masked, status, check, keep=None, lanes=None):
        ls = self.ls_layer
        if ls.order > 3:
            raise NotImplementedError("Requested order {} for polynomial fit is not implemented".format(ls.order))
        Wm = W.reshape(-1, ls.nclasses, ls.H, ls.W)
        beta, masked = _ops.lsq_warp(Wm, warp, ls.order, mask_rows, act, ls.reg_ls_value, ls.use_cholesky, want_masked,
                                     status, keep, lanes)
        if check:
            # the status word holds the warp's guard as well as the solve's: one host read, as torch.inverse's raise
            st = int(status.item())
            if st:
                raise RuntimeError(_ops.status_message(st))
        return beta, masked
