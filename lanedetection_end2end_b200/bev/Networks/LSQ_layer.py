"""Birds_Eye_View_Loss/Networks/LSQ_layer.py mirror.

Differences from the BP variant (all served by the same fused kernel, csrc/lsq.cu):
  * normalised image coordinates in [0,1) and a fixed normalised homography (reference :17-32, :66-87);
    the grid is rebuilt by ``project_layer(M)`` every forward (:324);
  * ``y = 1 - y'`` (:109), orders 0..2 only (:110-118), beta returned as float32 (:167);
  * ``Net.forward(input, end_to_end)`` -> (beta0, beta1, beta2, beta3, masked, M, output, line, horizon) (:326).
"""
from math import ceil

import numpy as np
import torch
import torch.nn as nn

from ._pkg import bp

_L = bp("LSQ_layer")
_U = bp("utils")
activation_layer = _L.activation_layer
square_tensor = _L.square_tensor
return_tensor = _L.return_tensor


def Init_Projective_transform(nclasses, batch_size, resize):
    """Normalised trapezoid -> band homography and its inverse, float32, expanded over the batch."""
    size = torch.Size([batch_size, nclasses, resize, 2 * resize])
    top, bottom = 0.3, 1
    src = np.float32([[0.45, top], [0.55, top], [0.1, bottom], [0.9, bottom]])
    dst = np.float32([[0.45, top], [0.55, top], [0.45, bottom], [0.55, bottom]])
    M = torch.from_numpy(_U._perspective_transform(src, dst)).unsqueeze_(0).expand([batch_size, 3, 3]).float()
    M_inv = torch.from_numpy(_U._perspective_transform(dst, src)).unsqueeze_(0).expand([batch_size, 3, 3]).float()
    return size, M, M_inv


class ProjectiveGridGenerator(nn.Module):
    """grid = perspective-divided (x, y, 1) @ theta^T over normalised pixel centres (reference :66-87)."""

    def __init__(self, size, theta, no_cuda):
        super().__init__()
        self.N, self.C, self.H, self.W = size
        ys, xs = torch.meshgrid(torch.linspace(0, 1 - 1 / self.H, self.H), torch.linspace(0, 1 - 1 / self.W, self.W),
                                indexing="ij")
        self.base_grid = torch.stack((xs, ys, torch.ones_like(xs)), dim=-1).view(1, self.H * self.W, 3)
        if not no_cuda:
            self.base_grid = self.base_grid.cuda()
        self._cache = None

    def forward(self, theta):
        key = (theta.data_ptr(), theta._version, str(theta.device))
        if self._cache is None or self._cache[0] != key:
            base = self.base_grid.to(theta.device)
            g = torch.bmm(base, theta[0:1].transpose(1, 2))
            g = torch.div(g[:, :, 0:2], g[:, :, 2:])
            self._cache = (key, g.expand(theta.size(0), self.H * self.W, 2))
        return self._cache[1]


class Weighted_least_squares(_L.Weighted_least_squares):
    def __init__(self, size, nclasses, order, no_cuda, reg_ls=0, use_cholesky=False):
        super().__init__(size, nclasses, order, no_cuda, reg_ls, use_cholesky, y_const=1.0, out_dtype=torch.float32)

    def forward(self, W, grid):
        beta, _ = self.forward_all(W, grid, max_order=2)      # order > 2 raises like reference :117-118
        return self._split(beta)


Classification = _L.Classification


class Net(nn.Module):
    takes_gt_line = False           # forward(input, end_to_end): engine.model_forward calls it without the BP gt_line

    def __init__(self, args):
        super().__init__()
        from . import define_model
        if getattr(args, "seg_proxy", False):
            raise ValueError("--seg_proxy is not supported by the bird's-eye-view Net: its ERFNet has no second decoder")
        resize = args.resize
        size, M, _ = Init_Projective_transform(args.nclasses, args.batch_size, args.resize)
        self.M = M
        self.nclasses = args.nclasses
        out_channels = args.nclasses + int(not args.end_to_end)
        self.net = define_model(mod=args.mod, layers=args.layers, in_channels=args.channels_in,
                                out_channels=out_channels, pretrained=args.pretrained, pool=args.pool)
        self.activation = activation_layer(args.activation_layer, args.no_cuda)
        self.project_layer = ProjectiveGridGenerator(size, M, args.no_cuda)
        self.ls_layer = Weighted_least_squares(size, args.nclasses, args.order, args.no_cuda, args.reg_ls,
                                               args.use_cholesky)
        self.zero_rows = ceil(resize * args.mask_percentage)
        self.idx_row = torch.linspace(0, self.zero_rows - 1, self.zero_rows).long()
        self.end_to_end = args.end_to_end
        self.pretrained = args.pretrained
        self.classification_branch = args.clas
        if not args.no_cuda:
            self.M = self.M.cuda()
            self.idx_row = self.idx_row.cuda()
        self.defer_status_check = False
        self.lsq_status = None

    def forward(self, input, end_to_end):
        line, horizon = None, None
        shared_encoder, output = self.net(input, end_to_end * self.pretrained)
        if self.M.device != output.device:
            self.M = self.M.to(output.device)
        grid = self.project_layer(self.M)[:output.size(0)]
        status = None
        if self.defer_status_check:
            if self.lsq_status is None or self.lsq_status.device != output.device:
                self.lsq_status = torch.zeros(1, dtype=torch.int32, device=output.device)
            status = self.lsq_status
        if not end_to_end:
            labels = torch.max(output.detach(), 1)[1].float()
            activated = torch.stack([labels * (labels == (k + 1)).float() for k in range(2)], 1)
            masked = activated.index_fill(2, self.idx_row.to(output.device), 0)
            with torch.no_grad():
                beta, _ = self.ls_layer.forward_all(masked, grid, status_out=status, max_order=2)
        else:
            beta, masked = self.ls_layer.forward_all(output, grid, mask_rows=self.zero_rows, act=self.activation.kind,
                                                     want_masked=True, status_out=status, max_order=2)
        beta0, beta1, beta2, beta3 = self.ls_layer._split(beta)
        return beta0, beta1, beta2, beta3, masked, self.M, output, line, horizon
