"""Host-side mirror of the reference's ``Networks/ERFNet.py`` (BP/Networks/ERFNet.py:11-176):
same class names, constructor arguments, sub-module / parameter names (so ``state_dict``s
and ``define_init_weights`` work unchanged) and forward signatures.  The ``nn.Conv2d`` /
``nn.BatchNorm2d`` / ``nn.ConvTranspose2d`` children are PARAMETER CONTAINERS only -- their
own forward is never called; every block runs as one autograd Function over the sm_90a
kernels (ops_net.py).  Feature maps travel between blocks as NHWC memory viewed with the
reference's NCHW shape (channels_last), so chaining blocks costs no layout change.
A BatchNorm container converted by ``torch.nn.SyncBatchNorm.convert_sync_batchnorm`` makes its block normalise with the
statistics of every rank of its ``process_group`` in training mode (ops_net.BNSync); eval mode is unchanged.
"""
import torch
import torch.nn as nn

from ._pkg import submodule

import os

_ops = submodule("ops_net")
_eval = submodule("ops_eval")
# eval-mode inference with every BatchNorm folded into the convolution weights (ops_eval.py); LANEFIT_EVAL_FUSED=0 keeps
# the unfused eval path (the training kernels with running statistics)
EVAL_FUSED = os.environ.get("LANEFIT_EVAL_FUSED", "1") != "0"


_PENDING_COUNTERS = None      # when a list: BatchNorm step counters to bump with ONE fused launch


def _track(bn, training):
    """nn.BatchNorm2d bookkeeping (num_batches_tracked += 1 per training forward).  Inside ``Net.forward``
    the 41 counters are collected and incremented by a single ``torch._foreach_add_`` instead of 41 launches."""
    if training and bn.track_running_stats and bn.num_batches_tracked is not None:
        if _PENDING_COUNTERS is not None:
            _PENDING_COUNTERS.append(bn.num_batches_tracked)
        else:
            bn.num_batches_tracked += 1


# ---------------------------------------------------------------------------------------------
# parameter containers: layer specs -> torch modules (names / shapes / registration order fixed by the
# reference's checkpoints; the modules' own forward() is never used)
# ---------------------------------------------------------------------------------------------
_BN_EPS = 1e-3


def _conv(cin, cout, kernel, stride=1, pad=0, dil=1):
    return nn.Conv2d(cin, cout, kernel, stride=stride, padding=pad, dilation=dil, bias=True)


def _batchnorm(c):
    return nn.BatchNorm2d(c, eps=_BN_EPS)


def _factorised_specs(d):
    """(attribute, kernel, padding, dilation) of the four 1-D convolutions of a residual block with dilation d."""
    return (("conv3x1_1", (3, 1), (1, 0), (1, 1)), ("conv1x3_1", (1, 3), (0, 1), (1, 1)),
            ("conv3x1_2", (3, 1), (d, 0), (d, 1)), ("conv1x3_2", (1, 3), (0, d), (1, d)))


# (kind, *args) per stage; "down"/"up": (cin, cout), "res": (channels, dropout p, dilation)
_ENCODER_STAGES = ([("down", 16, 64)] + [("res", 64, 0.03, 1)] * 5 + [("down", 64, 128)]
                   + [("res", 128, 0.3, d) for _ in range(2) for d in (2, 4, 8, 16)])
_DECODER_STAGES = [("up", 128, 64), ("res", 64, 0, 1), ("res", 64, 0, 1), ("up", 64, 16), ("res", 16, 0, 1), ("res", 16, 0, 1)]


def _build_stage(spec):
    kind, args = spec[0], spec[1:]
    return {"down": DownsamplerBlock, "up": UpsamplerBlock, "res": non_bottleneck_1d}[kind](*args)


class DownsamplerBlock(nn.Module):
    """relu(bn(cat[conv3x3 stride 2 (x), maxpool2x2 (x)]))  (reference :11-22)."""

    def __init__(self, ninput, noutput):
        super().__init__()
        self.ninput = ninput
        self.conv = _conv(ninput, noutput - ninput, 3, stride=2, pad=1)   # the other `ninput` channels come from the pool
        self.pool = nn.MaxPool2d(2, stride=2)
        self.bn = _batchnorm(noutput)

    def forward(self, input):
        need_dx = input.requires_grad and torch.is_grad_enabled()
        if self.ninput % 4 != 0:
            if need_dx:
                raise NotImplementedError("input gradient of a DownsamplerBlock with %d input channels" % self.ninput)
            x = _ops.image_to_nhwc_pad(input, (self.ninput + 3) // 4 * 4)
        else:
            x = _ops.as_nhwc(input)
        if _ops.fp8_mode():
            _ops.require_inference_mode(self.training, x, self.conv.weight)
        if not self.training and x.is_cuda and EVAL_FUSED and _eval.inference_only(x, self.conv.weight):
            y = _eval.down(x, self)
            if y is not None:
                return _ops.as_nchw_view(y)
        y = _ops.DownFunction.apply(x, self.ninput, self.conv.weight, self.conv.bias, self.bn.weight, self.bn.bias,
                                    self.bn.running_mean, self.bn.running_var, self.training, need_dx,
                                    _ops.bn_sync(self.bn, self.training))
        _track(self.bn, self.training)
        return _ops.as_nchw_view(y)


class non_bottleneck_1d(nn.Module):
    """Factorised residual block: 3x1 -> relu -> 1x3 -> bn -> relu -> 3x1(d) -> relu -> 1x3(d) -> bn ->
    dropout2d -> (+x) -> relu  (reference :25-60)."""

    def __init__(self, chann, dropprob, dilated):
        super().__init__()
        self.dilated = dilated
        specs = _factorised_specs(dilated)
        for k, (attr, kernel, pad, dil) in enumerate(specs):
            setattr(self, attr, _conv(chann, chann, kernel, pad=pad, dil=dil))
            if k % 2 == 1:                                   # a BatchNorm after each (3x1, 1x3) pair: bn1, bn2
                setattr(self, "bn%d" % (k // 2 + 1), _batchnorm(chann))
        self.dropout = nn.Dropout2d(dropprob)
        self.drop_mask_override = None      # tests inject a fixed [N,C] mask here

    def _drop_mask(self, x):
        if self.drop_mask_override is not None:
            return self.drop_mask_override.to(device=x.device, dtype=torch.float32).contiguous()
        pending = self.__dict__.pop("_pending_drop_mask", None)      # drawn for the whole net by fused_dropout_masks()
        if pending is not None and self.training and pending.shape[0] == x.shape[0] and pending.device == x.device:
            return pending
        p = self.dropout.p
        if not self.training or p == 0:
            return None
        N, _, _, C = x.shape
        keep = (torch.rand(N, C, device=x.device) >= p).float()      # Dropout2d: whole channels (:41,57-58)
        return (keep / (1.0 - p)).contiguous()

    def forward(self, input):
        x = _ops.as_nhwc(input)
        if _ops.fp8_mode():             # fp8: the folded eval path below or an error (Nb1dFunction refuses the mode)
            _ops.require_inference_mode(self.training, x, self.conv3x1_1.weight)
        if not self.training and x.is_cuda and EVAL_FUSED and _eval.inference_only(x, self.conv3x1_1.weight):
            y = _eval.nb1d(x, self)                  # BatchNorm folded into the weights: 4 conv launches, nothing else
            if y is not None:
                return _ops.as_nchw_view(y)
        y = _ops.Nb1dFunction.apply(
            x, self.conv3x1_1.weight, self.conv3x1_1.bias, self.conv1x3_1.weight, self.conv1x3_1.bias,
            self.bn1.weight, self.bn1.bias, self.conv3x1_2.weight, self.conv3x1_2.bias,
            self.conv1x3_2.weight, self.conv1x3_2.bias, self.bn2.weight, self.bn2.bias,
            self.bn1.running_mean, self.bn1.running_var, self.bn2.running_mean, self.bn2.running_var,
            self.dilated, self._drop_mask(x), self.training, _ops.bn_sync(self.bn1, self.training),
            _ops.bn_sync(self.bn2, self.training))
        _track(self.bn1, self.training)
        _track(self.bn2, self.training)
        return _ops.as_nchw_view(y)


_DROP_PLANS = {}
_FUSE_DROPOUT = True


def fused_dropout_masks(blocks, batch, device):
    """Dropout2d channel masks ([batch, C] each, values 0 or 1/(1-p)) for all `blocks` from ONE uniform draw:
    3 launches per step instead of ~4 per block (13 encoder blocks use dropout).  Each block receives a contiguous
    slice of the flat result through ``_pending_drop_mask``."""
    spec = tuple((b.conv3x1_1.out_channels, float(b.dropout.p)) for b in blocks)
    key = (spec, batch, str(device))
    plan = _DROP_PLANS.get(key)
    if plan is None:
        thr = torch.cat([torch.full((batch * c,), p) for c, p in spec])
        scale = torch.cat([torch.full((batch * c,), 1.0 / (1.0 - p)) for c, p in spec])
        plan = _DROP_PLANS[key] = (thr.to(device), scale.to(device))
    thr, scale = plan
    u = torch.rand(thr.numel(), device=device)
    flat = (u >= thr).to(torch.float32) * scale
    off = 0
    masks = []
    for (c, _), b in zip(spec, blocks):
        m = flat[off:off + batch * c].view(batch, c)
        off += batch * c
        b.__dict__["_pending_drop_mask"] = m
        masks.append(m)
    return masks


class Encoder(nn.Module):
    def __init__(self, in_channels, num_classes):
        super().__init__()
        self.initial_block = DownsamplerBlock(in_channels, 16)
        self.layers = nn.ModuleList(_build_stage(spec) for spec in _ENCODER_STAGES)
        # only used in encoder-only mode (reference :84,92-93); a 1x1 conv on 128 channels
        self.output_conv = _conv(128, num_classes, 1)

    def forward(self, input, predict=False):
        feat = self.initial_block(input)
        for stage in self.layers:
            feat = stage(feat)
        if not predict:
            return feat
        # encoder-only pretraining head: not on the end-to-end hot path (SURVEY.md 2)
        return torch.nn.functional.conv2d(feat, self.output_conv.weight, self.output_conv.bias)


class UpsamplerBlock(nn.Module):
    """relu(bn(convT3x3 stride 2 (x)))  (reference :98-107)."""

    def __init__(self, ninput, noutput):
        super().__init__()
        self.conv = nn.ConvTranspose2d(ninput, noutput, 3, stride=2, padding=1, output_padding=1, bias=True)
        self.bn = _batchnorm(noutput)

    def forward(self, input):
        x = _ops.as_nhwc(input)
        if _ops.fp8_mode():
            _ops.require_inference_mode(self.training, x, self.conv.weight)
        if not self.training and x.is_cuda and EVAL_FUSED and _eval.inference_only(x, self.conv.weight):
            y = _eval.up(x, self)
            if y is not None:
                return _ops.as_nchw_view(y)
        y = _ops.UpFunction.apply(x, self.conv.weight, self.conv.bias, self.bn.weight, self.bn.bias,
                                  self.bn.running_mean, self.bn.running_var, self.training,
                                  _ops.bn_sync(self.bn, self.training))
        _track(self.bn, self.training)
        return _ops.as_nchw_view(y)


class _OutputConvT(nn.ConvTranspose2d):
    """ConvTranspose2d(16 -> L, 2, stride 2) emitting planar NCHW maps (reference :124,152)."""

    def forward(self, input):
        return _ops.OutConvFunction.apply(_ops.as_nhwc(input), self.weight, self.bias)


class Decoder(nn.Module):
    def __init__(self, num_classes, pretrain, do_segmentation=False):
        super().__init__()
        def head(n_out):                 # 2x2 stride-2 transposed conv from the 16-channel decoder features
            return _OutputConvT(16, n_out, 2, stride=2, padding=0, output_padding=0, bias=True)

        self.pretrain = pretrain
        self.layers = nn.ModuleList(_build_stage(spec) for spec in _DECODER_STAGES)
        self.output_conv = head(num_classes)
        if pretrain:
            self.output_conv2 = head(num_classes + 1)
        self.do_segmentation = do_segmentation
        if do_segmentation:              # second decoder for the segmentation branch (same stages + its own head)
            self.layers1 = nn.ModuleList([_build_stage(spec) for spec in _DECODER_STAGES] + [head(num_classes + 1)])

    def forward(self, input, flag):
        feat = input
        for stage in self.layers:
            feat = stage(feat)
        head = self.output_conv2 if (self.pretrain and not flag) else self.output_conv
        seg = input
        if self.do_segmentation:
            for stage in self.layers1:
                seg = stage(seg)
        return head(feat), seg


class Net(nn.Module):
    """ERFNet.  forward(input, flag, only_encode=False) -> (encoder_output, decoder_output, output_seg)
    (reference :164-176; the BEV variant returns the first two only, see ERFNet_bev).
    ``do_segmentation=True`` builds the decoder's second branch (``decoder.layers1``: the decoder's six stages and a
    16 -> out_channels + 1 head on the shared encoder output), whose logits are then ``output_seg``; without it
    ``output_seg`` is the encoder output, as in the reference, which never passes the flag."""

    def __init__(self, layers=18, in_channels=1, out_channels=1, pretrained=False, pool=False, do_segmentation=False):
        super().__init__()
        self.encoder = Encoder(in_channels, out_channels)
        self.decoder = Decoder(out_channels, pretrained, do_segmentation=do_segmentation)

    def forward(self, input, flag, only_encode=False):
        global _PENDING_COUNTERS
        if _ops.fp8_mode():             # inference-only mode: refuse a training or autograd forward before any launch
            _ops.require_inference_mode(self.training, input, *self.parameters())
        if only_encode:
            return self.encoder.forward(input, predict=True)
        _PENDING_COUNTERS = []
        if input.is_cuda:
            # one launch re-packs every layer's GEMM-layout weight operand from the current parameters
            packs = self.__dict__.get("_weight_packs")
            if packs is None:
                packs = self.__dict__["_weight_packs"] = _ops.WeightPackCache(self)
            packs.refresh()
            _ops.ACTIVE_PACKS = packs
        global _FUSE_DROPOUT
        if _FUSE_DROPOUT and self.training and input.is_cuda:
            drops = [m for m in self.modules() if isinstance(m, non_bottleneck_1d) and m.dropout.p > 0
                     and m.drop_mask_override is None]
            if drops:
                try:
                    fused_dropout_masks(drops, input.shape[0], input.device)
                except Exception:                      # pragma: no cover -- the blocks then draw their own masks
                    _FUSE_DROPOUT = False
                    for m in drops:
                        m.__dict__.pop("_pending_drop_mask", None)
        try:
            encoder_output = self.encoder(input)
            decoder_output, output_seg = self.decoder.forward(encoder_output, flag)
        finally:
            pending, _PENDING_COUNTERS = _PENDING_COUNTERS, None
            if pending:
                torch._foreach_add_(pending, 1)
        return encoder_output, decoder_output, output_seg
