"""Image side of the reference's loader on the GPU (SURVEY.md 8f-3): what BP/Dataloader/Load_Data_new.py:127-131,
166-167,178-181 does per image with PIL on a DataLoader worker -- crop the bottom 640 rows, BILINEAR resize to
(resize, 2*resize), optional horizontal flip, ToTensor().float() -- as one launch over a batch of decoded frames.

    pre = FramePreprocessor(resize=256)                       # tables for 1280x720 TuSimple frames
    x = pre(frames_u8)                                        # [N,720,1280,3] uint8 cuda -> [N,3,256,512] float32
    x = pre(frames_u8, flip=mask, layout="nhwc4")             # or straight into the stem convolution's layout

The output is bit-identical to the reference's loader (Pillow's fixed-point resample is reproduced, csrc/input_pipe.cu).
LabelPreprocessor does the same for the ground-truth label map (:129,131,160-184): crop, NEAREST resize, class rules, flip.

    gt = LabelPreprocessor(256, nclasses=4)(maps_u8, flip=mask)   # [N,720,1280] uint8 cuda -> [N,1,256,512] int64

Decoding is outside this module (jpeg.JpegDecoder and png.PngDecoder deliver the frames and maps).  Dataloader/Load_Data_new.py
joins the decoders, these tables and the lane labels of the loader (lane coordinates / 2.5, valid-point mask, horizon
vector, line types; :133-160) into a loader with a device cache (csrc/loader.cu)."""
import math

import numpy as np
import torch

from . import _capi

PRECISION_BITS = 32 - 8 - 2      # Pillow: 8 bits of pixel, 2 bits of headroom in a 32-bit accumulator


def resample_tables(in_size, out_size):
    """Per-axis tables of Pillow's ImagingResample for the BILINEAR (triangle, support 1) filter over [0, in_size):
    bounds int32 [out_size][2] (first source index, number of taps) and integer coefficients int32 [out_size][ksize]
    (Resample.c precompute_coeffs / normalize_coeffs_8bpc; float64 arithmetic in the same order as the C code)."""
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    inv = 1.0 / filterscale
    one = float(1 << PRECISION_BITS)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [0.0] * xmax
        ww = 0.0
        for x in range(xmax):
            t = abs((x + xmin - center + 0.5) * inv)
            w[x] = 1.0 - t if t < 1.0 else 0.0
            ww += w[x]
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(v * one - 0.5) if v < 0 else int(v * one + 0.5)
        bounds[xx] = (xmin, xmax)
    return bounds, kk


class FramePreprocessor:
    def __init__(self, resize, frame_hw=(720, 1280), crop_rows=640, device="cuda"):
        self.resize, self.frame_hw, self.crop_rows = int(resize), tuple(frame_hw), int(crop_rows)
        H, W = self.frame_hw
        if self.crop_rows > H:
            raise ValueError("crop_rows %d exceeds the frame height %d" % (self.crop_rows, H))
        self.Ho, self.Wo = self.resize, 2 * self.resize
        xb, xk = resample_tables(W, self.Wo)
        yb, yk = resample_tables(self.crop_rows, self.Ho)
        dev = torch.device(device)
        self.tables = [torch.from_numpy(t).to(dev).contiguous() for t in (xb, xk, yb, yk)]
        self.kx, self.ky = xk.shape[1], yk.shape[1]

    def __call__(self, frames, flip=None, layout="nchw"):
        _capi.require_cuda(frames)
        H, W = self.frame_hw
        if frames.dtype != torch.uint8 or frames.dim() != 4 or tuple(frames.shape[1:]) != (H, W, 3):
            raise ValueError("expected uint8 frames [N,%d,%d,3], got %s %s" % (H, W, frames.dtype, tuple(frames.shape)))
        frames = frames.contiguous()
        N = frames.shape[0]
        if layout == "nchw":
            out, lay = torch.empty(N, 3, self.Ho, self.Wo, dtype=torch.float32, device=frames.device), 0
        elif layout == "nhwc4":
            out, lay = torch.empty(N, self.Ho, self.Wo, 4, dtype=torch.float32, device=frames.device), 1
        else:
            raise ValueError(layout)
        fl = None
        if flip is not None:
            fl = torch.as_tensor(flip, device=frames.device).to(torch.uint8).contiguous()
            if fl.numel() != N:
                raise ValueError("flip must have one entry per frame")
        xb, xk, yb, yk = self.tables
        _capi.call("lf_frame_preprocess", _capi.ptr(frames), N, H, W, H - self.crop_rows, self.crop_rows, _capi.ptr(xb), _capi.ptr(xk),
                   self.kx, _capi.ptr(yb), _capi.ptr(yk), self.ky, self.Ho, self.Wo, _capi.ptr(fl), lay, _capi.ptr(out),
                   _capi.stream_ptr(), nbytes=N * self.crop_rows * W * 3 + out.numel() * 4)
        return out


def nearest_table(in_size, out_size):
    """Source index of every output index of Pillow's NEAREST resize over [0, in_size) (Geometry.c ImagingScaleAffine:
    the position starts at half a step and adds the step in float64, truncated per pixel).  This differs from
    floor((o + 0.5) * in / out) for many sizes, where the accumulated sum lands just below an integer."""
    step = in_size / out_size
    pos = step * 0.5
    idx = np.empty(out_size, np.int32)
    for o in range(out_size):
        idx[o] = int(pos)
        pos += step
    if idx.min() < 0 or idx.max() >= in_size:
        raise ValueError("NEAREST resize %d -> %d leaves the source" % (in_size, out_size))
    return idx


class LabelPreprocessor:
    """The loader's label map on the device (Load_Data_new.py:129,131,160-184): crop the bottom `crop_rows` rows, Pillow
    NEAREST resize to (resize, 2*resize), nclasses < 3 turns classes 3 and 4 into 0, an optional horizontal flip mirrors
    the map and swaps classes 1 and 2, and the result is the int64 [N,1,resize,2*resize] of (ToTensor(gt)*255).long().

    The flip reproduces a quirk of the reference: its masks of classes 3 and 4 are taken BEFORE the flip and applied
    after it, so in a flipped sample every pixel where the unflipped map held 3 (4) becomes 4 (3), at the unflipped
    position.  With nclasses < 3 a flipped sample therefore carries labels 3 and 4 again (the 2D cross-entropy ignores
    targets outside its classes).  `flip` follows FramePreprocessor(flip=): one entry per image, so one mask drives both."""

    def __init__(self, resize, nclasses, frame_hw=(720, 1280), crop_rows=640, device="cuda"):
        self.resize, self.nclasses, self.frame_hw, self.crop_rows = int(resize), int(nclasses), tuple(frame_hw), int(crop_rows)
        H, W = self.frame_hw
        if self.crop_rows > H or self.crop_rows < 1 or self.resize < 1:
            raise ValueError("crop_rows %d / resize %d do not fit the frame height %d" % (self.crop_rows, self.resize, H))
        self.Ho, self.Wo = self.resize, 2 * self.resize
        dev = torch.device(device)
        self.xs = torch.from_numpy(nearest_table(W, self.Wo)).to(dev)
        self.ys = torch.from_numpy(nearest_table(self.crop_rows, self.Ho)).to(dev)

    def __call__(self, maps, flip=None):
        _capi.require_cuda(maps)
        H, W = self.frame_hw
        if maps.dtype != torch.uint8 or maps.dim() != 3 or tuple(maps.shape[1:]) != (H, W):
            raise ValueError("expected uint8 maps [N,%d,%d], got %s %s" % (H, W, maps.dtype, tuple(maps.shape)))
        maps = maps.contiguous()
        N = maps.shape[0]
        out = torch.empty(N, 1, self.Ho, self.Wo, dtype=torch.int64, device=maps.device)
        fl = None
        if flip is not None:
            fl = torch.as_tensor(flip, device=maps.device).to(torch.uint8).contiguous()
            if fl.numel() != N:
                raise ValueError("flip must have one entry per map")
        _capi.call("lf_label_preprocess", _capi.ptr(maps), N, H, W, H - self.crop_rows, _capi.ptr(self.xs), _capi.ptr(self.ys),
                   self.Ho, self.Wo, self.nclasses, _capi.ptr(fl), _capi.ptr(out), _capi.stream_ptr(),
                   nbytes=N * self.Ho * self.Wo * (2 + 8))
        return out
