#!/usr/bin/env python
"""Diagnostic (GPU): non_bottleneck_1d(128, dil) at 32x64 in tf32x3 and fp32 modes vs the fp64 oracle: per-parameter gradient
errors, ReLU-flip counts, and the x3-vs-fp32 difference; plus the 3xTF32 weight gradient (ops_net.wgrad3) alone on the
block's own (t3, d4) operands."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import inputs, erfnet_oracle as eo          # noqa: E402
from lanedetection_end2end_b200 import ops_net as o     # noqa: E402
from lanedetection_end2end_b200.Networks import ERFNet  # noqa: E402
import test_net_gpu as T                                # noqa: E402

for (C, dil, H, W, drop) in [(128, 16, 32, 64, True), (128, 16, 32, 64, False), (128, 4, 32, 64, True), (128, 8, 32, 64, True)]:
    P_np = {k[4:]: v for k, v in inputs.make_erfnet_params(3, 2, seed=6).items()}
    prefix = "encoder.layers.7"
    N = 3
    keep = (torch.rand(N, C, generator=torch.Generator().manual_seed(2)) >= 0.3).float() / 0.7 if drop else None
    x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(3))
    P = T.oracle_params(prefix, P_np)
    x64 = x.double().requires_grad_(True)
    gy = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(0))
    yo = eo.non_bottleneck_1d(x64, P, prefix, dil, True, keep.double() if drop else None)
    yo.backward(gy.double())
    grads = {}
    for mode in ("fp32", "tf32x3"):
        o.set_conv_mode(mode)
        blk = ERFNet.non_bottleneck_1d(C, 0.3 if drop else 0.0, dil).cuda().train()
        T.load_params(blk, {k: v.float() for k, v in P.items()}, prefix)
        blk.drop_mask_override = keep
        xg = x.cuda().requires_grad_(True)
        y = blk(xg)
        y.backward(gy.cuda())
        torch.cuda.synchronize()
        d = (xg.grad.double().cpu() - x64.grad).abs()
        sc = float(x64.grad.abs().max())
        rep = {"mode": mode, "C": C, "dil": dil, "drop": drop, "y_err": T.rel(y, yo), "dx_bad_entries": int((d > 1e-4 * sc).sum()),
               "dx_median": float(d.median() / sc)}
        for n, p in blk.named_parameters():
            ref = P[prefix + "." + n].grad
            rep["g/" + n] = float((p.grad.double().cpu() - ref).abs().max() / max(float(ref.abs().max()), 1e-30))
        grads[mode] = {n: p.grad.clone() for n, p in blk.named_parameters()}
        print(json.dumps(rep), flush=True)
    print(json.dumps({"x3_vs_fp32": {n: float((grads["tf32x3"][n] - grads["fp32"][n]).abs().max() / grads["fp32"][n].abs().max().clamp_min(1e-30))
                                     for n in grads["fp32"]}}), flush=True)

# operand level: wgrad x3 vs fp32 vs fp64, vertical d = 16 / 8 on post-ReLU-like operands
import torch.nn.functional as F                          # noqa: E402
for (N, C, H, W, vertical, dil) in [(3, 128, 32, 64, True, 16), (3, 128, 32, 64, True, 8), (3, 128, 32, 64, False, 8)]:
    g = torch.Generator().manual_seed(1)
    xx = torch.randn(N, H, W, C, generator=g).clamp_min(0).cuda()
    dy = (torch.randn(N, H, W, C, generator=g) * (torch.rand(N, H, W, C, generator=g) > 0.5)).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = torch.zeros(C, C, kh, kw, device="cuda")
    res = {}
    for mode in ("fp32", "tf32x3"):
        o.set_conv_mode(mode)
        res[mode] = o.wgrad3(xx, dy, w, vertical, dil)[0]
        torch.cuda.synchronize()
    wd = torch.zeros(C, C, kh, kw, dtype=torch.float64, requires_grad=True)
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    F.conv2d(xx.double().cpu().permute(0, 3, 1, 2), wd, None, 1, pad, dl).backward(dy.double().cpu().permute(0, 3, 1, 2))
    sc = float(wd.grad.abs().max())
    print(json.dumps({"wgrad": [N, C, H, W, vertical, dil], "x3_err": float((res["tf32x3"].double().cpu() - wd.grad).abs().max()) / sc,
                      "fp32_err": float((res["fp32"].double().cpu() - wd.grad).abs().max()) / sc}), flush=True)
