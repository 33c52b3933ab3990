#!/usr/bin/env python
"""Per-kernel timing of one non_bottleneck_1d block (forward + backward) at the bench shapes, in fp32 (CUDA-core)
and tf32 (tensor-core) conv modes.  CUDA events around every C-ABI launch (the _capi.TRACE hook)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lanedetection_end2end_b200 import _capi, ops_net  # noqa: E402
from lanedetection_end2end_b200.Networks import ERFNet  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--modes", nargs="+", default=["fp32", "tf32"])
    ap.add_argument("--shapes", nargs="+", default=["128,32,64,2", "64,64,128,1"])   # C,H,W,dil
    ap.add_argument("--variant", type=int, default=2, help="tensor-core conv variant (2 = halo slab, 1 = per-tap boxes)")
    a = ap.parse_args()
    _capi.lib().lf_conv1d_tc_set_variant(a.variant)
    for shp in a.shapes:
        C, H, W, dil = [int(v) for v in shp.split(",")]
        torch.manual_seed(0)
        blk = ERFNet.non_bottleneck_1d(C, 0.3, dil).cuda().train()
        x = torch.randn(a.batch, H, W, C, device="cuda").permute(0, 3, 1, 2)
        gy = torch.randn(a.batch, H, W, C, device="cuda").permute(0, 3, 1, 2)
        for mode in a.modes:
            ops_net.set_conv_mode(mode)
            for _ in range(2):
                xi = x.detach().requires_grad_(True)
                blk(xi).backward(gy)
            torch.cuda.synchronize()
            _capi.TRACE = []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                xi = x.detach().requires_grad_(True)
                blk(xi).backward(gy)
            e1.record()
            torch.cuda.synchronize()
            trace, _capi.TRACE = _capi.TRACE, None
            agg = {}
            for name, s, e, flops, nbytes in trace:
                d = agg.setdefault(name, {"n": 0, "ms": 0.0, "flops": 0, "bytes": 0})
                d["n"] += 1
                d["ms"] += s.elapsed_time(e)
                d["flops"] += flops
                d["bytes"] += nbytes
            out = {"bench": "nb1d_block", "C": C, "H": H, "W": W, "dil": dil, "batch": a.batch, "mode": mode, "tc_variant": a.variant,
                   "ms_per_iter_traced": e0.elapsed_time(e1) / a.iters, "kernels": {}}
            for k, d in sorted(agg.items(), key=lambda kv: -kv[1]["ms"]):
                ms = d["ms"] / a.iters
                out["kernels"][k] = {"launches": d["n"] // a.iters, "ms": round(ms, 4),
                                     "TFLOPs": round(d["flops"] / a.iters / ms / 1e9, 2) if d["flops"] else None,
                                     "GBps": round(d["bytes"] / a.iters / ms / 1e6, 1) if d["bytes"] else None}
            print(json.dumps(out), flush=True)
        ops_net.set_conv_mode("fp32")


if __name__ == "__main__":
    main()
