#!/usr/bin/env python
"""Inference throughput per convolution mode: the eval forward (BatchNorm folded, ops_eval.py) under torch.no_grad(),
256x512, replayed as one CUDA graph (engine.GraphedInference) in tf32x3, bf16 and fp8 mode.  The three modes' graphs are
captured from three copies of one randomly initialised model and replayed alternately, three rounds, in one process.
Configs: 2 (batch 32, 2 lanes, order 2) and 3 (batch 64, 4 lanes, order 3).  Then, at batch 32, the CUDA-event time of
every 3-tap convolution launch (lf_conv1d_tc_bf16 / lf_conv1d_tc_fp8) of one eager forward, grouped by layer shape.

Writes one JSON record (default profiles/h100/bench_infer_fp8.json) with the card's name, power limit and max SM clock
read in the same run, and prints it."""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lanedetection_end2end_b200 import _capi, ops_net                 # noqa: E402
from lanedetection_end2end_b200.engine import GraphedInference        # noqa: E402
from lanedetection_end2end_b200.Networks.LSQ_layer import Net         # noqa: E402
from lanedetection_end2end_b200.Networks.utils import define_args     # noqa: E402

MODES = ("tf32x3", "bf16", "fp8")
CONFIGS = {"config2": (32, 2, 2), "config3": (64, 4, 3)}   # batch, lanes, order


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name()}


def model_for(batch, lanes, order):
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(lanes), "--order", str(order),
                                     "--batch_size", str(batch)])
    torch.manual_seed(0)
    m = Net(args).cuda().eval()
    m.defer_status_check = True
    return m


def time_graphs(base, x, iters, rounds):
    graphs = {}
    for mode in MODES:                       # one model copy per mode: each keeps its own cached operands alive
        ops_net.set_conv_mode(mode)
        graphs[mode] = GraphedInference(copy.deepcopy(base), x)
    ms = {m: [] for m in MODES}
    for _ in range(rounds):
        for mode, gi in graphs.items():
            for _ in range(3):
                gi.graph.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                gi.graph.replay()
            e1.record()
            torch.cuda.synchronize()
            ms[mode].append(e0.elapsed_time(e1) / iters)
    return ms


# the 68 3-tap convolutions of one forward, in launch order: 5 C = 64 encoder blocks, 8 C = 128 (dilated) encoder blocks,
# 2 C = 64 decoder blocks, 2 C = 16 decoder blocks (super-pixel view), 4 launches each
GROUPS = [("C=64 encoder, 64x128", 20), ("C=128 encoder, 32x64, d in {1,2,4,8,16}", 32), ("C=64 decoder, 64x128", 8),
          ("C=16 decoder, 128x256 (super-pixel view, C=64 at 128x64)", 8)]


def group_of(i):
    for name, n in GROUPS:
        if i < n:
            return name
        i -= n
    raise ValueError(i)


def kernel_times(base, x, reps):
    """{mode: {layer group: [ms of each launch]}} of the 3-tap convolutions of `reps` eager forwards."""
    out = {}
    for mode, entry in (("bf16", "lf_conv1d_tc_bf16"), ("fp8", "lf_conv1d_tc_fp8")):
        ops_net.set_conv_mode(mode)
        m = copy.deepcopy(base)
        with torch.no_grad():
            for _ in range(2):
                m(x, torch.zeros(x.shape[0], 4), True)
            torch.cuda.synchronize()
            _capi.TRACE = []
            try:
                for _ in range(reps):
                    m(x, torch.zeros(x.shape[0], 4), True)
                torch.cuda.synchronize()
                tr = [e0.elapsed_time(e1) for name, e0, e1, _, _ in _capi.TRACE if name == entry]
            finally:
                _capi.TRACE = None
        per = len(tr) // reps
        assert per == sum(n for _, n in GROUPS), per
        d = {}
        for i, t in enumerate(tr):
            d.setdefault(group_of(i % per), []).append(t)
        out[mode] = d
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_infer_fp8.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer_modes.py needs a CUDA device")
    rec = {"card": card(), "workload": "eval forward (BatchNorm folded) + LSQ, 256x512, one CUDA-graph replay per forward",
           "configs": {}}
    kt = None
    for cname, (batch, lanes, order) in CONFIGS.items():
        base = model_for(batch, lanes, order)
        x = torch.rand(batch, 3, 256, 512, device="cuda")
        ms = time_graphs(base, x, a.iters, a.rounds)
        rec["configs"][cname] = {
            "batch": batch, "lanes": lanes, "order": order,
            "modes": {m: {"ms_per_forward_rounds": v, "ms_per_forward": min(v), "images_per_s": batch / min(v) * 1e3}
                      for m, v in ms.items()}}
        print(json.dumps({cname: rec["configs"][cname]}), flush=True)
        if cname == "config2":
            kt = kernel_times(base, x, 3)
        del base
        torch.cuda.empty_cache()
    rows = []
    for g, _ in GROUPS:
        b = sorted(kt["bf16"][g])[len(kt["bf16"][g]) // 2]
        q = sorted(kt["fp8"][g])[len(kt["fp8"][g]) // 2]
        rows.append({"layers": g, "launches_per_forward": len(kt["bf16"][g]) // 3, "gflop_per_launch": 6.442450944,
                     "bf16_ms_median": b, "fp8_ms_median": q, "speedup": b / q})
    rec["per_kernel_batch32"] = {
        "note": "CUDA events around each 3-tap convolution launch of 3 eager eval forwards, median per layer group "
                "(every launch is 2 * 32 * H * W * 3 * C^2 = 6.44 GFLOP)",
        "rows": rows,
        "total_bf16_ms": sum(sum(v) for v in kt["bf16"].values()) / 3,
        "total_fp8_ms": sum(sum(v) for v in kt["fp8"].values()) / 3}
    ops_net.set_conv_mode("tf32x3")
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(rec, fh, indent=1)
    print(json.dumps(rec["per_kernel_batch32"]), flush=True)


if __name__ == "__main__":
    main()
