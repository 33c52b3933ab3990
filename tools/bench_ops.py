#!/usr/bin/env python
"""Per-shape timing of the 3-tap convolution / input-gradient / weight-gradient kernels in every conv mode.

    python tools/bench_ops.py [--batch 32] [--modes tf32x3 tf32 bf16] > ops.jsonl

One JSON line per (mode, op, shape): mean launch time over `--iters` back-to-back launches on tensors larger than L2 in
aggregate (each op cycles through `--rot` independent input sets), CUDA events on the launching stream.  In bf16 mode the
"bf16 ..." ops read (and the forward writes) the bf16 activations non_bottleneck_1d stores in that mode."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

SHAPES = [  # C, H, W, vertical, dil   (per 256x512 image)
    (64, 64, 128, True, 1), (64, 64, 128, False, 1),
    (128, 32, 64, True, 1), (128, 32, 64, False, 1), (128, 32, 64, True, 2), (128, 32, 64, False, 4),
    (128, 32, 64, True, 8), (128, 32, 64, False, 8), (128, 32, 64, True, 16), (128, 32, 64, False, 16),
    (16, 128, 256, True, 1), (16, 128, 256, False, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rot", type=int, default=4)
    ap.add_argument("--modes", nargs="+", default=["tf32x3", "tf32"])
    a = ap.parse_args()
    from lanedetection_end2end_b200 import ops_net as o
    dev = torch.device("cuda")
    for C, H, W, vertical, dil in SHAPES:
        N = a.batch
        xs = [torch.randn(N, H, W, C, device=dev) for _ in range(a.rot)]
        xh = [t.bfloat16() for t in xs]
        gs = [torch.randn(N, H, W, C, device=dev) for _ in range(a.rot)]
        kh, kw = (3, 1) if vertical else (1, 3)
        w = torch.randn(C, C, kh, kw, device=dev) / (3 * C) ** 0.5
        b = torch.randn(C, device=dev)
        for mode in a.modes:
            o.set_conv_mode(mode)
            # weight operands are packed outside the timed region (in the model one lf_pack_gather launch per step does it)
            def taps(sgn):
                return [((sgn * (k - 1) * dil, 0) if vertical else (0, sgn * (k - 1) * dil)) for k in range(3)]
            if C == 16:
                wf, wd = o.pack_tc_super(w, vertical, False), o.pack_tc_super(w, vertical, True)
                tf, td = [((k - 1, 0) if vertical else (0, k - 1)) for k in range(3)], [((1 - k, 0) if vertical else (0, 1 - k)) for k in range(3)]
                view = lambda t: t.view(N, H, W // 4, 64)
                bb = b.repeat(4)
            else:
                wf, wd, tf, td, view, bb = o.pack_tc_fwd(w), o.pack_tc_dgrad(w), taps(1), taps(-1), (lambda t: t), b
            wf, wd = o.tc_operand(wf), o.tc_operand(wd)   # tf32x3: the TF32 hi / lo pair; bf16: bf16 operands
            outs = [torch.empty_like(view(xs[0])) for _ in range(a.rot)]
            outh = [torch.empty_like(view(xh[0])) for _ in range(a.rot)]
            # op -> (launch, bytes per element of the activation-sized operands it moves)
            ops = {
                "fwd_bias_relu": (lambda i: o.run_conv_tc(tf, view(xs[i]), wf, outs[i], bias=bb, relu=True), 8),
                "dgrad_mask": (lambda i: o.run_conv_tc(td, view(gs[i]), wd, outs[i], mask_src=view(xs[i])), 12),
                "dgrad_add": (lambda i: o.run_conv_tc(td, view(gs[i]), wd, outs[i], add_src=view(xs[i]),
                                                      add_mask=view(xs[(i + 1) % a.rot])), 16),
                "wgrad (+reduce)": (lambda i: o.wgrad3(xs[i], gs[i], w, vertical, dil, bias_grad="skip"), 8),
            }
            if mode == "bf16":
                ops.update({
                    "bf16 fwd_bias_relu (bf16 in, out)": (lambda i: o.run_conv_tc(tf, view(xh[i]), wf, outh[i], bias=bb, relu=True), 4),
                    "bf16 dgrad_mask (bf16 mask)": (lambda i: o.run_conv_tc(td, view(gs[i]), wd, outs[i], mask_src=view(xh[i])), 10),
                    "bf16 wgrad (+reduce) (bf16 x)": (lambda i: o.wgrad3(xh[i], gs[i], w, vertical, dil, bias_grad="skip"), 6),
                })
            for name, (fn, width) in ops.items():
                # a.iters launches (cycling through the input sets) captured into a CUDA graph: the replay time is GPU
                # time, not ctypes launch overhead (~25 us per eager launch)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    for i in range(a.rot):
                        fn(i)
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for i in range(a.iters):
                        fn(i % a.rot)
                g.replay()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / a.iters
                del g
                flops = 2.0 * N * H * W * 3 * C * C
                nbytes = float(width) * N * H * W * C
                print(json.dumps({"mode": mode, "op": name, "C": C, "H": H, "W": W, "vertical": vertical, "dil": dil, "batch": N,
                                  "us": round(us, 2), "tflops": round(flops / us / 1e6, 1), "gbs": round(nbytes / us / 1e3, 0)}),
                      flush=True)


if __name__ == "__main__":
    main()
