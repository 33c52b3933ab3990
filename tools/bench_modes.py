"""Step time of the CUDA-graphed training step (engine.GraphedTrainStep) per convolution mode, alternated in ONE process.

    python tools/bench_modes.py [--configs 2 3] [--modes tf32x3 tf32 bf16] [--rounds 3] [--steps 20] [--out FILE]

For every config the model, loss and batch are built once (bench.py's recipe: kaiming init, random images, synthetic
targets); each round then re-captures the step in every mode in turn and times `--steps` replays with CUDA events, so the
modes see the same card, clock and thermal state.  The card name, power limit and max SM clock come from a read-only
`nvidia-smi --query-gpu` in the same run.  `max_memory_allocated_mb` is torch.cuda.max_memory_allocated() from the
step's capture through its timed replays (the model, its gradients, the graph's memory pool), per mode, largest over
the rounds.  Prints one JSON document (and writes it to --out if given).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        f = [x.strip() for x in out.split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "sm_clock_max_mhz": float(f[2]), "sm_clock_now_mhz": float(f[3])}
    except Exception as e:                       # no nvidia-smi: the record says so
        return {"error": "%s: %s" % (type(e).__name__, e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", type=int, default=[2, 3])
    ap.add_argument("--modes", nargs="+", default=["tf32x3", "tf32", "bf16"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import contextlib
    import io
    import torch
    import bench
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep

    rec = {"gpu_before": gpu_info(), "modes": a.modes, "rounds": a.rounds, "steps": a.steps, "configs": {}}
    default = ops_net.CONV_MODE
    for c in a.configs:
        cfg = bench.CONFIGS[c]
        args = bench.build_args(cfg)
        torch.manual_seed(0)
        model = Net(args)
        with contextlib.redirect_stdout(io.StringIO()):
            define_init_weights(model, "kaiming")
        model = model.cuda().train()
        model.defer_status_check = True
        crit = backprojection_loss(args)
        hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
        dx, dxgt, dvalid = hx.cuda(), hxgt.cuda(), hvalid.cuda()
        ms = {m: [] for m in a.modes}
        peak = {m: 0 for m in a.modes}
        losses = {}
        for _ in range(a.rounds):
            for m in a.modes:
                ops_net.set_conv_mode(m)
                try:
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    g = GraphedTrainStep(model, crit, cfg["nclasses"], dx, dxgt, dvalid, None)
                    for _ in range(3):
                        g()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.steps):
                        loss = g()
                    e1.record()
                    torch.cuda.synchronize()
                    ms[m].append(e0.elapsed_time(e1) / a.steps)
                    peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
                    losses[m] = float(loss)
                    del g
                finally:
                    ops_net.set_conv_mode(default)
        rec["configs"][cfg["name"]] = {
            "batch": cfg["batch"],
            "ms_per_step": {m: [round(v, 3) for v in ms[m]] for m in a.modes},
            "median_ms": {m: round(statistics.median(ms[m]), 3) for m in a.modes},
            "images_per_s": {m: round(cfg["batch"] * 1000.0 / statistics.median(ms[m]), 1) for m in a.modes},
            "max_memory_allocated_mb": {m: round(peak[m] / 2 ** 20, 1) for m in a.modes},
            "last_loss": losses,
        }
        del model
        torch.cuda.empty_cache()
    rec["gpu_after"] = gpu_info()
    txt = json.dumps(rec, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
