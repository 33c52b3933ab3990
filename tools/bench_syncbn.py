"""Cost of SyncBatchNorm on one GPU: the graphed config-2 training step with nn.SyncBatchNorm containers against
nn.BatchNorm2d containers, alternated in ONE process.

    python tools/bench_syncbn.py [--rounds 3] [--steps 50] [--out FILE]

One model: the two arms swap its BatchNorm containers in place, and the SyncBatchNorm containers share the parameters
and running statistics of the BatchNorm2d ones (torch.nn.SyncBatchNorm.convert_sync_batchnorm), so both arms train the
same tensors.  Without a process group the converted arm runs the collapse and finalize-from-totals launches of every
BatchNorm, forward and backward, and no collective: this times exactly the launches SyncBatchNorm adds.  The cost of the
all-reduces of a multi-GPU run is not measured here.

Per round and arm, engine.GraphedTrainStep is re-captured (3 eager warm-up steps, then the capture), replayed 3 times,
then timed with CUDA events around `--steps` replays.  launches/step is the number of C-ABI launches of one step: the
launches counted while the step object is built, over its 3 warm-up steps and the capture, divided by 4 (the first round
is left out: its first warm-up step registers the packed weight operands).  The card name, power limit and SM clocks
come from a read-only `nvidia-smi --query-gpu` in the same run.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

WARMUP = 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import bench
    from bench_modes import gpu_info
    from lanedetection_end2end_b200 import _capi
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    assert torch.cuda.is_available(), "bench_syncbn.py times the GPU; there is no CPU fallback"

    cfg = bench.CONFIGS[2]
    args = bench.build_args(cfg)
    torch.manual_seed(0)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")       # matches BatchNorm2d containers: initialise before converting
    model = model.cuda().train()
    # (parent, attribute, BatchNorm2d, SyncBatchNorm sharing its parameters and buffers)
    slots = [(parent, name, child, torch.nn.SyncBatchNorm.convert_sync_batchnorm(child))
             for parent in list(model.modules()) for name, child in parent.named_children()
             if isinstance(child, torch.nn.BatchNorm2d)]

    def use(arm):
        for parent, name, plain, sync in slots:
            setattr(parent, name, sync if arm == "syncbatchnorm_world1" else plain)

    crit = backprojection_loss(args)
    hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
    dx, dxgt, dvalid = hx.cuda(), hxgt.cuda(), hvalid.cuda()
    arms = ("batchnorm2d", "syncbatchnorm_world1")
    rec = {"gpu_before": gpu_info(), "config": cfg["name"], "batch": cfg["batch"], "rounds": a.rounds, "steps": a.steps,
           "batchnorms": len(slots)}
    ms = {k: [] for k in arms}
    launches = {k: [] for k in arms}
    losses = {}
    try:
        for r in range(a.rounds):
            for arm in arms:
                use(arm)
                n0 = _capi.LAUNCHES
                g = GraphedTrainStep(model, crit, cfg["nclasses"], dx, dxgt, dvalid, None, warmup=WARMUP)
                if r > 0:
                    launches[arm].append((_capi.LAUNCHES - n0) / (WARMUP + 1))
                for _ in range(3):
                    g()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    loss = g()
                e1.record()
                torch.cuda.synchronize()
                ms[arm].append(e0.elapsed_time(e1) / a.steps)
                losses[arm] = float(loss)
                del g
    finally:
        use("batchnorm2d")
    med = {k: statistics.median(ms[k]) for k in arms}
    rec["arms"] = {k: {"ms_per_step": [round(v, 3) for v in ms[k]], "median_ms": round(med[k], 3),
                       "images_per_s": round(cfg["batch"] * 1000.0 / med[k], 1),
                       "launches_per_step": launches[k][-1] if launches[k] else None, "last_loss": losses[k]} for k in arms}
    rec["overhead_ms_per_step"] = round(med["syncbatchnorm_world1"] - med["batchnorm2d"], 3)
    rec["overhead_pct"] = round(100.0 * (med["syncbatchnorm_world1"] / med["batchnorm2d"] - 1.0), 2)
    rec["collectives_per_step_multi_gpu"] = 2 * len(slots)
    rec["collective_cost"] = "not measured (needs >= 2 GPUs)"
    rec["gpu_after"] = gpu_info()
    txt = json.dumps(rec, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
