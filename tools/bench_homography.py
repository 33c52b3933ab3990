"""What --learn_homography costs: train.sh's graphed training step (4 lanes, order 3, --clas 1, batch 32, resize 256,
fused Adam in the graph) with the fixed warp against the learned warp, and the least-squares forward with and without
the row sums the warp's gradient needs.  Writes profiles/h100/bench_homography.json (or --out).

    python tools/bench_homography.py [--out PATH] [--rounds 3] [--steps 30] [--launches 200]

Step: engine.GraphedTrainStep over the model, the fused back-projection loss and FusedOptimizer("adam"), on synthetic
device-resident inputs; per round and arm, CUDA events around --steps replays after a warm-up; the two arms (each with
its own model and optimizer) alternate --rounds times in one process.  LSQ forward: lf_lsq_fwd (fixed-warp tables)
against lf_lsq_fwd_rowsums (the learned warp's tables) on the same [32, 4, 256, 512] fp32 maps, --launches launches per
round and arm, alternated.  The card, its power limit and SM clock are read with nvidia-smi in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BATCH, RESIZE, LANES, ORDER = 32, 256, 4, 3


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(zip(("name", "power_limit_w", "sm_clock_max_mhz", "sm_clock_mhz"), out))


def make_step(learn):
    import torch
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    from lanedetection_end2end_b200.optim import FusedOptimizer
    args = define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--loss_policy", "backproject", "--batch_size",
                                     str(BATCH), "--resize", str(RESIZE), "--nclasses", str(LANES), "--order", str(ORDER),
                                     "--clas", "True", "--mask_percentage", "0.2", "--learn_homography", str(learn)])
    torch.manual_seed(0)
    model = Net(args).cuda()
    crit = backprojection_loss(args)
    if learn:
        crit.bind(model)
    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=g)
    xgt = torch.rand(BATCH, 4, 56, device="cuda", dtype=torch.float64, generator=g) * 200 + 150
    valid = torch.ones(BATCH, 4, 56, device="cuda", dtype=torch.float64)
    return GraphedTrainStep(model, crit, LANES, x, xgt, valid, optimizer=opt)


def time_events(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def lsq_arms():
    import torch
    from lanedetection_end2end_b200 import _capi, homography as hg, ops_lsq
    from lanedetection_end2end_b200.Networks.LSQ_layer import ProjectiveGridGenerator
    from lanedetection_end2end_b200.Networks.utils import get_homography
    B, L, H, W, mask = BATCH, LANES, RESIZE, 2 * RESIZE, 52
    o = torch.randn(B, L, H, W, device="cuda")
    M, _ = get_homography(RESIZE)
    grid = ProjectiveGridGenerator((B, L, H, W), torch.from_numpy(M).unsqueeze(0).float(), False)
    fixed = ops_lsq.grid_tables(grid, H, W, 255.0)
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    warp = hg.LearnedHomography(RESIZE, mask).cuda()(st)
    n = ORDER + 1
    beta = torch.empty(B, L, n, dtype=torch.float64, device="cuda")
    zinv = torch.empty(B, L, n, n, dtype=torch.float64, device="cuda")
    masked = torch.empty(B, L, H, W, device="cuda")
    rowsums = torch.empty(B, L, H, 3, device="cuda")
    nbytes = _capi.lib().lf_lsq_workspace_bytes(B, L, H, W, ORDER)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    p, sq = _capi.ptr, _capi.ACT_IDS["square"]

    def plain():
        _capi.call("lf_lsq_fwd", p(o), 0, p(fixed.xtab), None, p(fixed.yrow), B, L, H, W, ORDER, mask, sq, 0.0, 0, p(beta),
                   p(zinv), p(masked), p(st), p(ws), ws.numel(), _capi.stream_ptr())

    def sums():
        _capi.call("lf_lsq_fwd_rowsums", p(o), 0, p(warp.xtab), p(warp.yrow), B, L, H, W, ORDER, mask, sq, 0.0, 0, p(beta),
                   p(zinv), p(masked), p(st), p(rowsums), p(ws), ws.numel(), _capi.stream_ptr())
    return plain, sums


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_homography.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_homography.py needs a GPU")
    steps = {"fixed_warp": make_step(False), "learned_warp": make_step(True)}
    plain, sums = lsq_arms()
    lsq = {"lf_lsq_fwd": plain, "lf_lsq_fwd_rowsums": sums}
    for f in list(steps.values()) + list(lsq.values()):
        time_events(f, 3)
    rec = {"step_ms": {k: [] for k in steps}, "lsq_fwd_ms": {k: [] for k in lsq}}
    for _ in range(a.rounds):
        for k, f in steps.items():
            rec["step_ms"][k].append(time_events(f, a.steps))
        for k, f in lsq.items():
            rec["lsq_fwd_ms"][k].append(time_events(f, a.launches))
    out = {"gpu": gpu_info(), "workload": "train.sh step: batch %d, %dx%d, %d lanes, order %d, --clas 1, fused Adam, one "
           "graph replay per step; LSQ forward on [%d, %d, %d, %d] fp32, mask 52 rows" % (BATCH, RESIZE, 2 * RESIZE, LANES,
                                                                                          ORDER, BATCH, LANES, RESIZE, 2 * RESIZE),
           "rounds": a.rounds, "steps_per_round": a.steps, "launches_per_round": a.launches, **rec,
           "median": {g: {k: statistics.median(v) for k, v in rec[g].items()} for g in ("step_ms", "lsq_fwd_ms")}}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["median"]), out["gpu"])


if __name__ == "__main__":
    main()
