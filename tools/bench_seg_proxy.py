"""What the proxy segmentation decoder (--seg_proxy) costs: the graphed training step of config 2 (2 lanes, order 2) and of
train.sh (4 lanes, order 3, --clas 1), both at batch 32 and 256x512 with fused Adam in the graph, with and without the
branch and its cross-entropy term; the graphed eval forward (GraphedInference, batch 32) with and without it; the peak
memory each arm allocates; and lf_seg_confusion per launch at batch 32.  Writes profiles/h100/bench_seg_proxy.json (or
--out).

    python tools/bench_seg_proxy.py [--out PATH] [--rounds 3] [--steps 20] [--launches 200]

Per round and arm: CUDA events around --steps replays (--launches launches) after a warm-up; the arms alternate
--rounds times in one process.  Peak memory: torch.cuda.max_memory_allocated over building the arm's graph and three
replays, above what was allocated before it.  The card, its power limit and SM clock are read with nvidia-smi in the
same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BATCH, RESIZE = 32, 256
CONFIGS = {"config2": (2, 2, False, 0.3), "trainsh": (4, 3, True, 0.2)}      # lanes, order, clas, mask_percentage


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return dict(zip(("name", "power_limit_w", "sm_clock_max_mhz", "sm_clock_mhz"), out))


def make_args(config, proxy):
    from lanedetection_end2end_b200.Networks.utils import define_args
    L, order, clas, mask = CONFIGS[config]
    return define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--loss_policy", "backproject", "--batch_size",
                                     str(BATCH), "--resize", str(RESIZE), "--nclasses", str(L), "--order", str(order),
                                     "--clas", str(clas), "--mask_percentage", str(mask), "--seg_proxy", str(proxy)])


def inputs(L):
    import torch
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=g)
    xgt = torch.rand(BATCH, 4, 56, device="cuda", dtype=torch.float64, generator=g) * 200 + 150
    valid = torch.ones(BATCH, 4, 56, device="cuda", dtype=torch.float64)
    gt = torch.randint(0, L + 1, (BATCH, RESIZE, 2 * RESIZE), device="cuda", generator=g)
    line = torch.randint(0, 2, (BATCH, 4), device="cuda", generator=g).float()
    horizon = torch.randint(0, 2, (BATCH, RESIZE), device="cuda", generator=g).float()
    return x, xgt, valid, gt, line, horizon


def make_step(config, proxy):
    """engine.train_epoch's step: the fused fit loss, --clas's head terms, the proxy term when the model has the branch."""
    import torch
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import define_loss_crit, fused_backprojection_loss, seg_proxy_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.optim import FusedOptimizer
    args = make_args(config, proxy)
    L = args.nclasses
    torch.manual_seed(0)
    model = Net(args).cuda()
    crit, crit_seg = define_loss_crit(args)
    bce = torch.nn.BCEWithLogitsLoss()
    x, xgt, valid, gt, line, horizon = inputs(L)

    def loss_fn(out):
        loss, _ = fused_backprojection_loss(crit, out[:L], xgt, valid)
        if args.clas:
            loss = loss * args.weight_fit + (bce(out[6], line).double() + bce(out[7], horizon).double()) * args.weight_class
        if proxy:
            loss, _ = seg_proxy_loss(loss, crit_seg, out[8], gt, args.weight_seg_proxy)
        return loss

    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    return GraphedTrainStep(model, crit, L, x, xgt, valid, optimizer=opt, loss_fn=loss_fn)


def make_eval(config, proxy):
    import torch
    from lanedetection_end2end_b200.engine import GraphedInference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    args = make_args(config, proxy)
    torch.manual_seed(0)
    model = Net(args).cuda().eval()
    g = GraphedInference(model, inputs(args.nclasses)[0])
    return g.graph.replay


def measured(build):
    """(callable, peak MB allocated while building it and replaying it three times, above the allocation before)."""
    import torch
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn = build()
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    return fn, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def time_events(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def confusion_arms():
    import torch
    from lanedetection_end2end_b200.Loss_crit import seg_confusion
    arms = {}
    for C in (3, 5):
        x = torch.randn(BATCH, C, RESIZE, 2 * RESIZE, device="cuda")
        t = torch.randint(0, C, (BATCH, RESIZE, 2 * RESIZE), device="cuda")
        counts = torch.zeros(C * C, dtype=torch.int64, device="cuda")
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        arms["C%d" % C] = (lambda x=x, t=t, counts=counts, st=st: seg_confusion(x, t, counts, st),
                           x.numel() * 4 + t.numel() * 8)
    return arms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_seg_proxy.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_proxy.py needs a GPU")
    info = gpu_info()
    arms, peak = {}, {}
    for config in CONFIGS:
        for proxy in (False, True):
            k = "%s_%s" % (config, "seg_proxy" if proxy else "plain")
            arms["step/" + k], peak["step/" + k] = measured(lambda: make_step(config, proxy))
    for proxy in (False, True):
        k = "eval/trainsh_%s" % ("seg_proxy" if proxy else "plain")
        arms[k], peak[k] = measured(lambda: make_eval("trainsh", proxy))
    conf = confusion_arms()
    for f in list(arms.values()) + [f for f, _ in conf.values()]:
        time_events(f, 3)
    rec = {k: [] for k in arms}
    rec_conf = {k: [] for k in conf}
    for _ in range(a.rounds):
        for k, f in arms.items():
            rec[k].append(time_events(f, a.steps))
        for k, (f, _) in conf.items():
            rec_conf[k].append(time_events(f, a.launches))
    med_conf = {k: statistics.median(v) for k, v in rec_conf.items()}
    out = {"gpu": info, "gpu_after": gpu_info(),
           "workload": "batch %d, %dx%d; step: one graph replay of forward, loss (fused back-projection loss, --clas heads on "
           "trainsh, the proxy cross-entropy with seg_proxy), backward and fused Adam; eval: one GraphedInference replay "
           "of the trainsh model; lf_seg_confusion on [%d, C, %d, %d] fp32 logits and int64 targets"
           % (BATCH, RESIZE, 2 * RESIZE, BATCH, RESIZE, 2 * RESIZE),
           "configs": {k: dict(zip(("lanes", "order", "clas", "mask_percentage"), v)) for k, v in CONFIGS.items()},
           "rounds": a.rounds, "steps_per_round": a.steps, "launches_per_round": a.launches,
           "ms": rec, "median_ms": {k: statistics.median(v) for k, v in rec.items()},
           "peak_alloc_mb": peak,
           "seg_confusion_ms": rec_conf, "seg_confusion_median_ms": med_conf,
           "seg_confusion_gb_per_s": {k: conf[k][1] / (v * 1e-3) / 1e9 for k, v in med_conf.items()}}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"median_ms": out["median_ms"], "peak_alloc_mb": peak, "seg_confusion_median_ms": med_conf}), info)


if __name__ == "__main__":
    main()
