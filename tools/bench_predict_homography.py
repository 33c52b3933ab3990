"""What --predict_homography costs: train.sh's graphed training step (4 lanes, order 3, --clas 1, batch 32, resize 256,
fused Adam in the graph) and the graphed eval forward (GraphedInference) with and without the flag, in the tf32x3 and
bf16 convolution modes; the per-launch time of each new kernel; the peak memory of each arm.  Writes
profiles/h100/bench_predict_homography.json (or --out).  ``--corners source`` times the source-corner
parametrisation (--predict_homography_corners source) instead: the fixed warp, the destination corners and the source
corners side by side, and the tables kernel and its backward in both parametrisations; it writes
profiles/h100/bench_predict_homography_source.json.

    python tools/bench_predict_homography.py [--corners destination|source] [--out PATH] [--rounds 3] [--steps 30]
                                             [--launches 200]

Step: engine.GraphedTrainStep over the model, the fused back-projection loss and FusedOptimizer("adam"), on synthetic
device-resident inputs; eval: one GraphedInference replay.  CUDA events around --steps replays after a warm-up; every arm
alternates with its partner --rounds times in one process.  Kernels: each new entry point on the train.sh shapes
([32, 4, 256, 512] float32 maps, 52 masked rows, distinct per-image warps), --launches launches per round, CUDA events
around them.  Peak memory: torch.cuda.max_memory_allocated while an arm is built and replayed three times, above what was
allocated before it.  The card, its power limit and SM clock are read with nvidia-smi in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_homography import BATCH, LANES, ORDER, RESIZE, gpu_info, time_events  # noqa: E402

MASK_ROWS = 52          # ceil(256 * 0.2), train.sh's --mask_percentage 0.2


def make_args(predict, corners="destination"):
    from lanedetection_end2end_b200.Networks.utils import define_args
    return define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--loss_policy", "backproject", "--batch_size",
                                     str(BATCH), "--resize", str(RESIZE), "--nclasses", str(LANES), "--order", str(ORDER),
                                     "--clas", "True", "--mask_percentage", "0.2", "--predict_homography", str(predict),
                                     "--predict_homography_corners", corners])


def make_step(predict, mode, corners="destination"):
    import torch
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.optim import FusedOptimizer
    ops_net.set_conv_mode(mode)
    args = make_args(predict, corners)
    torch.manual_seed(0)
    model = Net(args).cuda()
    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=g)
    xgt = torch.rand(BATCH, 4, 56, device="cuda", dtype=torch.float64, generator=g) * 200 + 150
    valid = torch.ones(BATCH, 4, 56, device="cuda", dtype=torch.float64)
    crit = backprojection_loss(args)
    if predict:
        crit.bind(model)
    step = GraphedTrainStep(model, crit, LANES, x, xgt, valid, optimizer=opt)

    def run():
        ops_net.set_conv_mode(mode)      # the mode is read when the first call captures the graph
        step()
    return run


def make_eval(predict, mode, corners="destination"):
    import torch
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.engine import GraphedInference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    ops_net.set_conv_mode(mode)
    torch.manual_seed(0)
    model = Net(make_args(predict, corners)).cuda().eval()
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    g = GraphedInference(model, x)

    def run():
        ops_net.set_conv_mode(mode)
        g.graph.replay()
    return run


def kernel_arms():
    """{entry point: launch function} for the new kernels on the train.sh shapes."""
    import torch
    from lanedetection_end2end_b200 import _capi
    B, L, H, W, n = BATCH, LANES, RESIZE, 2 * RESIZE, ORDER + 1
    g = torch.Generator(device="cuda").manual_seed(2)
    f64 = dict(dtype=torch.float64, device="cuda")
    z = torch.randn(B, 3, device="cuda", generator=g) * 0.5
    delta, M, Minv = torch.empty(B, 3, **f64), torch.empty(B, 9, **f64), torch.empty(B, 9, **f64)
    rowp, yk = torch.empty(B, H, 3, **f64), torch.empty(B, 56, **f64)
    xtab, yrow = torch.empty(B, H * W, device="cuda"), torch.empty(B, H, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    p = _capi.ptr
    tables = lambda: _capi.call("lf_predicted_homography_tables", p(z), B, H, MASK_ROWS, 255.0, p(delta), p(M), p(Minv),
                                p(rowp), p(xtab), p(yrow), p(yk), p(st), _capi.stream_ptr())
    tables()
    g_rowp = torch.randn(B, H, 3, generator=g, **f64)
    g_minv, g_yk = torch.randn(B, 9, generator=g, **f64), torch.randn(B, 56, generator=g, **f64)
    g_z = torch.empty(B, 3, device="cuda")
    o = torch.randn(B, L, H, W, device="cuda", generator=g) * 0.5 + 0.7
    beta, zinv = torch.empty(B, L, n, **f64), torch.empty(B, L, n, n, **f64)
    gbeta = torch.randn(B, L, n, generator=g, **f64)
    masked, d_o = torch.empty(B, L, H, W, device="cuda"), torch.empty_like(o)
    rowsums = torch.empty(B, L, H, 3, device="cuda")
    nb = _capi.lib().lf_lsq_workspace_bytes(B, L, H, W, ORDER)
    ws = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    sq, dt = _capi.ACT_IDS["square"], _capi.dtype_id(o)

    def fwd(rs):
        return lambda: _capi.call("lf_lsq_fwd_per_image", p(o), dt, p(xtab), p(yrow), None, B, L, H, W, ORDER, MASK_ROWS, sq,
                                  0.0, 0, p(beta), p(zinv), p(masked), p(st), p(rs), p(ws), nb, _capi.stream_ptr())
    fwd(rowsums)()
    x_gt = torch.rand(B, L, 56, generator=g, **f64) * 200 + 150
    valid = torch.ones(B, L, 56, **f64)
    lane, loss, dbeta, xcal = torch.empty(L, **f64), torch.empty(1, **f64), torch.empty_like(beta), torch.empty(B, L, 56, **f64)
    scratch = torch.empty(int(_capi.lib().lf_backproj_loss_per_image_scratch(B, L)), **f64)
    g_const = torch.empty(B, 65, **f64)
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    g_grid = torch.empty(B, H, 3, **f64)
    return {
        "lf_predicted_homography_tables": tables,
        "lf_predicted_homography_bwd": lambda: _capi.call("lf_predicted_homography_bwd", p(z), B, H, MASK_ROWS, p(g_rowp),
                                                          p(g_minv), p(g_yk), p(g_z), _capi.stream_ptr()),
        "lf_lsq_fwd_per_image": fwd(None),
        "lf_lsq_fwd_per_image+rowsums": fwd(rowsums),
        "lf_lsq_bwd_per_image": lambda: _capi.call("lf_lsq_bwd_per_image", p(o), dt, p(xtab), p(yrow), None, B, L, H, W, ORDER,
                                                   MASK_ROWS, sq, p(beta), p(zinv), p(gbeta), p(d_o), _capi.stream_ptr()),
        "lf_lsq_grid_grad_per_image": lambda: _capi.call("lf_lsq_grid_grad_per_image", p(rowsums), p(yrow), p(beta), p(zinv),
                                                         p(gbeta), B, L, H, ORDER, MASK_ROWS, p(g_grid), _capi.stream_ptr()),
        "lf_backproj_loss_per_image": lambda: _capi.call("lf_backproj_loss_per_image", p(yk), p(Minv), p(beta), p(x_gt),
                                                         p(valid), B, L, n, p(lane), p(loss), p(dbeta), p(xcal), p(scratch),
                                                         p(g_const), p(ticket), _capi.stream_ptr()),
    }


def source_kernel_arms():
    """The tables kernel and its backward of both parametrisations on the train.sh shapes, distinct per-image warps."""
    import torch
    from lanedetection_end2end_b200 import _capi
    B, H = BATCH, RESIZE
    g = torch.Generator(device="cuda").manual_seed(2)
    f64 = dict(dtype=torch.float64, device="cuda")
    M, Minv = torch.empty(B, 9, **f64), torch.empty(B, 9, **f64)
    rowp, yk = torch.empty(B, H, 3, **f64), torch.empty(B, 56, **f64)
    xtab, yrow = torch.empty(B, H * 2 * H, device="cuda"), torch.empty(B, H, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    g_rowp = torch.randn(B, H, 3, generator=g, **f64)
    g_minv, g_yk = torch.randn(B, 9, generator=g, **f64), torch.randn(B, 56, generator=g, **f64)
    p = _capi.ptr
    arms = {}
    for name, nz, pdt, extra in (("lf_predicted_homography", 3, torch.float64, ()),
                                 ("lf_predicted_homography_source", 5, torch.float32, (None,))):
        z = torch.randn(B, nz, device="cuda", generator=g) * 0.5
        prm, g_z = torch.empty(B, nz, dtype=pdt, device="cuda"), torch.empty(B, nz, device="cuda")
        arms[name + "_tables"] = (lambda name=name, z=z, prm=prm: _capi.call(
            name + "_tables", p(z), B, H, MASK_ROWS, 255.0, p(prm), p(M), p(Minv), p(rowp), p(xtab), p(yrow), p(yk), p(st),
            _capi.stream_ptr()))
        arms[name + "_bwd"] = (lambda name=name, z=z, g_z=g_z, extra=extra: _capi.call(
            name + "_bwd", p(z), B, H, MASK_ROWS, p(g_rowp), p(g_minv), p(g_yk), p(g_z), *extra, _capi.stream_ptr()))
    return arms


def measured(build):
    """(callable, peak MB allocated while building it and running it three times, above the allocation before)."""
    import torch
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn = build()
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    return fn, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corners", choices=["destination", "source"], default="destination")
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    if a.out is None:
        a.out = os.path.join(ROOT, "profiles", "h100", "bench_predict_homography%s.json"
                             % ("_source" if a.corners == "source" else ""))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict_homography.py needs a GPU")
    from lanedetection_end2end_b200 import ops_net
    default_mode = ops_net.CONV_MODE
    arms, peak = {}, {}
    if a.corners == "source":
        # (label, --predict_homography, --predict_homography_corners): each arm next to the others every round
        variants = (("fixed", False, "destination"), ("destination", True, "destination"), ("source", True, "source"))
    else:
        variants = (("fixed", False, "destination"), ("predict", True, "destination"))
    for mode in ("tf32x3", "bf16"):
        for label, predict, corners in variants:
            k = "%s/%s" % (mode, label)
            arms["step/" + k], peak["step/" + k] = measured(lambda: make_step(predict, mode, corners))
    for label, predict, corners in variants:
        k = "eval/tf32x3/%s" % label
        arms[k], peak[k] = measured(lambda: make_eval(predict, "tf32x3", corners))
    ops_net.set_conv_mode(default_mode)
    kern = source_kernel_arms() if a.corners == "source" else kernel_arms()
    for f in list(arms.values()) + list(kern.values()):
        time_events(f, 3)
    rec = {"arm_ms": {k: [] for k in arms}, "kernel_ms": {k: [] for k in kern}}
    for _ in range(a.rounds):
        for k, f in arms.items():             # each arm next to its partners (fixed first), every round
            rec["arm_ms"][k].append(time_events(f, a.steps))
        for k, f in kern.items():
            rec["kernel_ms"][k].append(time_events(f, a.launches))
    ops_net.set_conv_mode(default_mode)
    med = {g: {k: statistics.median(v) for k, v in d.items()} for g, d in rec.items()}
    out = {"gpu": gpu_info(),
           "workload": "train.sh shape: batch %d, %d lanes, order %d, resize %d, --clas 1, --mask_percentage 0.2; step: one "
                       "graph replay of forward, fused loss, backward and fused Adam; eval: one GraphedInference replay; "
                       "kernels: per launch on [%d, %d, %d, %d] float32 maps, distinct per-image warps"
                       % (BATCH, LANES, ORDER, RESIZE, BATCH, LANES, RESIZE, 2 * RESIZE),
           "rounds": a.rounds, "steps_per_round": a.steps, "launches_per_round": a.launches, **rec, "median": med,
           "peak_allocated_mb": peak}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(med), json.dumps(peak), out["gpu"])


if __name__ == "__main__":
    main()
