"""What --trapezium_mask costs: the least-squares forward and backward per launch with and without the keep map, and
train.sh's graphed training step (4 lanes, order 3, --clas 1, batch 32, resize 256, fused Adam in the graph) with and
without the flag, in the tf32x3 and bf16 convolution modes.  Writes profiles/h100/bench_trapezium.json (or --out).

    python tools/bench_trapezium.py [--out PATH] [--rounds 3] [--steps 30] [--launches 200]

LSQ: lf_lsq_fwd / lf_lsq_bwd against lf_lsq_fwd_keep / lf_lsq_bwd_keep on the same [32, 4, 256, 512] maps (float32, as
the tf32x3 mode hands them over, and bfloat16), the fixed warp's row-separable tables, 52 masked rows, the Net's own
trapezium keep map; --launches launches per round and arm, CUDA events around them.  Step: engine.GraphedTrainStep over
the model, the fused back-projection loss and FusedOptimizer("adam"), on synthetic device-resident inputs; CUDA events
around --steps replays after a warm-up.  Every arm alternates with its partner --rounds times in one process.  The card,
its power limit and SM clock are read with nvidia-smi in the same run."""
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


def make_step(trapezium, mode):
    import torch
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    from lanedetection_end2end_b200.optim import FusedOptimizer
    ops_net.set_conv_mode(mode)
    args = define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--loss_policy", "backproject", "--batch_size",
                                     str(BATCH), "--resize", str(RESIZE), "--nclasses", str(LANES), "--order", str(ORDER),
                                     "--clas", "True", "--mask_percentage", "0.2", "--trapezium_mask", str(trapezium)])
    torch.manual_seed(0)
    model = Net(args).cuda()
    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=g)
    xgt = torch.rand(BATCH, 4, 56, device="cuda", dtype=torch.float64, generator=g) * 200 + 150
    valid = torch.ones(BATCH, 4, 56, device="cuda", dtype=torch.float64)
    step = GraphedTrainStep(model, backprojection_loss(args), LANES, x, xgt, valid, optimizer=opt)

    def run():
        ops_net.set_conv_mode(mode)      # the mode is read when the first call captures the graph
        step()
    return run


def lsq_arms(dtype):
    """{arm: launch function} for one map dtype: the plain and keep forward and backward."""
    import torch
    from lanedetection_end2end_b200 import _capi, ops_lsq
    from lanedetection_end2end_b200.Networks.LSQ_layer import ProjectiveGridGenerator, trapezium_keep
    from lanedetection_end2end_b200.Networks.utils import get_homography
    B, L, H, W, n = BATCH, LANES, RESIZE, 2 * RESIZE, ORDER + 1
    g = torch.Generator(device="cuda").manual_seed(2)
    o = (torch.randn(B, L, H, W, device="cuda", generator=g) * 0.5).to(dtype)
    M, _ = get_homography(RESIZE)
    grid = ProjectiveGridGenerator((B, L, H, W), torch.from_numpy(M).unsqueeze(0).float(), False)
    t = ops_lsq.grid_tables(grid, H, W, 255.0)
    keep = trapezium_keep(RESIZE, MASK_ROWS).cuda()
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    beta = torch.empty(B, L, n, dtype=torch.float64, device="cuda")
    zinv = torch.empty(B, L, n, n, dtype=torch.float64, device="cuda")
    gbeta = torch.randn(B, L, n, dtype=torch.float64, device="cuda", generator=g)
    masked = torch.empty(B, L, H, W, device="cuda")
    d_o = torch.empty_like(o)
    nbytes = _capi.lib().lf_lsq_workspace_bytes(B, L, H, W, ORDER)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    p, sq, dt = _capi.ptr, _capi.ACT_IDS["square"], _capi.dtype_id(o)

    def fwd(k):
        kp = () if k is None else (p(k),)
        return lambda: _capi.call("lf_lsq_fwd" + ("" if k is None else "_keep"), p(o), dt, p(t.xtab), None, p(t.yrow), *kp,
                                  B, L, H, W, ORDER, MASK_ROWS, sq, 0.0, 0, p(beta), p(zinv), p(masked), p(st), p(ws),
                                  ws.numel(), _capi.stream_ptr())

    def bwd(k):
        kp = () if k is None else (p(k),)
        return lambda: _capi.call("lf_lsq_bwd" + ("" if k is None else "_keep"), p(o), dt, p(t.xtab), None, p(t.yrow), *kp,
                                  B, L, H, W, ORDER, MASK_ROWS, sq, p(beta), p(zinv), p(gbeta), p(d_o), _capi.stream_ptr())
    fwd(None)()
    return {"fwd": fwd(None), "fwd_keep": fwd(keep), "bwd": bwd(None), "bwd_keep": bwd(keep)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_trapezium.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_trapezium.py needs a GPU")
    from lanedetection_end2end_b200 import ops_net
    default_mode = ops_net.CONV_MODE
    lsq = {"f32": lsq_arms(torch.float32), "bf16": lsq_arms(torch.bfloat16)}
    steps = {mode: {"plain": make_step(False, mode), "trapezium": make_step(True, mode)} for mode in ("tf32x3", "bf16")}
    ops_net.set_conv_mode(default_mode)
    for arms in list(lsq.values()) + list(steps.values()):
        for f in arms.values():
            time_events(f, 3)
    rec = {"lsq_ms": {dt: {k: [] for k in arms} for dt, arms in lsq.items()},
           "step_ms": {m: {k: [] for k in arms} for m, arms in steps.items()}}
    for _ in range(a.rounds):
        for dt, arms in lsq.items():
            for k, f in arms.items():
                rec["lsq_ms"][dt][k].append(time_events(f, a.launches))
        for m, arms in steps.items():
            for k, f in arms.items():
                rec["step_ms"][m][k].append(time_events(f, a.steps))
    ops_net.set_conv_mode(default_mode)
    med = {g: {s: {k: statistics.median(v) for k, v in d.items()} for s, d in rec[g].items()} for g in rec}
    out = {"gpu": gpu_info(),
           "workload": "LSQ: [%d, %d, %d, %d] maps, order %d, square, %d masked rows, fixed warp (row-separable), per launch; "
                       "step: train.sh shape, batch %d, --clas 1, fused Adam, one graph replay per step"
                       % (BATCH, LANES, RESIZE, 2 * RESIZE, ORDER, MASK_ROWS, BATCH),
           "rounds": a.rounds, "steps_per_round": a.steps, "launches_per_round": a.launches, **rec, "median": med}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(med), out["gpu"])


if __name__ == "__main__":
    main()
