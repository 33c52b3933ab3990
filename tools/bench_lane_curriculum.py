"""What an egolane epoch of --lane_curriculum saves: the least-squares forward and backward per launch fitting K = 2 of
the 4 lane maps (lf_lsq_fwd_lanes / lf_lsq_bwd_lanes) against all 4 (lf_lsq_fwd / lf_lsq_bwd), and train.sh's graphed
training step (4 lanes, order 3, a --clas 1 model whose heads run in the forward, batch 32, resize 256, fused Adam in the
graph) with model.fit_lanes = 2 and the fit loss over lanes 0 and 1 against the full step, in the tf32x3 and bf16
convolution modes.  The step's loss is the fit loss only (as in tools/bench_trapezium.py): the heads' losses and their
backward are not in it, in either arm.  Writes
profiles/h100/bench_lane_curriculum.json (or --out).

    python tools/bench_lane_curriculum.py [--out PATH] [--rounds 3] [--steps 30] [--launches 200]

LSQ: the same [32, 4, 256, 512] maps (float32, as the tf32x3 mode hands them over, and bfloat16), the fixed warp's
row-separable tables, 52 masked rows, square activation; --launches launches per round and arm, CUDA events around
them.  Step: engine.GraphedTrainStep over the model, the fused back-projection loss and FusedOptimizer("adam"), on
synthetic device-resident inputs; CUDA events around --steps replays after a warm-up.  Every arm alternates with its
partner --rounds times in one process.  The card, its power limit and SM clock are read with nvidia-smi in the same
run."""
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
EGO = 2                 # lanes an egolane epoch fits


def make_step(K, mode):
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
                                     "--clas", "True", "--mask_percentage", "0.2"])
    torch.manual_seed(0)
    model = Net(args).cuda()
    model.fit_lanes = K if K < LANES else None
    opt = FusedOptimizer([p for p in model.parameters() if p.requires_grad], "adam", lr=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(BATCH, 3, RESIZE, 2 * RESIZE, device="cuda", generator=g)
    xgt = torch.rand(BATCH, 4, 56, device="cuda", dtype=torch.float64, generator=g) * 200 + 150
    valid = torch.ones(BATCH, 4, 56, device="cuda", dtype=torch.float64)
    # the step's loss is fused_backprojection_loss over its first K lanes, train_epoch's loss in an egolane epoch
    step = GraphedTrainStep(model, backprojection_loss(args), K, x, xgt, valid, optimizer=opt)

    def run():
        ops_net.set_conv_mode(mode)      # the mode is read when the first call captures the graph
        step()
    return run


def lsq_arms(dtype):
    """{arm: launch function} for one map dtype: forward and backward fitting all lanes and the first EGO lanes."""
    import torch
    from lanedetection_end2end_b200 import _capi, ops_lsq
    from lanedetection_end2end_b200.Networks.LSQ_layer import ProjectiveGridGenerator
    from lanedetection_end2end_b200.Networks.utils import get_homography
    B, Lmap, H, W, n = BATCH, LANES, RESIZE, 2 * RESIZE, ORDER + 1
    g = torch.Generator(device="cuda").manual_seed(2)
    o = (torch.randn(B, Lmap, H, W, device="cuda", generator=g) * 0.5).to(dtype)
    M, _ = get_homography(RESIZE)
    grid = ProjectiveGridGenerator((B, Lmap, H, W), torch.from_numpy(M).unsqueeze(0).float(), False)
    t = ops_lsq.grid_tables(grid, H, W, 255.0)
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    beta = torch.empty(B, Lmap, n, dtype=torch.float64, device="cuda")
    zinv = torch.empty(B, Lmap, n, n, dtype=torch.float64, device="cuda")
    gbeta = torch.randn(B, Lmap, n, dtype=torch.float64, device="cuda", generator=g)
    masked = torch.empty(B, Lmap, H, W, device="cuda")
    d_o = torch.empty_like(o)
    nbytes = _capi.lib().lf_lsq_workspace_bytes(B, Lmap, H, W, ORDER)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    p, sq, dt = _capi.ptr, _capi.ACT_IDS["square"], _capi.dtype_id(o)

    def Ls(K):
        return ("", (K,)) if K == Lmap else ("_lanes", (K, Lmap))

    def fwd(K):
        sfx, ls = Ls(K)
        return lambda: _capi.call("lf_lsq_fwd" + sfx, p(o), dt, p(t.xtab), None, p(t.yrow), B, *ls, H, W, ORDER,
                                  MASK_ROWS, sq, 0.0, 0, p(beta), p(zinv), p(masked), p(st), p(ws), ws.numel(),
                                  _capi.stream_ptr())

    def bwd(K):
        sfx, ls = Ls(K)
        return lambda: _capi.call("lf_lsq_bwd" + sfx, p(o), dt, p(t.xtab), None, p(t.yrow), B, *ls, H, W, ORDER,
                                  MASK_ROWS, sq, p(beta), p(zinv), p(gbeta), p(d_o), _capi.stream_ptr())
    fwd(Lmap)()
    return {"fwd_k4": fwd(Lmap), "fwd_k2": fwd(EGO), "bwd_k4": bwd(Lmap), "bwd_k2": bwd(EGO)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_lane_curriculum.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_curriculum.py needs a GPU")
    from lanedetection_end2end_b200 import ops_net
    default_mode = ops_net.CONV_MODE
    lsq = {"f32": lsq_arms(torch.float32), "bf16": lsq_arms(torch.bfloat16)}
    steps = {mode: {"k4": make_step(LANES, mode), "k2": make_step(EGO, mode)} for mode in ("tf32x3", "bf16")}
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
    for dt, d in med["lsq_ms"].items():
        d["fwd_bwd_k4"], d["fwd_bwd_k2"] = d["fwd_k4"] + d["bwd_k4"], d["fwd_k2"] + d["bwd_k2"]
    out = {"gpu": gpu_info(),
           "workload": "LSQ: [%d, %d, %d, %d] maps, order %d, square, %d masked rows, fixed warp (row-separable), per "
                       "launch, fitting K = %d or all %d lanes; step: train.sh shape, batch %d, a --clas 1 model (heads in "
                       "the forward, fit loss only), fused Adam, one graph replay per step, model.fit_lanes = K and the "
                       "loss over K lanes"
                       % (BATCH, LANES, RESIZE, 2 * RESIZE, ORDER, MASK_ROWS, EGO, LANES, BATCH),
           "rounds": a.rounds, "steps_per_round": a.steps, "launches_per_round": a.launches, **rec, "median": med}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(med), out["gpu"])


if __name__ == "__main__":
    main()
