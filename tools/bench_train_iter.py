"""Training iteration with the optimizer update: today's loop against the fully graphed one, alternated in ONE process.

    python tools/bench_train_iter.py [--configs 2 3] [--modes tf32x3 bf16] [--rounds 3] [--steps 20] [--launches 200]
                                     [--out FILE]

Arms, per config and convolution mode, each re-captured every round (bench.py's model, loss and batch recipe):
  (a) torch_adam: an engine.GraphedTrainStep replay (zero grads -> forward -> loss -> backward), then an eager
      torch.optim.Adam step (foreach, torch's default on CUDA);
  (b) fused:      one replay of the GraphedTrainStep that ends with optim.FusedOptimizer's guarded Adam update.
ms/step comes from CUDA events around `--steps` iterations.

The update alone ("update_kernels"): one launch over the model's parameters with a gradient (2 lanes, with and
without --clas), timed with CUDA events over `--launches` launches after a warm-up: the fused kernel (Adam, SGD, RMSprop)
against torch.optim.Adam with foreach=True and with fused=True.  Achieved GB/s counts the bytes the algorithm must move:
28 B per element for Adam and RMSprop (read p, g and two state tensors, write p and both states), 20 B for SGD.
The card name, power limit and SM clocks come from a read-only `nvidia-smi --query-gpu` in the same run.
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


def _timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _model(cfg):
    import torch
    import bench
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    args = bench.build_args(cfg)
    torch.manual_seed(0)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")
    return model.cuda().train(), args


def iteration_arms(cfg, modes, rounds, steps):
    import torch
    import bench
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, args = _model(cfg)
    crit = backprojection_loss(args)
    hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
    dx, dxgt, dvalid = hx.cuda(), hxgt.cuda(), hvalid.cuda()
    L = cfg["nclasses"]
    torch_adam = torch.optim.Adam(model.parameters(), lr=1e-4)
    fused = FusedOptimizer(model.parameters(), "adam", 1e-4, 0)
    ms = {(m, arm): [] for m in modes for arm in ("torch_adam", "fused")}
    default = ops_net.CONV_MODE
    try:
        for _ in range(rounds):
            for m in modes:
                ops_net.set_conv_mode(m)
                for arm in ("torch_adam", "fused"):
                    if arm == "torch_adam":
                        g = GraphedTrainStep(model, crit, L, dx, dxgt, dvalid, None)

                        def it():
                            g()
                            torch_adam.step()
                    else:
                        g = GraphedTrainStep(model, crit, L, dx, dxgt, dvalid, None, optimizer=fused)
                        it = g
                    for _ in range(3):
                        it()
                    torch.cuda.synchronize()
                    ms[(m, arm)].append(_timed(it, steps))
                    del g, it
    finally:
        ops_net.set_conv_mode(default)
    return {m: {arm: {"ms_per_step": [round(v, 3) for v in ms[(m, arm)]], "median_ms": round(statistics.median(ms[(m, arm)]), 3)}
                for arm in ("torch_adam", "fused")} for m in modes}


def update_kernels(cfg, launches):
    import torch
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, _ = _model(cfg)
    params = [p for n, p in model.named_parameters() if "encoder.output_conv" not in n]   # never has a gradient
    gen = torch.Generator(device="cuda").manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda", generator=gen) * 1e-3
    numel = sum(p.numel() for p in params)
    rows = {"tensors": len(params), "elements": numel}

    def row(name, fn, per_elem):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        t = _timed(fn, launches)
        rows[name] = {"us_per_launch": round(t * 1e3, 2), "bytes_per_element": per_elem,
                      "achieved_gb_s": round(per_elem * numel / (t * 1e-3) / 1e9, 1)}

    for kind, per_elem in (("adam", 28), ("sgd", 20), ("rmsprop", 28)):
        opt = FusedOptimizer(params, kind, 1e-6, 0)
        opt.prepare(opt.grad_params())
        opt.sync_hyperparameters()
        row("fused_kernel_" + kind, opt.launch, per_elem)
    row("torch_adam_foreach", torch.optim.Adam(params, lr=1e-6, foreach=True).step, 28)
    row("torch_adam_fused", torch.optim.Adam(params, lr=1e-6, fused=True).step, 28)
    del model
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", type=int, default=[2, 3])
    ap.add_argument("--modes", nargs="+", default=["tf32x3", "bf16"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import bench
    from bench_modes import gpu_info
    assert torch.cuda.is_available(), "bench_train_iter.py times the GPU; there is no CPU fallback"
    rec = {"gpu_before": gpu_info(), "rounds": a.rounds, "steps": a.steps, "iteration": {}, "update_kernels": {}}
    for c in a.configs:
        cfg = bench.CONFIGS[c]
        rec["iteration"][cfg["name"]] = iteration_arms(cfg, a.modes, a.rounds, a.steps)
        torch.cuda.empty_cache()
    base = bench.CONFIGS[2]
    for clas in (False, True):
        cfg = dict(base, clas=True) if clas else base
        rec["update_kernels"]["2lane" + ("_clas" if clas else "")] = update_kernels(cfg, a.launches)
    rec["gpu_after"] = gpu_info()
    txt = json.dumps(rec, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
