"""Gradient clipping in the fused optimizer: the norm launch, the update with and without the clip, and the graphed
training step with and without clipping, in ONE process.

    python tools/bench_grad_clip.py [--modes tf32x3 bf16] [--rounds 3] [--steps 20] [--launches 200] [--out FILE]

Kernels ("kernels"), over the gradients of the model's parameters (2 lanes, with and without --clas; bench.py config 2),
each timed with CUDA events over `--launches` launches after a warm-up:
  grad_norm         lf_grad_norm alone.  The algorithm reads each fp32 gradient once: 4 B per element.
  update_<kind>     lf_optim_step (no clipping), 28 B per element for Adam and RMSprop, 20 B for SGD.
  update_clip_<kind> lf_optim_step_clip alone (the clipped update; it reads the coefficient the norm launch wrote).
  norm_and_update_clip_<kind>  FusedOptimizer(max_grad_norm=1.0).launch(): the norm launch, then the clipped update.
Achieved GB/s counts the bytes the algorithm must move over the measured time.

Graphed step ("iteration"): bench.py's model, loss and batch (config 2: 2 lanes, batch 32, 256x512), one replay of
engine.GraphedTrainStep ending with FusedOptimizer's Adam update, without clipping ("fused") and with max_grad_norm=1.0
("fused_clip"), each re-captured every round; the two arms alternate within each round and the median of `--rounds`
rounds is reported.  ms/step comes from CUDA events around `--steps` replays.
The card name, power limit and SM clocks come from a read-only `nvidia-smi --query-gpu` in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

ARMS = ("fused", "fused_clip")


def iteration_arms(cfg, modes, rounds, steps):
    import torch
    import bench
    from bench_train_iter import _model, _timed
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, args = _model(cfg)
    crit = backprojection_loss(args)
    hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
    dx, dxgt, dvalid = hx.cuda(), hxgt.cuda(), hvalid.cuda()
    L = cfg["nclasses"]
    opts = {"fused": FusedOptimizer(model.parameters(), "adam", 1e-4, 0),
            "fused_clip": FusedOptimizer(model.parameters(), "adam", 1e-4, 0, max_grad_norm=1.0)}
    ms = {(m, arm): [] for m in modes for arm in ARMS}
    norms = []
    default = ops_net.CONV_MODE
    try:
        for _ in range(rounds):
            for m in modes:
                ops_net.set_conv_mode(m)
                for arm in ARMS:
                    g = GraphedTrainStep(model, crit, L, dx, dxgt, dvalid, None, optimizer=opts[arm])
                    for _ in range(3):
                        g()
                    torch.cuda.synchronize()
                    ms[(m, arm)].append(_timed(g, steps))
                    if arm == "fused_clip":
                        norms.append(float(opts[arm].grad_norm))
                    del g
    finally:
        ops_net.set_conv_mode(default)
    out = {m: {arm: {"ms_per_step": [round(v, 3) for v in ms[(m, arm)]],
                     "median_ms": round(statistics.median(ms[(m, arm)]), 3)} for arm in ARMS} for m in modes}
    for m in modes:
        out[m]["clip_over_plain"] = round(out[m]["fused_clip"]["median_ms"] / out[m]["fused"]["median_ms"], 4)
    out["grad_norms_seen"] = [round(n, 4) for n in norms]
    out["skipped"] = {arm: opts[arm].skipped for arm in ARMS}
    out["nonfinite_skipped"] = opts["fused_clip"].nonfinite_skipped
    return out


def kernels(cfg, launches):
    import torch
    from bench_train_iter import _model, _timed
    from lanedetection_end2end_b200 import _capi
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, _ = _model(cfg)
    params = [p for n, p in model.named_parameters() if "encoder.output_conv" not in n]   # never has a gradient
    gen = torch.Generator(device="cuda").manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda", generator=gen) * 1e-3
    numel = sum(p.numel() for p in params)
    rows = {"tensors": len(params), "elements": numel, "norm_bytes_mb": round(4 * numel / 1e6, 2)}

    def row(name, fn, per_elem):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        t = _timed(fn, launches)
        rows[name] = {"us_per_launch": round(t * 1e3, 2), "bytes_per_element": per_elem,
                      "achieved_gb_s": round(per_elem * numel / (t * 1e-3) / 1e9, 1)}

    for kind, per_elem in (("adam", 28), ("sgd", 20), ("rmsprop", 28)):
        plain = FusedOptimizer(params, kind, 1e-6, 0)
        plain.prepare(plain.grad_params())
        plain.sync_hyperparameters()
        row("update_" + kind, plain.launch, per_elem)
        clip = FusedOptimizer(params, kind, 1e-6, 0, max_grad_norm=1.0)
        clip.prepare(clip.grad_params())
        clip.sync_hyperparameters()
        norm = lambda: _capi.call("lf_grad_norm", _capi.ptr(clip._table), clip._nsegs, clip._nchunks,   # noqa: E731
                                  _capi.ptr(clip._clip), _capi.ptr(clip._norm_ws), clip._norm_ws.numel() * 8,
                                  _capi.stream_ptr())
        if kind == "adam":
            row("grad_norm", norm, 4)
            rows["grad_norm_value"] = float(clip.grad_norm)
        norm()
        update = lambda: _capi.call("lf_optim_step_clip", clip.algo, _capi.ptr(clip._table), clip._nsegs,  # noqa: E731
                                    clip._nchunks, _capi.ptr(clip._hyper), _capi.ptr(clip._counters), None,
                                    _capi.ptr(clip._clip), _capi.stream_ptr())
        row("update_clip_" + kind, update, per_elem)
        row("norm_and_update_clip_" + kind, clip.launch, per_elem + 4)
        del plain, clip
    del model
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", nargs="+", default=["tf32x3", "bf16"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import bench
    from bench_modes import gpu_info
    assert torch.cuda.is_available(), "bench_grad_clip.py times the GPU; there is no CPU fallback"
    rec = {"gpu_before": gpu_info(), "rounds": a.rounds, "steps": a.steps, "launches": a.launches, "kernels": {}}
    base = bench.CONFIGS[2]
    for clas in (False, True):
        cfg = dict(base, clas=True) if clas else base
        rec["kernels"]["2lane" + ("_clas" if clas else "")] = kernels(cfg, a.launches)
    rec["iteration"] = {base["name"]: iteration_arms(base, a.modes, a.rounds, a.steps)}
    rec["gpu_after"] = gpu_info()
    txt = json.dumps(rec, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
