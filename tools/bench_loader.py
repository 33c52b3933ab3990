"""Throughput of the GPU TuSimple loader (Dataloader/Load_Data_new.py) against the reference's loader, and the graphed config-2
training step fed by it.  Writes profiles/h100/bench_loader.json (or --out).

    python tools/bench_loader.py [--out PATH] [--rounds 3] [--steps 80] [--ref-batches 30]

The dataset is the synthetic 3626-file TuSimple-shaped directory of tests/golden/loader_tusimple.npz (1280x720 JPEG frames and
PNG label maps behind unpadded names, tiled label rows; oracle/make_loader_golden.py), batch 32, resize 256, flip on.
Arms, in one process, with the card's name / power limit / clocks read at the start:
  loader     images/s of one training epoch (2,900 samples, 90 batches) of get_loader: epoch 1 (read, decode, stage into the
             cache), a cached epoch, and an epoch with the cache off (cache_bytes=0); host threads = usable cores;
  reference  images/s of the reference's get_loader (its Load_Data_new.py from the checkout or oracle/_ref/, Pillow on
             DataLoader workers, num_workers = usable cores) over --ref-batches batches after 3 warm-up batches; when its
             imports do not resolve, the record says so and the arm is skipped;
  step       the graphed config-2 training step (tf32x3, batch 32) over --steps steps: with a static batch, fed by the cached
             loader, and fed by a fresh loader in its first epoch (decoding), alternated --rounds times; ms per step and
             the median of the rounds.  A loader arm fetches the epoch's first batch before the timed window and then runs
             the training loop's order (load, step, next batch)."""
import argparse
import contextlib
import io
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

BATCH, RESIZE, NCLASSES = 32, 256, 2


def make_loaders(L, paths, workers, **kw):
    import torch
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        return L.get_loader(3626, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"], True, BATCH, BATCH,
                            True, workers, True, RESIZE, NCLASSES, line_file=paths["line_file"], **kw)


def time_epoch(loader):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for b in loader:
        n += b[0].shape[0]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"images": n, "seconds": round(dt, 3), "images_per_s": round(n / dt, 1)}


def loader_arm(L, paths, workers):
    train, _, _ = make_loaders(L, paths, workers)
    import torch
    from lanedetection_end2end_b200 import _capi
    rec = {"epoch1_decode": time_epoch(train), "cached_epoch": time_epoch(train)}
    _capi.TRACE = []                              # device time of the assembly launches of one more cached epoch
    try:
        time_epoch(train)
        ms = [e0.elapsed_time(e1) for name, e0, e1, _, _ in _capi.TRACE if name == "lf_loader_assemble"]
    finally:
        _capi.TRACE = None
    rec["assemble_kernel_ms_per_batch"] = round(statistics.median(ms), 4)
    del train
    torch.cuda.empty_cache()
    off, _, _ = make_loaders(L, paths, workers, cache_bytes=0)
    rec["cache_off_epoch"] = time_epoch(off)
    return rec


def reference_arm(paths, workers, nbatches):
    import torch
    from oracle import make_loader_golden as mlg
    from oracle import reference_import as ri
    try:
        mod = mlg.load_reference()
    except Exception as e:                        # the reference's imports do not resolve here
        return {"skipped": "%s: %s" % (type(e).__name__, e)}
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        train, _, _ = mod.get_loader(3626, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"], True, BATCH,
                                     BATCH, True, workers, True, RESIZE, NCLASSES)
    it = iter(train)
    for _ in range(3):
        next(it)
    t0 = time.perf_counter()
    for _ in range(nbatches):
        next(it)
    dt = time.perf_counter() - t0
    del it
    return {"timed": "the reference's own Load_Data_new.py from %s" % ri.REFERENCE_ROOT, "num_workers": workers,
            "batches": nbatches, "seconds": round(dt, 3), "images_per_s": round(nbatches * BATCH / dt, 1)}


def step_arm(L, paths, workers, rounds, steps):
    import torch
    import bench
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    cfg = bench.CONFIGS[2]
    args = bench.build_args(cfg)
    torch.manual_seed(0)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")
    model = model.cuda().train()
    hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
    g = GraphedTrainStep(model, backprojection_loss(args), cfg["nclasses"], hx.cuda(), hxgt.cuda(), hvalid.cuda(), None, warmup=3)
    cached, _, _ = make_loaders(L, paths, workers)
    for _ in cached:                              # fill the cache
        pass

    def run(arm):
        loader = cached
        if arm == "loader_epoch1":
            loader, _, _ = make_loaders(L, paths, workers)
        it = iter(loader) if arm != "static" else None
        b = next(it) if it is not None else None      # the epoch's first batch comes before the timed window
        for _ in range(3):
            g()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):                        # the training loop's order: load, step, next batch
            if it is not None:
                g.load(b[0], b[2], b[-1])
            g()
            if it is not None:
                b = next(it)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    res = {"static": [], "loader_cached": [], "loader_epoch1": []}
    for _ in range(rounds):
        for arm in res:
            res[arm].append(round(run(arm), 3))
    out = {arm: {"ms_per_step": v, "median_ms": round(statistics.median(v), 3)} for arm, v in res.items()}
    out["config"] = cfg["name"] + " (tf32x3, graphed)"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_loader.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=80)
    ap.add_argument("--ref-batches", type=int, default=30)
    a = ap.parse_args()
    import json
    import torch
    from bench_modes import gpu_info
    from oracle import make_loader_golden as mlg
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    assert torch.cuda.is_available(), "bench_loader.py times the GPU; there is no CPU fallback"
    workers = len(os.sched_getaffinity(0))
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "host_cpus_usable": workers, "batch": BATCH, "resize": RESIZE,
           "dataset": "synthetic 3626-file TuSimple-shaped directory (tests/golden/loader_tusimple.npz): 1280x720 JPEG frames "
                      "and PNG label maps, 2,900 training samples"}
    z = np.load(os.path.join(ROOT, "tests", "golden", "loader_tusimple.npz"))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        paths = mlg.from_fixture(z, d)
        rec["loader"] = loader_arm(L, paths, workers)
        print("loader", rec["loader"], flush=True)
        os.chdir(d)                               # the reference reads Labels/label_new.json
        try:
            rec["reference"] = reference_arm(paths, workers, a.ref_batches)
        finally:
            os.chdir(cwd)
        print("reference", rec["reference"], flush=True)
        rec["step"] = step_arm(L, paths, workers, a.rounds, a.steps)
        print("step", rec["step"], flush=True)
    rec["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
