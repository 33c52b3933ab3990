"""Throughput of the GPU bird's-eye-view loader (bev/Dataloader/Load_Data_new.py) against the reference's BEV loader.
Writes profiles/h100/bench_loader_bev.json (or --out).

    python tools/bench_loader_bev.py [--out PATH] [--ref-batches 30]

The dataset is the synthetic 2535-file BEV directory of tests/golden/loader_bev.npz (1280x720 JPEG frames and PNG label maps
behind unpadded names drawn from 1..3625, tiled label rows; oracle/make_loader_bev_golden.py), batch 32, resize 256.
Arms, in one process, with the card's name / power limit / clocks read at the start and the end:
  loader     images/s of one training epoch (2,016 samples, 63 batches) of get_loader with flip on: epoch 1 (read, decode,
             stage into the cache, record the label rows), a cached epoch, and an epoch with the cache off (cache_bytes=0);
             host threads = usable cores;
  reference  images/s of the reference's BEV get_loader (its Load_Data_new.py from the checkout or oracle/_ref/, Pillow on
             DataLoader workers, num_workers = usable cores) with flip off -- its flip path cannot run -- over --ref-batches
             batches after 3 warm-up batches; when its imports do not resolve, the record says so and the arm is skipped."""
import argparse
import contextlib
import io
import json
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

BATCH, RESIZE, COUNT = 32, 256, 2535


def make_loaders(get_loader, paths, workers, flip_on, **kw):
    import torch
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        return get_loader(COUNT, paths["json_file"], paths["image_dir"], paths["gt_dir"], flip_on, BATCH, True, workers, True, RESIZE,
                          **kw)


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
    import torch
    from lanedetection_end2end_b200 import _capi
    kw = {"line_file": paths["line_file"]}
    train, _, _ = make_loaders(L.get_loader, paths, workers, True, **kw)
    rec = {"flip_on": True, "epoch1_decode": time_epoch(train), "cached_epoch": time_epoch(train)}
    _capi.TRACE = []                              # device time of the assembly launches of one more cached epoch
    try:
        time_epoch(train)
        ms = [e0.elapsed_time(e1) for name, e0, e1, _, _ in _capi.TRACE if name == "lf_loader_assemble_bev"]
    finally:
        _capi.TRACE = None
    rec["assemble_kernel_ms_per_batch"] = round(statistics.median(ms), 4)
    del train
    torch.cuda.empty_cache()
    off, _, _ = make_loaders(L.get_loader, paths, workers, True, cache_bytes=0, **kw)
    _capi.TRACE = []                              # and of the label-row search, which runs with every staged batch here
    try:
        rec["cache_off_epoch"] = time_epoch(off)
        ms = [e0.elapsed_time(e1) for name, e0, e1, _, _ in _capi.TRACE if name == "lf_loader_label_rows"]
    finally:
        _capi.TRACE = None
    rec["label_rows_kernel_ms_per_batch"] = round(statistics.median(ms), 4)
    return rec


def reference_arm(paths, workers, nbatches):
    from oracle import make_loader_bev_golden as mbg
    from oracle import reference_import as ri
    try:
        mod = mbg.load_reference()
    except Exception as e:                        # the reference's imports do not resolve here
        return {"skipped": "%s: %s" % (type(e).__name__, e)}
    train, _, _ = make_loaders(mod.get_loader, paths, workers, False)
    it = iter(train)
    for _ in range(3):
        next(it)
    t0 = time.perf_counter()
    for _ in range(nbatches):
        next(it)
    dt = time.perf_counter() - t0
    del it
    return {"timed": "the reference's own BEV Load_Data_new.py from %s" % ri.REFERENCE_ROOT, "flip_on": False, "num_workers": workers,
            "batches": nbatches, "seconds": round(dt, 3), "images_per_s": round(nbatches * BATCH / dt, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_loader_bev.json"))
    ap.add_argument("--ref-batches", type=int, default=30)
    a = ap.parse_args()
    import torch
    from bench_modes import gpu_info
    from oracle import make_loader_bev_golden as mbg
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    assert torch.cuda.is_available(), "bench_loader_bev.py times the GPU; there is no CPU fallback"
    workers = len(os.sched_getaffinity(0))
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "host_cpus_usable": workers, "batch": BATCH, "resize": RESIZE,
           "dataset": "synthetic 2535-file BEV directory (tests/golden/loader_bev.npz): 1280x720 JPEG frames and PNG label maps, "
                      "2,016 training samples after the split and the trim to whole batches"}
    z = np.load(os.path.join(ROOT, "tests", "golden", "loader_bev.npz"))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        paths = mbg.from_fixture(z, d)
        rec["loader"] = loader_arm(L, paths, workers)
        print("loader", rec["loader"], flush=True)
        os.chdir(d)                               # the reference reads Labels/label_new.json
        try:
            rec["reference"] = reference_arm(paths, workers, a.ref_batches)
        finally:
            os.chdir(cwd)
        print("reference", rec["reference"], flush=True)
    rec["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
