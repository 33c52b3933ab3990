#!/usr/bin/env python
"""Wall-clock of one test-set evaluation pass (BP/test.py test_model + LaneEval.bench_one_submit) on the train.sh model
(4 lanes, order 3, --clas 1, 256x512, batch 32) over 2,782 seeded synthetic frames (the size of the TuSimple test set)
that sit on the device, so loading is not timed.  The ground truth is a seeded synthetic test_label.json, 56 samples per
row, 3-5 straight lanes.  Writes profiles/h100/bench_test_eval.json (or --out).

    python tools/bench_test_eval.py [--images 2782] [--rounds 3] [--out PATH]

Arms, alternated --rounds times in one process:
  host    what the repository offered before inference.test_model: GraphedInference forward, the head ops,
          Projections.compute_all, lanes_from_predictions (host copy per batch) and write_tusimple_predictions, then the
          reference's own LaneEval.bench_one_submit (eval_lane.py from oracle/_ref, sklearn on the host); reported as not
          run when the reference module or sklearn is missing
  graphed inference.test_model: one graph replay per batch (forward, heads, Projections, lf_tusimple_score), the file
          and the metric at the end
Both arms build their CUDA graph inside the timed pass, as an epoch does.  The scorer's one-time ground-truth table
build is timed on its own.  The two arms' files must be byte-identical and their [accuracy, fp, fn] equal."""
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

H = list(range(160, 720, 10))


def synthetic_ground_truth(n, seed):
    rng = np.random.default_rng(seed)
    y = np.asarray(H, np.float64)
    rows = []
    for i in range(n):
        lanes = []
        for _ in range(int(rng.integers(3, 6))):
            x = rng.uniform(100, 1180) + rng.uniform(-1.2, 1.2) * (y - 400)
            x = np.where((x >= 0) & (x <= 1279) & (y >= rng.uniform(160, 300)), np.round(x), -2).astype(int)
            lanes.append(x.tolist())
        rows.append({"lanes": lanes, "h_samples": H, "raw_file": "clips/synthetic/%05d/20.jpg" % i})
    return rows


def load_lane_eval():
    try:
        import sklearn  # noqa: F401
        from oracle.make_tusimple_golden import load_lane_eval as load
        return load(), None
    except Exception as e:
        return None, "%s: %s" % (type(e).__name__, e)


def host_arm(model, args, batches, rows, gt_file, pred_file, LaneEval):
    import torch
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.engine import GraphedInference
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    proj = inference.Projections(args)
    gi = GraphedInference(model, batches[0])
    first = 0
    with torch.no_grad(), open(pred_file, "w") as f:
        for xb in batches:
            n = xb.shape[0]
            gi.x[:n].copy_(xb, non_blocking=True)
            gi.graph.replay()
            out = [t[:n] if torch.is_tensor(t) else t for t in gi.out]
            horizon_pred = torch.sigmoid(out[7]).sum(dim=1)
            horizon_pred = (torch.round((inference.resize_coordinates(horizon_pred) + 80) / 10) * 10).int()
            line_pred = torch.round(torch.sigmoid(out[6]))
            lanes = inference.lanes_from_predictions(proj.compute_all(out[:4]), line_pred, horizon_pred)
            inference.write_tusimple_predictions(f, rows, lanes, first)
            first += n
    gi.check()
    res = LaneEval.bench_one_submit(pred_file, gt_file)
    return time.perf_counter() - t0, [float(v) for v in res]


def graphed_arm(model, args, batches, gt_file):
    import torch
    from lanedetection_end2end_b200 import inference
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        inference.test_model(batches, model, None, None, None, None, args)
    dt = time.perf_counter() - t0
    return dt, inference._scorer_for(gt_file, batches[0].device).result()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=2782)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_test_eval.json"))
    a = ap.parse_args()
    import torch
    import bench
    from bench_modes import gpu_info
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    assert torch.cuda.is_available(), "bench_test_eval.py times the GPU; there is no CPU fallback"
    cfg = dict(nclasses=4, order=3, mask=0.2, resize=256, batch=32, clas=True)
    args = bench.build_args(cfg)
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "host_cpus_usable": len(os.sched_getaffinity(0)),
           "workload": "train.sh model (4 lanes, order 3, --clas 1, 256x512, kaiming init, seed 0), batch 32, %d synthetic "
                       "frames on the device; synthetic test_label.json with 56 samples and 3-5 lanes per row" % a.images}
    torch.manual_seed(0)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")
    model = model.cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1234)
    frames = torch.rand(a.images, 3, 256, 512, device="cuda", generator=g)
    batches = list(frames.split(cfg["batch"]))
    rows = synthetic_ground_truth(a.images, 99)
    LaneEval, why = load_lane_eval()
    with tempfile.TemporaryDirectory() as d:
        args.test_dir = args.save_path = d
        gt_file, host_file = os.path.join(d, "test_label.json"), os.path.join(d, "host_predictions.json")
        with open(gt_file, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
        t0 = time.perf_counter()
        inference._scorer_for(gt_file, frames.device)
        rec["scorer_table_build_s"] = round(time.perf_counter() - t0, 3)
        times = {"host": [], "graphed": []}
        results = {}
        for _ in range(a.rounds):
            if LaneEval is not None:
                dt, results["host"] = host_arm(model, args, batches, rows, gt_file, host_file, LaneEval)
                times["host"].append(round(dt, 3))
            dt, results["graphed"] = graphed_arm(model, args, batches, gt_file)
            times["graphed"].append(round(dt, 3))
            print(times, flush=True)
        graphed_file = os.path.join(d, "test_set_predictions.json")
        if LaneEval is not None:
            with open(host_file, "rb") as f1, open(graphed_file, "rb") as f2:
                rec["files_identical"] = f1.read() == f2.read()
            rec["triples_equal"] = results["host"] == results["graphed"]
            assert rec["files_identical"] and rec["triples_equal"], (results, rec)
        else:
            rec["host_arm"] = "not run: " + why
    rec["accuracy_fp_fn"] = results["graphed"]
    rec["pass_s"] = times
    rec["median_pass_s"] = {k: round(statistics.median(v), 3) for k, v in times.items() if v}
    if times["host"]:
        rec["speedup_host_over_graphed"] = round(rec["median_pass_s"]["host"] / rec["median_pass_s"]["graphed"], 2)
    print(json.dumps(rec, indent=1))
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
