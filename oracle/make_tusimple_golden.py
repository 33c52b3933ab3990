"""Write tests/golden/tusimple_eval.npz: the TuSimple metric of the reference's own LaneEval (BP/eval_lane.py) on ground-truth
rows of the reference's label files, with seeded predictions and hand-built edge cases.  CPU only; needs the reference
checkout (oracle/reference_import.py) and sklearn.

    python -m oracle.make_tusimple_golden [--rows 290] [--out tests/golden/tusimple_eval.npz]

Contents:
  gt_jsonl      uint8, the ground-truth rows as UTF-8 JSON lines (raw_file, lanes, h_samples): rows of
                label_data_0531/0601.json with 56 samples and 2-5 lanes, then the hand-built rows (raw_file 'edge/...')
  x_cal         [N, 4, 56] f64 predicted lanes in 1280-wide pixels; line_pred [N, 4] f32 (head order); horizon_pred [N] int32
  lanes         [N, 4, 56] int32 gated lanes of inference.lanes_from_predictions (the reference's own gating line does not
                run on torch 2, so the existing host path is the reference for gating)
  thresh        [N, 8] f64 LaneEval.pixel_thresh / cos(LaneEval.get_angle(lane)) per ground-truth lane (0 past the last)
  per_image     [N, 3] f64 LaneEval.bench of each row; file [3] f64 LaneEval.bench_one_submit of the whole file
  n_edge        number of hand-built rows at the end
"""
import argparse
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

S = 56
H = list(range(160, 720, 10))


def install_eval_lane():
    """Copy the reference's eval_lane.py verbatim into oracle/_ref/ (git-ignored), next to the modules
    reference_import.install() copies there, so tools/bench_test_eval.py can time the reference's own scorer where the
    checkout is absent.  Called by __graft_entry__.build(); no-op (False) when the checkout is absent or unreadable."""
    import shutil
    from oracle import reference_import as ri
    src = os.path.join(ri.SOURCE_ROOT, "Backprojection_Loss", "eval_lane.py")
    if not os.access(src, os.R_OK):
        return False
    dst = os.path.join(ri.INSTALLED_ROOT, "Backprojection_Loss", "eval_lane.py")
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    shutil.copyfile(src, dst)
    return True


def load_lane_eval():
    """The reference's LaneEval class, imported unmodified; its `import ujson as json` gets the standard json module."""
    from oracle import reference_import as ri
    path = os.path.join(ri.REFERENCE_ROOT, "Backprojection_Loss", "eval_lane.py")
    sys.modules.setdefault("ujson", types.SimpleNamespace(loads=json.loads, dumps=json.dumps))
    spec = importlib.util.spec_from_file_location("_ref_eval_lane", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.LaneEval


def label_rows(n, seed):
    from oracle import reference_import as ri
    rows = []
    for name in ("label_data_0531.json", "label_data_0601.json"):
        with open(os.path.join(ri.REFERENCE_ROOT, "Backprojection_Loss", "Labels", name)) as f:
            rows += [json.loads(line) for line in f if line.strip()]
    rows = [{"raw_file": r["raw_file"], "lanes": r["lanes"], "h_samples": r["h_samples"]} for r in rows
            if len(r["h_samples"]) == S and 2 <= len(r["lanes"]) <= 5]
    pick = np.sort(np.random.default_rng(seed).choice(len(rows), n, replace=False))
    return [rows[i] for i in pick]


def predict(rows, seed):
    """Seeded predictions near the ground truth: each predicted lane follows one ground-truth lane with 2-40 px of noise
    (continued linearly past its labelled samples), or is a random straight line; heads mostly on."""
    rng = np.random.default_rng(seed)
    N = len(rows)
    x_cal = np.empty((N, 4, S))
    y = np.asarray(H, np.float64)
    for i, r in enumerate(rows):
        for p in range(4):
            if p < len(r["lanes"]) and rng.random() < 0.85:
                g = np.asarray(r["lanes"][p], np.float64)
                ok = g >= 0
                if ok.sum() >= 2:
                    k, c = np.polyfit(y[ok], g[ok], 1)
                    base = np.where(ok, g, k * y + c)
                else:
                    base = rng.uniform(0, 1280) + 0 * y
                x_cal[i, p] = base + rng.normal(0, rng.choice([2., 6., 12., 40.]), S)
            else:
                x_cal[i, p] = rng.uniform(-200, 1500) + rng.uniform(-1.5, 1.5) * (y - 160)
    line_pred = (rng.random((N, 4)) < 0.85).astype(np.float32)
    horizon_pred = (rng.integers(8, 40, N) * 10).astype(np.int32)
    return x_cal, line_pred, horizon_pred


def edge_rows():
    """Hand-built rows: (gt row, x_cal [4, 56], line_pred [4], horizon)."""
    out = []
    on =np.ones(4, np.float32)

    def row(name, lanes):
        return {"raw_file": "edge/%s.jpg" % name, "lanes": [list(map(int, l)) for l in lanes], "h_samples": H}

    def far():
        return np.full(S, 3000.0)

    # |pred - gt| exactly 20 against a vertical lane (threshold exactly 20): not a hit; 19 is
    g0, g1, g2 = np.full(S, 600), np.full(S, 300), np.full(S, 900)
    x = np.stack([np.where(np.arange(S) < 40, 620.0, 581.0), g1 - 20.0, g2 + 19.0, far()])
    out.append((row("thresh20", [g0, g1, g2]), x, on, 160))
    # slope exactly 0.75 on every other row (threshold 20 / cos(arctan(0.75)) = 25): |diff| 25 and 24
    s75 = np.where(np.arange(S) % 2 == 0, 200 + 15 * (np.arange(S) // 2), -2)
    x = np.stack([np.where(s75 >= 0, s75 + 25.0, -2.0), np.where(s75 >= 0, s75 - 24.0, -2.0), g1 + 0.0, far()])
    out.append((row("thresh25", [s75, s75, g1]), x, on, 160))
    # clipping before rounding, and round half to even
    vals = [1279.3, 1279.49, 1279.5, 1279.0, 1278.5, -0.5, -0.4, -0.01, 0.0, 0.49, 0.5, 1.5, 2.5, 100.5, 101.5, 102.5]
    edge = np.full(S, 640.0)
    edge[:len(vals)] = vals
    x = np.stack([edge, np.full(S, 640.5), np.full(S, 641.5), np.full(S, 300.0)])
    out.append((row("round", [np.full(S, 640), np.full(S, 641)]), x, on, 160))
    # a lane switched off by the line-type head (head order: lane j reads line_pred[[1, 2, 0, 3][j]]) and one by half
    x = np.stack([g0 + 1.0, g1 + 1.0, g2 + 1.0, far()])
    out.append((row("gated", [g0, g1, g2]), x, np.asarray([1, 0, 1, 1], np.float32), 160))
    out.append((row("gated2", [g0, g1, g2]), x, np.asarray([0, 1, 1, 0], np.float32), 160))
    # horizon below 160, between rows, and past 720 (every sample cut)
    for h in (80, 155, 165, 175, 300, 800):
        out.append((row("horizon%d" % h, [g0, g1, g2]), np.stack([g0 + 3.0, g1 + 3.0, g2 + 3.0, far()]), on, h))
    # an all -2 ground-truth lane
    out.append((row("gt_missing", [g0, np.full(S, -2), g1]), np.stack([g0 + 3.0, np.full(S, -7.0), far(), far()]), on, 160))
    # G = 0 and G = 1: LaneEval's early return (0, 0, 1)
    out.append((row("g0", []), np.stack([g0 + 0.0] * 4), on, 160))
    out.append((row("g1", [g0]), np.stack([g0 + 0.0] * 4), on, 160))
    # G = 5: min removal; with a miss (fn > 0 is decremented) and all matched
    five = [np.full(S, 100 + 250 * k) for k in range(5)]
    out.append((row("g5_miss", five), np.stack([five[0] + 1.0, five[1] + 1.0, five[2] + 1.0, five[3] + 1.0]), on, 200))
    x = np.stack([five[0] + 1.0, five[1] + 1.0, five[2] + 1.0, five[3] + 1.0])
    x[3, :50] = five[4][:50]                # lane 3 covers gt lane 4 on most rows, gt lane 3 on the rest
    out.append((row("g5_partial", five), x, on, 160))
    # six lanes (the table holds 8)
    six = [np.full(S, 100 + 200 * k) for k in range(6)]
    out.append((row("g6", six), np.stack([six[0] + 2.0, six[2] - 2.0, six[4] + 0.0, six[5] + 30.0]), on, 160))
    # no match at all
    out.append((row("nomatch", [g0, g1, g2]), np.stack([g0 + 60.0, g1 - 80.0, far(), far()]), on, 160))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=290)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "tusimple_eval.npz"))
    a = ap.parse_args()
    import torch
    from lanedetection_end2end_b200.inference import lanes_from_predictions, write_tusimple_predictions
    LaneEval = load_lane_eval()
    rows = label_rows(a.rows, a.seed)
    x_cal, line_pred, horizon_pred = predict(rows, a.seed + 1)
    edges = edge_rows()
    rows += [e[0] for e in edges]
    x_cal = np.concatenate([x_cal, np.stack([e[1] for e in edges])])
    line_pred = np.concatenate([line_pred, np.stack([e[2] for e in edges])])
    horizon_pred = np.concatenate([horizon_pred, np.asarray([e[3] for e in edges], np.int32)])
    N = len(rows)
    lanes = lanes_from_predictions(torch.from_numpy(x_cal), torch.from_numpy(line_pred), torch.from_numpy(horizon_pred))
    thresh = np.zeros((N, 8))
    per_image = np.zeros((N, 3))
    for i, r in enumerate(rows):
        for j, lane in enumerate(r["lanes"]):
            thresh[i, j] = LaneEval.pixel_thresh / np.cos(LaneEval.get_angle(np.array(lane), np.array(r["h_samples"])))
        per_image[i] = LaneEval.bench(lanes[i], r["lanes"], r["h_samples"], 20)
    gt_text = "".join(json.dumps(r) + "\n" for r in rows)
    with tempfile.TemporaryDirectory() as d:
        gt_file, pred_file = os.path.join(d, "gt.json"), os.path.join(d, "pred.json")
        with open(gt_file, "w") as f:
            f.write(gt_text)
        with open(pred_file, "w") as f:
            write_tusimple_predictions(f, rows, lanes, 0)
        file_triple = np.asarray(LaneEval.bench_one_submit(pred_file, gt_file), np.float64)
    np.savez_compressed(a.out, gt_jsonl=np.frombuffer(gt_text.encode(), np.uint8), x_cal=x_cal, line_pred=line_pred,
                        horizon_pred=horizon_pred, lanes=np.asarray(lanes, np.int32), thresh=thresh, per_image=per_image,
                        file_triple=file_triple, n_edge=np.int64(len(edges)))
    print("wrote %s: %d rows (%d hand-built), file triple %s, %.1f kB" % (a.out, N, len(edges), file_triple.tolist(),
                                                                          os.path.getsize(a.out) / 1024))


if __name__ == "__main__":
    main()
