"""Restatement of the TuSimple lane metric (LaneEval of BP/eval_lane.py) in plain Python, for the tests.

  threshold(xs, ys)              per ground-truth lane: 20 / cos(arctan(k)), k the least-squares slope of x over y through
                                 the samples with x >= 0 (0 below two of them), fitted as sklearn's LinearRegression does
                                 (centre both, then scipy.linalg.lstsq) so the value is LaneEval's to the bit
  bench(pred, gt, ys, run_time)  (accuracy, fp, fn) of one image
  bench_one_submit(pred, gt)     [accuracy, fp, fn] of a prediction file against a ground-truth file (paths or row lists)

Samples are compared as integers (a negative one counts as -100), a line accuracy is a hit count over the lane length, and
the sums run in lane / file order in float64, so the values are exact restatements, not approximations.
"""
import json

import numpy as np
import scipy.linalg

PIXEL_THRESH = 20
PT_THRESH = 0.85


def threshold(xs, ys):
    xs, ys = np.asarray(xs), np.asarray(ys)
    sel = xs >= 0
    if np.count_nonzero(sel) < 2:
        return PIXEL_THRESH / np.cos(0)
    a = ys[sel].astype(np.float64).reshape(-1, 1)
    b = xs[sel].astype(np.float64)
    slope = scipy.linalg.lstsq(a - a.mean(axis=0), b - b.mean(), cond=1e-6)[0][0]
    return PIXEL_THRESH / np.cos(np.arctan(slope))


def line_accuracy(pred, gt, thresh):
    hits = 0
    for p, g in zip(pred, gt):
        p = p if p >= 0 else -100
        g = g if g >= 0 else -100
        if abs(p - g) < thresh:
            hits += 1
    return hits / len(gt)


def bench(pred, gt, ys, run_time=20):
    if any(len(p) != len(ys) for p in pred):
        raise ValueError("a predicted lane does not have one sample per h_sample")
    if run_time > 200 or len(gt) + 2 < len(pred):
        return 0., 0., 1.
    best = []
    matched = fn = 0.
    for lane in gt:
        t = threshold(lane, ys)
        m = max((line_accuracy(p, lane, t) for p in pred), default=0.)
        best.append(m)
        if m >= PT_THRESH:
            matched += 1
        else:
            fn += 1
    fp = len(pred) - matched
    total = 0.
    for m in best:
        total += m
    if len(gt) > 4:
        if fn > 0:
            fn -= 1
        total -= min(best)
    den = max(min(4., len(gt)), 1.)
    return total / den, (fp / len(pred) if pred else 0.), fn / den


def _rows(x):
    if isinstance(x, str):
        with open(x) as f:
            return [json.loads(line) for line in f.readlines()]
    return list(x)


def bench_one_submit(pred, gt):
    pred, gt = _rows(pred), _rows(gt)
    if len(pred) != len(gt):
        raise ValueError("%d predictions for %d ground-truth rows" % (len(pred), len(gt)))
    by_name = {r["raw_file"]: r for r in gt}
    acc = fp = fn = 0.
    for r in pred:
        g = by_name[r["raw_file"]]
        a, p, n = bench(r["lanes"], g["lanes"], g["h_samples"], r["run_time"])
        acc += a
        fp += p
        fn += n
    num = len(by_name)
    return [acc / num, fp / num, fn / num]
