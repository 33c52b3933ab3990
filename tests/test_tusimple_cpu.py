"""Host side of the TuSimple scorer (inference.lane_threshold, TuSimpleScorer's ground-truth checks, test_model's argument
checks) and the metric's oracle restatement, against the reference LaneEval's values in tests/golden/tusimple_eval.npz
(oracle/make_tusimple_golden.py)."""
import json
import os
import types

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import tusimple_oracle as to
from lanedetection_end2end_b200 import inference

H = list(range(160, 720, 10))


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "tusimple_eval.npz"))
    d = {k: z[k] for k in z.files}
    d["rows"] = [json.loads(line) for line in bytes(d["gt_jsonl"]).decode().splitlines()]
    return d


def _lanes(golden):
    for i, r in enumerate(golden["rows"]):
        for j, lane in enumerate(r["lanes"]):
            yield i, j, lane, r["h_samples"]


def test_fixture_covers_the_metric(golden):
    """The fixture exercises matched and unmatched lanes, the early return, the G > 4 rules and exact-threshold rows."""
    rows, pi = golden["rows"], golden["per_image"]
    G = np.asarray([len(r["lanes"]) for r in rows])
    assert len(rows) >= 300 and int(golden["n_edge"]) >= 15
    assert set(G.tolist()) >= {0, 1, 2, 3, 4, 5, 6}
    assert ((pi[:, 2] > 0) & (pi[:, 2] < 1)).sum() > 20 and (pi[:, 0] > 0.9).sum() > 20
    assert np.all(pi[G + 2 < 4] == [0., 0., 1.])
    assert 25.0 - 1e-9 < golden["thresh"][[i for i, r in enumerate(rows) if r["raw_file"] == "edge/thresh25.jpg"][0], 0] < 25.0 + 1e-9


def test_lane_threshold_is_lane_eval_bitwise(golden):
    th = golden["thresh"]
    for i, j, lane, h in _lanes(golden):
        assert inference.lane_threshold(lane, h) == th[i, j], (i, j)
        assert to.threshold(lane, h) == th[i, j], (i, j)


def test_lane_threshold_is_sklearn_bitwise(golden):
    sk = pytest.importorskip("sklearn.linear_model")
    lr = sk.LinearRegression()
    for i, j, lane, h in _lanes(golden):
        xs, ys = np.asarray(lane), np.asarray(h)
        xs, ys = xs[xs >= 0], ys[xs >= 0]
        theta = np.arctan(lr.fit(ys[:, None], xs).coef_[0]) if len(xs) > 1 else 0
        assert inference.lane_threshold(lane, h) == 20 / np.cos(theta), (i, j)


def test_oracle_reproduces_lane_eval(golden):
    rows, lanes = golden["rows"], golden["lanes"].tolist()
    for i, r in enumerate(rows):
        assert to.bench(lanes[i], r["lanes"], r["h_samples"], 20) == tuple(golden["per_image"][i]), i
    pred = [dict(r, lanes=lanes[i], run_time=20) for i, r in enumerate(rows)]
    assert to.bench_one_submit(pred, rows) == golden["file_triple"].tolist()


def test_host_gating_matches_fixture(golden):
    """lanes_from_predictions on the fixture's inputs gives the fixture's lanes (the fixture was written by it)."""
    import torch
    got = inference.lanes_from_predictions(torch.from_numpy(golden["x_cal"]), torch.from_numpy(golden["line_pred"]),
                                           torch.from_numpy(golden["horizon_pred"]))
    assert np.array_equal(np.asarray(got), golden["lanes"])


def _row(name, lanes, h=H):
    return {"raw_file": name, "lanes": lanes, "h_samples": h}


@pytest.mark.parametrize("rows, what", [
    ([_row("a.jpg", [[-2] * 48, [5] * 48], list(range(240, 720, 10)))], "48 h_samples"),
    ([_row("a.jpg", [[-2] * 56, [5] * 55])], "lane 1 has 55 samples"),
    ([_row("a.jpg", [[5] * 56] * 9)], "9 lanes"),
    ([_row("a.jpg", [[5] * 56]), _row("b.jpg", []), _row("a.jpg", [])], "duplicate raw_file"),
    ([_row("a.jpg", [[5.5] * 56])], "not int32"),
])
def test_scorer_rejects_ground_truth_lane_eval_cannot_score(rows, what):
    with pytest.raises(ValueError) as e:
        inference.TuSimpleScorer(rows, "cpu")
    assert "a.jpg" in str(e.value) and what in str(e.value)


def test_scorer_reads_a_ground_truth_file(golden, tmp_path):
    """Ground-truth tables built from a file equal LaneEval's thresholds and hold every lane (on the CPU: no launch)."""
    p = tmp_path / "test_label.json"
    p.write_bytes(bytes(golden["gt_jsonl"]))
    s = inference.TuSimpleScorer(str(p), "cpu")
    assert s.N == len(golden["rows"]) and s.rows == golden["rows"]
    assert np.array_equal(s.thresh.numpy(), golden["thresh"])
    assert s.gt_lanes.tolist() == [len(r["lanes"]) for r in golden["rows"]]
    for i, r in enumerate(golden["rows"]):
        assert s.gt_x[i, :len(r["lanes"])].tolist() == r["lanes"]


def _args(**kw):
    a = dict(end_to_end=True, clas=True, nclasses=4, draw_testset=False, test_dir="/nonexistent", save_path="/nonexistent")
    a.update(kw)
    return types.SimpleNamespace(**a)


@pytest.mark.parametrize("kw", [dict(end_to_end=False), dict(clas=False), dict(nclasses=2)])
def test_test_model_refuses_what_the_reference_cannot_score(kw):
    with pytest.raises(ValueError):
        inference.test_model([], None, None, None, None, None, _args(**kw))


def test_test_model_refuses_draw_testset():
    with pytest.raises(NotImplementedError):
        inference.test_model([], None, None, None, None, None, _args(draw_testset=True))
