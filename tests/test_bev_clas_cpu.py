"""The bird's-eye-view --clas run without a GPU: the Net's state_dict against the reference's (tests/golden/bev_clas.npz,
oracle/make_bev_clas_golden.py), the argument checks, the validation score's ground-truth tables over 48- and
56-sample rows, and lf_bev_lane_score's declaration and register report."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from lanedetection_end2end_b200 import _capi, engine, inference
from lanedetection_end2end_b200.Networks import utils as nu


def _args(*extra):
    return nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--order", "2", "--loss_policy", "area",
                                        "--no_cuda"] + list(extra))


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "bev_clas.npz"))


def test_state_dict_keys_and_shapes_equal_the_reference(golden):
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    m = Net(_args("--nclasses", "4", "--clas", "True", "--batch_size", "2"))
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == json.loads(str(golden["net/keys"]))
    plain = Net(_args("--nclasses", "4", "--batch_size", "2"))
    assert not any(k.startswith(("line_classification.", "horizon_estimation.")) for k in plain.state_dict())


def test_argument_checks():
    engine.check_bev_args(_args("--nclasses", "4", "--clas", "True"))
    for extra in (("--nclasses", "2", "--clas", "True"), ("--nclasses", "4", "--clas", "True", "--end_to_end", "False")):
        with pytest.raises(ValueError, match="--clas"):
            engine.check_bev_args(_args(*extra))
    with pytest.raises(ValueError, match="--pretrained"):
        engine.check_bev_args(_args("--nclasses", "4", "--clas", "True", "--pretrained", "True"))


def _rows(golden):
    return [json.loads(line) for line in golden["score/rows_jsonl"].tobytes().decode().splitlines()]


def test_tables_over_48_and_56_sample_rows(golden):
    rows = _rows(golden)
    assert sorted({len(r["h_samples"]) for r in rows}) == [48, 56]
    s = inference.BevLaneScorer(rows, device="cpu")
    MS = _capi.TUSIMPLE_MAX_S
    assert s.gt_S.tolist() == [len(r["h_samples"]) for r in rows]
    assert s.gt_lanes.tolist() == [4] * len(rows)
    for i, r in enumerate(rows):
        S = len(r["h_samples"])
        assert s.h_samples[i, :S].tolist() == r["h_samples"] and not s.h_samples[i, S:MS].any()
        for j, lane in enumerate(r["lanes"]):
            assert s.gt_x[i, j, :S].tolist() == lane
            assert float(s.thresh[i, j]) == inference.lane_threshold(np.asarray(lane), r["h_samples"])
    # LaneEval.get_angle through sklearn's LinearRegression, where sklearn is installed
    sk = pytest.importorskip("sklearn.linear_model")
    lr = sk.LinearRegression()
    for i, r in enumerate(rows):
        ys = np.array(r["h_samples"])
        for j, lane in enumerate(r["lanes"]):
            xs = np.array(lane)
            theta = 0
            if (xs >= 0).sum() > 1:
                lr.fit(ys[xs >= 0][:, None], xs[xs >= 0])
                theta = np.arctan(lr.coef_[0])
            assert float(s.thresh[i, j]) == 20 / np.cos(theta)


def test_tables_refuse_malformed_rows(golden):
    rows = _rows(golden)
    bad = [dict(rows[0], lanes=rows[0]["lanes"][:3]), dict(rows[0], h_samples=list(range(65)), lanes=[[-2] * 65] * 4),
           dict(rows[0], lanes=[rows[0]["lanes"][0][:-1]] + rows[0]["lanes"][1:])]
    for b in bad:
        with pytest.raises(ValueError):
            inference.BevLaneScorer([b], device="cpu")
    with pytest.raises(ValueError, match="duplicate"):
        inference.BevLaneScorer([rows[0], rows[0]], device="cpu")


def test_prototype_matches_declaration_and_export():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+lf_bev_lane_score\s*\((.*?)\);", hdr, re.S)
    assert decl
    assert len(_capi.PROTOTYPES["lf_bev_lane_score"][1]) == len(decl.group(1).split(","))
    assert hasattr(_capi.lib(), "lf_bev_lane_score")


def test_score_kernels_do_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "tusimple.cu"), "-o",
                                             str(tmp_path / "k.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            found[name] = (int(m.group(1)), int(m.group(2)))
    for kernel in ("bev_lane_score_kernel", "tusimple_score_kernel"):
        k = [n for n in found if kernel in n]
        assert len(k) == 1, sorted(found)
        assert found[k[0]] == (0, 0), found


def test_finish_refuses_a_row_outside_the_validation_set(golden, tmp_path):
    rows = _rows(golden)
    s = inference.BevLaneScorer(rows, device="cpu")
    s.begin(4, 256)
    s.pos.fill_(2)
    s.row[:2] = torch.tensor([1, len(rows)])
    with pytest.raises(IndexError, match="outside the %d rows" % len(rows)):
        s.finish(str(tmp_path / "dst.json"), str(tmp_path / "ls.json"))
    assert not (tmp_path / "dst.json").exists()
    s.row[1] = 0
    s.scored[:2] = 1
    assert s.finish() is not None
