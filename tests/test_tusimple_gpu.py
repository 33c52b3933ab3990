"""lf_tusimple_score (csrc/tusimple.cu) through inference.TuSimpleScorer, and inference.test_model end to end: the gated lanes
and LaneEval's (accuracy, fp, fn) equal the reference values exactly -- the golden LaneEval run of
tests/golden/tusimple_eval.npz, inference.lanes_from_predictions, and the oracle restatement of the metric."""
import io
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import inputs, tusimple_oracle as to
from lanedetection_end2end_b200 import inference

pytestmark = pytest.mark.gpu
H = list(range(160, 720, 10))


@pytest.fixture(scope="module")
def golden():
    z = np.load(os.path.join(GOLDEN, "tusimple_eval.npz"))
    d = {k: z[k] for k in z.files}
    d["rows"] = [json.loads(line) for line in bytes(d["gt_jsonl"]).decode().splitlines()]
    return d


def _inputs(golden):
    return (torch.from_numpy(golden["x_cal"]).cuda(), torch.from_numpy(golden["line_pred"]).cuda(),
            torch.from_numpy(golden["horizon_pred"]).cuda())


def _check_against_golden(s, golden):
    assert torch.equal(s.lanes.cpu(), torch.from_numpy(golden["lanes"]))
    assert torch.equal(s.per_image.cpu(), torch.from_numpy(golden["per_image"]))
    assert s.result() == golden["file_triple"].tolist()


def test_kernel_equals_lane_eval_over_uneven_batches(golden):
    """Every row of the fixture (edge cases included), scored in batches that split the file unevenly."""
    x, lp, hp = _inputs(golden)
    s = inference.TuSimpleScorer(golden["rows"], "cuda")
    N, start = len(golden["rows"]), 0
    for B in [37, 101, 1, 64, 9, 1000]:
        stop = min(start + B, N)
        s.score(x[start:stop], lp[start:stop], hp[start:stop])
        start = stop
    assert start == N
    _check_against_golden(s, golden)


def test_kernel_fixed_batch_with_stale_tail(golden):
    """A fixed batch of 64 whose last call holds real rows in its leading slots and stale rows after them: the stale slots
    past the end of the file are not scored; pos ends past N."""
    x, lp, hp = _inputs(golden)
    s = inference.TuSimpleScorer(golden["rows"], "cuda")
    N, B = len(golden["rows"]), 64
    sx, slp, shp = x[:B].clone(), lp[:B].clone(), hp[:B].clone()
    for start in range(0, N, B):
        n = min(B, N - start)
        sx[:n], slp[:n], shp[:n] = x[start:start + n], lp[start:start + n], hp[start:start + n]
        s.score(sx, slp, shp)
    assert int(s.pos.item()) == -(-N // B) * B
    _check_against_golden(s, golden)
    s.reset()
    s.score(sx, slp, shp)
    with pytest.raises(RuntimeError):
        s.result()


def test_kernel_gating_equals_host_path_on_projections(golden):
    """x_cal of Projections.compute_all on random betas (values crossing 0 and 1279, exact halves are rare but rounding
    and clipping are exercised), gated by the kernel, equals lanes_from_predictions on the same tensors."""
    from lanedetection_end2end_b200.Networks.utils import define_args
    B, order = 48, 3
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", str(order),
                                     "--batch_size", str(B)])
    proj = inference.Projections(args)
    g = torch.Generator().manual_seed(7)
    betas = [(torch.randn(B, order + 1, 1, generator=g, dtype=torch.float64) * torch.tensor([1e-6, 3e-4, 0.15, 120.0]).view(1, -1, 1)
              + torch.tensor([0, 0, 0, 256.0]).view(1, -1, 1)).cuda() for _ in range(4)]
    x_cal = proj.compute_all(betas)
    xc = x_cal.cpu()
    assert (xc < 0).any() and (xc > 1279).any() and ((xc >= 0) & (xc <= 1279)).float().mean() > 0.3
    line_pred = torch.randint(0, 2, (B, 4), generator=g).float().cuda()
    horizon_pred = (torch.randint(5, 85, (B,), generator=g) * 10).int().cuda()
    s = inference.TuSimpleScorer(golden["rows"][:B], "cuda")
    s.score(x_cal, line_pred, horizon_pred)
    assert s.predictions() == inference.lanes_from_predictions(x_cal, line_pred, horizon_pred)
    s.reset()
    s.score(x_cal)
    assert s.predictions() == inference.lanes_from_predictions(x_cal)


def test_graph_replays_equal_eager_calls(golden):
    x, lp, hp = _inputs(golden)
    N, B = len(golden["rows"]), 40
    eager = inference.TuSimpleScorer(golden["rows"], "cuda")
    graphed = inference.TuSimpleScorer(golden["rows"], "cuda")
    sx, slp, shp = x[:B].clone(), lp[:B].clone(), hp[:B].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graphed.score(sx, slp, shp)            # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.score(sx, slp, shp)
    graphed.reset()
    for k, start in enumerate(range(0, N, B)):
        n = min(B, N - start)
        sx[:n], slp[:n], shp[:n] = x[start:start + n], lp[start:start + n], hp[start:start + n]
        graph.replay()
        eager.score(sx, slp, shp)
        assert int(graphed.pos.item()) == (k + 1) * B
    assert torch.equal(graphed.lanes, eager.lanes) and torch.equal(graphed.per_image, eager.per_image)
    assert graphed.result() == eager.result() == golden["file_triple"].tolist()


def _clas_model(B):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "3", "--batch_size",
                                     str(B), "--clas", "1", "--end_to_end", "True"])
    torch.manual_seed(0)
    model = Net(args).cuda().eval()
    return model, args


def _eager_host_path(model, args, batches):
    """What the reference's test loop computes per batch, eagerly: forward, head ops, Projections, host gating."""
    proj = inference.Projections(args)
    lanes = []
    with torch.no_grad():
        for xb in batches:
            out = model(xb.cuda(), torch.zeros(xb.shape[0], 4), True)
            horizon_pred = torch.sigmoid(out[7]).sum(dim=1)
            horizon_pred = (torch.round((inference.resize_coordinates(horizon_pred) + 80) / 10) * 10).int()
            line_pred = torch.round(torch.sigmoid(out[6]))
            x_cal = proj.compute_all(out[:4])
            lanes += inference.lanes_from_predictions(x_cal, line_pred, horizon_pred)
    return lanes


def _ground_truth(lanes, seed):
    """Ground-truth rows near the model's own gated lanes: 3 px of noise (matched), 35-45 px shifts (unmatched), lanes
    dropped or added (2-5 lanes), samples outside the frame as -2."""
    rng = np.random.default_rng(seed)
    rows = []
    for i, img in enumerate(lanes):
        gt = []
        for lane in np.asarray(img, np.float64):
            if rng.random() < 0.15:
                continue
            shift = rng.choice([-45.0, 35.0]) if rng.random() < 0.3 else 0.0
            v = np.round(lane + shift + rng.normal(0, 3, lane.shape))
            v = np.where((lane >= 0) & (v >= 0) & (v <= 1279), v, -2).astype(np.int64)
            gt.append(v.tolist())
        if rng.random() < 0.15:
            gt.append((np.arange(56) * 3 + 700).tolist())
        while len(gt) < 2:
            gt.append([-2] * 56)
        rows.append({"raw_file": "clips/%d/20.jpg" % i, "lanes": gt, "h_samples": H})
    return rows


def test_test_model_end_to_end(tmp_path, capsys):
    """inference.test_model on a 70-image synthetic test set (batches 32, 32, 6) through a random-weight --clas 4-lane order-3
    model: the file is byte-identical to the eager host path's, the accuracy is LaneEval's (oracle) on that file, and a
    second call (cached scorer, new graph) writes the same file."""
    N, B = 70, 32
    model, args = _clas_model(B)
    images = torch.from_numpy(inputs.make_images(N, 256, 512, seed=31))
    batches = [images[i:i + B] for i in range(0, N, B)]
    lanes = _eager_host_path(model, args, batches)
    rows = _ground_truth(lanes, 5)
    with open(tmp_path / "test_label.json", "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    want = io.StringIO()
    inference.write_tusimple_predictions(want, rows, lanes, 0)
    want = want.getvalue()
    pred_rows = [json.loads(line) for line in want.splitlines()]
    acc_want = to.bench_one_submit(pred_rows, rows)
    per_image = [to.bench(p["lanes"], r["lanes"], H) for p, r in zip(pred_rows, rows)]
    assert any(b[1] < 1 for b in per_image) and any(b[2] > 0 for b in per_image), acc_want     # matched and missed lanes
    args.test_dir = args.save_path = str(tmp_path)
    out_file = tmp_path / "test_set_predictions.json"
    key = (os.path.abspath(str(tmp_path / "test_label.json")), str(next(model.parameters()).device))
    scorers = []
    for call in range(2):
        acc = inference.test_model(batches, model, None, None, None, None, args)
        assert out_file.read_text() == want, call
        assert acc == acc_want[0], call
        assert "===> Average ACC on TESTSET is" in capsys.readouterr().out
        out_file.unlink()
        scorers.append(inference._SCORERS[key][1])
    assert scorers[0] is scorers[1]
    assert model.defer_status_check is False
