"""engine.train_epoch / inference.validate without a GPU: the argument checks, the lf_seg_lane_maps_line prototype and its
kernel's register use."""
import os
import re
import shutil
import subprocess
import types

import pytest
import torch

from lanedetection_end2end_b200 import _capi, engine, inference
from lanedetection_end2end_b200.Networks import utils as nu
from lanedetection_end2end_b200.optim import FusedOptimizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args(*extra):
    return nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "3",
                                        "--loss_policy", "backproject"] + list(extra))


class _Model(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(3))
        self.lsq_status = torch.zeros(1, dtype=torch.int32)
        self.defer_status_check = False


class _Graphed:
    """Stands in for GraphedInference / GraphedTrainStep: static inputs, a replay that does nothing."""

    def __init__(self, model, x, *a, **kw):
        self.x = x.clone()
        self.gt_line = torch.zeros(x.shape[0], 4)
        self.graph = types.SimpleNamespace(replay=lambda: None)
        self.out = self.post_out = None

    def __call__(self):
        return None


class _GraphedStep(_Graphed):
    def __init__(self, model, criterion, nclasses, x, *a, **kw):
        super().__init__(model, x)


def _batch(n, valid=False):
    b = [torch.zeros(n, 3, 8, 16), torch.zeros(n, 8, 16, dtype=torch.long), torch.zeros(n, 4, 56, dtype=torch.float64),
         torch.arange(n), torch.zeros(n, 4), torch.zeros(n, 8), torch.zeros(n, 4, 56, dtype=torch.float64)]
    if valid:
        b.insert(6, torch.arange(n))
    return tuple(b)


def test_train_epoch_needs_the_fused_optimizer():
    model = _Model()
    with pytest.raises(TypeError, match="FusedOptimizer"):
        engine.train_epoch([], model, torch.optim.Adam(model.parameters()), None, None, None, None, _args(), 0)


def test_train_epoch_refuses_pretrained():
    model = _Model()
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    with pytest.raises(ValueError, match="pretrained"):
        engine.train_epoch([], model, opt, None, None, None, None, _args("--pretrained", "True"), 0)


def test_a_later_batch_larger_than_the_first_raises(monkeypatch):
    monkeypatch.setattr(engine, "GraphedInference", _Graphed)
    monkeypatch.setattr(engine, "GraphedTrainStep", _GraphedStep)
    model = _Model()
    with pytest.raises(ValueError, match="batch of 3 images after a first batch of 2"):
        inference.validate([_batch(2, True), _batch(3, True)], model, None, None, None, None, _args())
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    with pytest.raises(ValueError, match="batch of 3 images after a first batch of 2"):
        engine.train_epoch([_batch(2), _batch(3)], model, opt, None, None, None, None, _args(), 0)
    assert model.defer_status_check is False


@pytest.mark.parametrize("loop", ["validate_bev", "skip_epoch"])
def test_other_loops_refuse_a_later_batch_of_another_size(monkeypatch, loop):
    """validate_bev refuses a larger later batch; the --pretrained skip epoch (epoch 0 < skip_epochs) any other size."""
    monkeypatch.setattr(engine, "GraphedInference", _Graphed)
    monkeypatch.setattr(engine, "GraphedTrainStep", _GraphedStep)
    model = _Model()
    if loop == "validate_bev":
        with pytest.raises(ValueError, match="batch of 3 images after a first batch of 2"):
            inference.validate_bev([_batch(2), _batch(3)], model, None, None, None, None, None,
                                   _args("--nclasses", "2", "--order", "2", "--loss_policy", "area"))
    else:
        opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0, per_param_step=True)
        for n in (1, 3):
            with pytest.raises(ValueError, match="batch of %d images after a first batch of 2" % n):
                engine.train_epoch([_batch(2), _batch(n)], model, opt, None, None, None, None,
                                   _args("--pretrained", "True"), 0)
    assert model.defer_status_check is False


def test_seg_lane_maps_line_prototype_matches_header():
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_seg_lane_maps", "lf_seg_lane_maps_line"):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(_capi.PROTOTYPES[name][1]) == len(decl.split(",")), name
        assert hasattr(_capi.lib(), name)


def test_seg_lane_maps_kernel_does_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "seg.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
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
    seg = [k for k in found if "seg_lane_maps_kernel" in k]
    assert len(seg) == 1, sorted(found)
    assert found[seg[0]] == (0, 0), found
