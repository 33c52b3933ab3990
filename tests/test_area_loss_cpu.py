"""lf_area_loss without a GPU: its host twin against the reference's Area_Loss (tests/golden/area_loss.npz) and the float64
oracle, its exact-area output and Loss_crit.polynomial against the reference's own polynomial (tests/golden/bev_exact_area.npz)
bit for bit; the prototype, the kernel's register use, and the refusals of fused_area_loss, train_epoch_bev and
validate_bev."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from lanedetection_end2end_b200 import _capi, engine, inference
from lanedetection_end2end_b200.Loss_crit import AREA_WEIGHTS, fused_area_loss, polynomial
from lanedetection_end2end_b200.Networks import utils as nu
from lanedetection_end2end_b200.optim import FusedOptimizer
from oracle import lsq_oracle as lo

T = 0.7


def host(beta, params, wf, L):
    """lf_area_loss_host -> (loss, dbeta [B, L, 3], exact [B], exact_mean), float32."""
    beta, params = np.ascontiguousarray(beta, np.float32), np.ascontiguousarray(params, np.float32)
    B = beta.shape[0]
    loss, mean = np.zeros(1, np.float32), np.zeros(1, np.float32)
    dbeta, exact = np.zeros((B, L, 3), np.float32), np.zeros(B, np.float32)
    rc = _capi.lib().lf_area_loss_host(beta.ctypes.data, params.ctypes.data, B, L, AREA_WEIGHTS.get(wf, 7), loss.ctypes.data,
                                       dbeta.ctypes.data, exact.ctypes.data, mean.ctypes.data)
    return rc, loss[0], dbeta, exact, mean[0]


def moments(wf):
    k = np.arange(5.0)
    m = T ** (k + 1) / (k + 1)
    if wf == "linear":
        m -= T ** (k + 2) / (k + 2)
    elif wf == "quadratic":
        m -= T ** (k + 1.5) / (k + 1.5)
    return m


def abs_terms(beta, gt, wf):
    """sum over the present images, divided by their count, of sum_ij |Q_ij d_i d_j|: the scale of the float64 sum."""
    m, p = moments(wf), np.array([2, 1, 0])
    d = beta.astype(np.float64) - gt.astype(np.float64)
    present = (gt != 0).all(1)
    if not present.any():
        return 0.0
    t = np.abs(d[:, :, None] * d[:, None, :] * m[p[:, None] + p[None, :]]).sum((1, 2))
    return float(t[present].sum() / present.sum())


@pytest.mark.parametrize("wf", sorted(AREA_WEIGHTS))
def test_host_twin_against_reference_golden_and_float64_oracle(wf):
    """The golden's case in one lane of a 2- and of a 4-lane batch, the other lanes absent or random: the value and the
    gradient within one float32 rounding plus 1e-12 of the sum of |terms| of the float64 oracle on the same float32 inputs,
    and within 2e-6 of the reference's own float32 and float64 runs (area_loss.npz)."""
    g = np.load(os.path.join(GOLDEN, "area_loss.npz"))
    beta1 = g["params"][:, :, 0].astype(np.float32)
    gt1 = g["gt"].astype(np.float32)
    B = beta1.shape[0]
    rng = np.random.default_rng(3)
    for L, lane in ((2, 0), (2, 1), (4, 2), (4, 3)):
        beta = (rng.normal(size=(B, L, 3)) * 0.3).astype(np.float32)
        params = np.zeros((B, 4, 3), np.float32)
        beta[:, lane], params[:, lane] = beta1, gt1
        if L == 4:
            params[:, 0] = (rng.normal(size=(B, 3)) * 0.3).astype(np.float32)
        rc, loss, dbeta, _, _ = host(beta, params, wf, L)
        assert rc == 0
        b64 = torch.from_numpy(beta.astype(np.float64)).requires_grad_(True)
        ref = sum(lo.area_loss(b64[:, l], torch.from_numpy(params[:, l].astype(np.float64)), 2, wf) for l in range(L))
        ref.backward()
        scale = sum(abs_terms(beta[:, l], params[:, l], wf) for l in range(L))
        assert abs(float(loss) - float(ref.detach())) <= 2 ** -24 * abs(float(ref.detach())) + 1e-12 * scale, (L, lane)
        gr = b64.grad.numpy()
        assert np.all(np.abs(dbeta - gr) <= 2 ** -24 * np.abs(gr) + 1e-12 * scale), (L, lane)
        assert not dbeta[:, 1 if L == 2 and lane == 0 else 0 if L == 2 else 1].any()    # absent lane: no gradient
        # the golden lane alone against the reference's own runs
        lane_only = lo.area_loss(torch.from_numpy(beta1.astype(np.float64)), torch.from_numpy(gt1.astype(np.float64)), 2, wf)
        for variant in ("Ba", "Bi"):
            for tag in ("f32", "f64"):
                want = float(g["%s/o2_%s_%s/loss" % (variant, wf, tag)])
                assert abs(float(lane_only) - want) <= 2e-6 * abs(want)
                wg = g["%s/o2_%s_%s/grad" % (variant, wf, tag)][:, :, 0]
                assert np.abs(dbeta[:, lane] - wg).max() <= 2e-6 * np.abs(wg).max(), (variant, tag)


def test_host_twin_no_lane_present_gives_zero():
    g = np.load(os.path.join(GOLDEN, "area_loss.npz"))
    beta = np.repeat(g["params"][:, None, :, 0], 2, 1).astype(np.float32)
    rc, loss, dbeta, _, _ = host(beta, np.zeros((6, 4, 3), np.float32), "none", 2)
    assert rc == 0 and loss == 0.0 == float(g["Bi/all_absent"]) and not dbeta.any()


def test_exact_area_bit_identical_to_reference_polynomial():
    """The host twin's per-image exact values and Loss_crit.polynomial against the reference's own polynomial, bit for bit;
    the batch mean within B 2^-24 of torch's .mean()."""
    z = np.load(os.path.join(GOLDEN, "bev_exact_area.npz"))
    cases = sorted({k.split("/")[0] for k in z.files})
    assert {"b1", "b32", "large", "same"} <= set(cases)
    for case in cases:
        beta, params = z[case + "/beta"], z[case + "/params"]
        B = beta.shape[0]
        for L in (2, 4):
            rc, _, _, exact, mean = host(beta[:, :L], params, "none", L)
            assert rc == 0 and exact.tobytes() == z[case + "/exact"].tobytes(), (case, L)
            want = float(z[case + "/mean"])
            assert abs(float(mean) - want) <= B * 2 ** -24 * abs(want), case
        b, p = torch.from_numpy(beta), torch.from_numpy(params)
        for l, key in ((0, "trap_left"), (1, "trap_right")):
            t = polynomial(b[:, l, :, None]).trapezoidal(polynomial(p[:, l]))
            assert t.dim() == (0 if B == 1 else 1)
            assert t.reshape(-1).numpy().tobytes() == z["%s/%s" % (case, key)].tobytes(), (case, l)


def test_area_loss_refuses_bad_arguments():
    beta, params = np.zeros((2, 4, 3), np.float32), np.ones((2, 4, 3), np.float32)
    assert host(beta[:, :3], params, "none", 3)[0] == _capi.lib().lf_area_loss_host(
        beta.ctypes.data, params.ctypes.data, 2, 3, 0, None, None, None, None) == -1
    assert host(beta[:, :1], params, "none", 1)[0] == -1
    assert host(beta, params, "cubic", 4)[0] == -1
    assert _capi.lib().lf_area_loss_host(beta.ctypes.data, params.ctypes.data, 0, 2, 0, None, None, None, None) == -1
    assert _capi.lib().lf_area_loss_host(None, params.ctypes.data, 2, 2, 0, None, None, None, None) == -1


def test_fused_area_loss_refusals():
    b = [torch.zeros(2, 3, 1)] * 2
    p = torch.ones(2, 4, 3)
    with pytest.raises(ValueError, match="weight_funct"):
        fused_area_loss(b, p, "cubic")
    with pytest.raises(ValueError, match="2 or 4 lanes"):
        fused_area_loss(b * 2 + b[:1], p, "none")
    with pytest.raises(ValueError, match="order 2"):
        fused_area_loss([torch.zeros(2, 2, 1)] * 2, p, "none")
    with pytest.raises(_capi.LanefitError, match="CUDA"):
        fused_area_loss(b, p, "none")


def test_area_loss_prototype_matches_header():
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_area_loss", "lf_area_loss_host"):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(_capi.PROTOTYPES[name][1]) == len(decl.split(",")), name
        assert hasattr(_capi.lib(), name)


def test_area_loss_kernel_does_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "loss.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            found[name] = tuple(int(x) for x in m.groups())
    area = [k for k in found if "area_loss_kernel" in k]
    assert len(area) == 1, sorted(found)
    assert found[area[0]] == (0, 0, 0), found


def test_bev_main_imports_resolve():
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, 'lanedetection_end2end_b200/bev'); "
                        "from Loss_crit import define_loss_crit, polynomial, fused_area_loss"], cwd=ROOT,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# refusals of the loops (before any device work)

def _args(*extra):
    return nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "2", "--order", "2",
                                        "--loss_policy", "area"] + list(extra))


class _Model(torch.nn.Module):
    takes_gt_line = False

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(3))
        self.lsq_status = torch.zeros(1, dtype=torch.int32)
        self.defer_status_check = False


class _GraphedStep:
    def __init__(self, model, criterion, nclasses, x, *a, **kw):
        self.x = x.clone()

    def __call__(self):
        return None


def _batch(n):
    return (torch.zeros(n, 3, 8, 16), torch.zeros(n, 1, 8, 16, dtype=torch.long), torch.ones(n, 4, 3), torch.arange(n),
            torch.zeros(n, 4), torch.zeros(n, 8))


REFUSED = [(("--clas", "True"), "--clas"), (("--pretrained", "True"), "--pretrained"), (("--loss_policy", "mse"), "mse"),
           (("--order", "1"), "order 1"), (("--weight_funct", "cubic"), "cubic"),
           (("--nclasses", "4", "--end_to_end", "False"), "needs 2 lanes")]


@pytest.mark.parametrize("extra,reason", REFUSED, ids=[r for _, r in REFUSED])
def test_loops_refuse_unsupported_settings(extra, reason):
    model = _Model()
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    with pytest.raises(ValueError, match=re.escape(reason)):
        engine.train_epoch_bev([], model, opt, None, None, None, None, _args(*extra), 0)
    with pytest.raises(ValueError, match=re.escape(reason)):
        inference.validate_bev([], model, None, None, None, None, None, _args(*extra))


def test_train_epoch_bev_needs_the_fused_optimizer():
    model = _Model()
    with pytest.raises(TypeError, match="FusedOptimizer"):
        engine.train_epoch_bev([], model, torch.optim.Adam(model.parameters()), None, None, None, None, _args(), 0)


def test_train_epoch_bev_refuses_a_later_batch_of_another_size(monkeypatch):
    monkeypatch.setattr(engine, "GraphedTrainStep", _GraphedStep)
    model = _Model()
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    for n in (1, 3):
        with pytest.raises(ValueError, match="batch of %d images after a first batch of 2" % n):
            engine.train_epoch_bev([_batch(2), _batch(n)], model, opt, None, None, None, None, _args(), 0)
    assert model.defer_status_check is False
