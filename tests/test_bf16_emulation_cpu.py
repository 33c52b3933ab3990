"""What does bf16 rounding of the convolution operands do to the REFERENCE?  This test re-runs the oracle's fp32
restatement of the reference with every convolution's operands rounded to bf16 (nearest even, 8 significant bits) and fp32
accumulation -- the arithmetic of the bf16 convolution mode -- and checks that the curve coefficients move from the fp64
golden by as much as the bf16 mode's beta does on the H100 (tests/golden/bf16_accuracy_*.json)."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import inputs, lsq_oracle as lo, erfnet_oracle as eo
from conftest import GOLDEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bf16(t):
    """Round fp32 to bf16 (nearest even) and back."""
    if t is None or t.dtype != torch.float32:
        return t
    return t.bfloat16().float()


def normwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float((np.abs(a - b).max(-1) / np.abs(b).max(-1)).max())


@pytest.mark.parametrize("name", ["net_l2_d2", "net_l4_d3"])
def test_reference_with_bf16_convolutions_moves_as_much_as_our_bf16_mode(name, monkeypatch):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(g["meta"]))
    L, order, B = meta["L"], meta["order"], meta["B"]
    P_np = inputs.make_erfnet_params(3, L, seed=meta["param_seed"])
    x_np = inputs.make_images(B, 256, 512, seed=meta["image_seed"])
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=meta["target_seed"])
    grid = torch.from_numpy(np.load(os.path.join(GOLDEN, "lsq_bp_l2_d2.npz"))["grid0"])
    hg = np.load(os.path.join(GOLDEN, "homography.npz"))
    crit = lo.BackprojectionLoss(order, 256, M=hg["M_256"], M_inv=hg["Minv_256"])

    real_conv, real_convT = F.conv2d, F.conv_transpose2d

    class BF16F:                       # the oracle module's view of torch.nn.functional
        def __getattr__(self, k):
            return getattr(F, k)

        @staticmethod
        def conv2d(x, w, b=None, *a, **kw):
            return real_conv(_bf16(x), _bf16(w), b, *a, **kw)

        @staticmethod
        def conv_transpose2d(x, w, b=None, *a, **kw):
            return real_convT(_bf16(x), _bf16(w), b, *a, **kw)

    monkeypatch.setattr(eo, "F", BF16F())
    P = {k[4:]: torch.from_numpy(v).float() for k, v in P_np.items()}
    with torch.no_grad():
        loss, beta, dec, masked = eo.full_step(
            torch.from_numpy(x_np).float(), P, grid, order, L, lo.mask_rows(256, meta["mask_pct"]),
            torch.from_numpy(xgt_np), torch.from_numpy(valid_np), loss_obj=crit)
    err_bf16_ref = normwise(beta.numpy(), g["beta_f64"])
    err_fp32_ref = normwise(g["beta_f32"], g["beta_f64"])
    rec = {"case": name, "beta_normwise_err_reference_with_bf16_convs": err_bf16_ref,
           "beta_normwise_err_reference_fp32": err_fp32_ref}
    # the bf16 mode's beta error on the same golden inputs, measured on the H100
    # (tests/test_bf16_gpu.py::test_full_path_bf16_mode_accuracy)
    ours = json.load(open(os.path.join(ROOT, "tests", "golden", "bf16_accuracy_%s.json" % name)))["beta_normwise_err_bf16"]
    rec["beta_normwise_err_ours_bf16_mode_h100"] = ours
    print(rec)
    # same order of magnitude: neither is more than 8x the other
    assert ours <= 8 * err_bf16_ref and err_bf16_ref <= 8 * ours, rec
    assert err_bf16_ref > 10 * err_fp32_ref, rec
