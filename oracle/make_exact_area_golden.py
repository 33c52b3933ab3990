"""Golden fixture of the bird's-eye-view exact-area metric: `python -m oracle.make_exact_area_golden`
-> tests/golden/bev_exact_area.npz.  TEST INFRASTRUCTURE; needs the reference checkout (oracle/reference_import.py).

It runs the reference's own `polynomial` class (Birds_Eye_View_Loss/Loss_crit.py:12-35, imported unmodified) on the CPU
as BEV/main.py:273-280 calls it: polynomial(beta_l.cpu()) against polynomial(gt_l.cpu()) for lanes 0 and 1, the beta a
float32 [B, 3, 1] tensor as Net.forward returns it, the ground truth the loader's float32 params[:, l] [B, 3].

Contents, per case <c>:
  <c>/beta [B, 4, 3] float32, <c>/params [B, 4, 3] float32   the inputs (lanes 2 and 3 feed only the 4-lane loss tests)
  <c>/trap_left, <c>/trap_right, <c>/exact [B] float32        trapezoidal per lane and ((left + right) / 2)
  <c>/mean [] float32                                         ((left + right) / 2).mean(), torch's CPU mean
Cases: B = 1 (squeeze gives 0-d tensors), 3 and 32 of random coefficients at the loader's scale, lanes with all-zero and
partly zero ground truth, large and negative coefficients, identical curves, and exact zeros in the prediction."""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "bev_exact_area.npz")
SCALE = np.array([0.5, 0.5, 0.5], np.float64)      # coefficient scale of the normalised BEV curves


def _reference_polynomial():
    from oracle import reference_import as ri
    path = os.path.join(ri.REFERENCE_ROOT, "Birds_Eye_View_Loss", "Loss_crit.py")
    spec = importlib.util.spec_from_file_location("_ref_bev_loss_crit", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.polynomial


def cases():
    rng = np.random.default_rng(20261017)
    out = {}

    def rand(B, scale=SCALE):
        return (rng.normal(size=(B, 4, 3)) * scale).astype(np.float32)

    out["b1"] = (rand(1), rand(1))
    out["b3"] = (rand(3), rand(3))
    beta, gt = rand(32), rand(32)
    gt[3, 0] = 0.0                                   # absent lanes (all zero) and one zero coefficient
    gt[5, 1] = 0.0
    gt[7, :2, 1] = 0.0
    gt[9, 2:] = 0.0
    out["b32"] = (beta, gt)
    beta, gt = rand(8, np.array([40.0, 300.0, 2e3])), rand(8, np.array([40.0, 300.0, 2e3]))
    beta[:4] = -np.abs(beta[:4])                     # large and negative coefficients
    gt[4:] = -np.abs(gt[4:])
    out["large"] = (beta, gt)
    beta = rand(5)
    gt = beta.copy()                                 # identical curves: every difference is 0
    gt[4, 1] = beta[4, 1] * np.float32(1 + 2 ** -23)
    beta[2, 0] = 0.0                                 # exact zeros in the prediction
    beta[3, :2] = -0.0
    out["same"] = (beta, gt)
    return out


def main():
    polynomial = _reference_polynomial()
    out = {}
    for name, (beta, gt) in cases().items():
        b, g = torch.from_numpy(beta), torch.from_numpy(gt)
        with torch.no_grad():
            tl = polynomial(b[:, 0, :, None]).trapezoidal(polynomial(g[:, 0, :]))
            tr = polynomial(b[:, 1, :, None]).trapezoidal(polynomial(g[:, 1, :]))
            exact = (tl + tr) / 2
        assert tl.dtype == torch.float32 and tl.dim() == (0 if beta.shape[0] == 1 else 1)
        out[name + "/beta"], out[name + "/params"] = beta, gt
        out[name + "/trap_left"] = tl.reshape(-1).numpy()
        out[name + "/trap_right"] = tr.reshape(-1).numpy()
        out[name + "/exact"] = exact.reshape(-1).numpy()
        out[name + "/mean"] = exact.mean().numpy()
    np.savez_compressed(GOLDEN, **out)
    print("wrote", GOLDEN, sorted(out))


if __name__ == "__main__":
    main()
