#!/usr/bin/env python
"""End-to-end training smoke: the loop of BP/main.py:239-340 (zero_grad -> model -> per-lane backprojection loss -> backward ->
optimizer.step, RuntimeError on a singular system skips the batch) on a fixed synthetic batch whose ground truth is a pair of
straight lanes -- the loss must go down.  Uses the reference-facing modules only (define_args / Net / define_loss_crit /
define_optim / define_init_weights), i.e. what a user of the reference would run after switching packages.

    python tools/train_synthetic.py [--steps 40] [--batch 4]        # prints one JSON line
"""
import argparse
import contextlib
import io
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def synthetic_batch(B, device, seed=0):
    """Images with two bright, slightly slanted stripes on noise + the x positions of those stripes at the 56 TuSimple rows
    (in 256x512 network coordinates), valid from sample 8 on (BP/Dataloader/Load_Data_new.py:140-141)."""
    g = torch.Generator().manual_seed(seed)
    H, W = 256, 512
    yy = torch.arange(H).view(1, H, 1).float()
    xx = torch.arange(W).view(1, 1, W).float()
    c = torch.tensor([180.0, 330.0]).view(2, 1, 1) + 20 * (torch.rand(B, 2, 1, 1, generator=g) - 0.5)
    s = torch.tensor([-0.45, 0.45]).view(2, 1, 1) + 0.1 * (torch.rand(B, 2, 1, 1, generator=g) - 0.5)
    centre = c + s * (yy - 128)                                           # [B, 2, H, 1]
    stripes = torch.exp(-0.5 * ((xx - centre) / 5.0) ** 2).sum(1)         # [B, H, W]
    img = (0.2 * torch.rand(B, 3, H, W, generator=g) + 0.8 * stripes.unsqueeze(1)).clamp(0, 1)
    rows = ((torch.arange(160, 720, 10) - 80).float() / 2.5)              # image rows of the h_samples
    x_gt = torch.zeros(B, 4, 56, dtype=torch.float64)
    x_gt[:, :2] = (c.view(B, 2, 1) + s.view(B, 2, 1) * (rows.view(1, 1, 56) - 128)).double()
    valid = torch.ones(B, 4, 56, dtype=torch.float64)
    valid[:, :, :8] = 0
    return img.to(device), x_gt.to(device), valid.to(device)


def run(steps=40, batch=4, lr=1e-3, seed=0, device="cuda", fused=False, graphed=False):
    """fused: the library's Adam (optim.FusedOptimizer) instead of torch.optim.Adam.  graphed (needs fused): the whole
    iteration, update included, as one CUDA graph replay per step (engine.GraphedTrainStep); a skipped step is counted
    from the optimizer's device counter once at the end."""
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args, define_init_weights, define_optim
    from lanedetection_end2end_b200.Loss_crit import define_loss_crit
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "2", "--order", "2", "--batch_size", str(batch),
                                     "--loss_policy", "backproject", "--end_to_end", "True"])
    torch.manual_seed(seed)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")
    model = model.to(device).train()
    criterion, _ = define_loss_crit(args)
    optimizer = define_optim("adam", model.parameters(), lr, 0, fused=fused or graphed)
    x, x_gt, valid = synthetic_batch(batch, device, seed)
    gt_line = torch.zeros(batch, 4)
    if graphed:
        from lanedetection_end2end_b200.engine import GraphedTrainStep
        step = GraphedTrainStep(model, criterion, 2, x, x_gt, valid, optimizer=optimizer)
        losses = [step().clone() for _ in range(steps)]
        losses = [float(v) for v in losses]
        return {"steps": steps, "batch": batch, "skipped": optimizer.skipped, "loss_first": losses[0], "loss_last": losses[-1],
                "loss_min": min(losses), "losses": [round(v, 2) for v in losses]}
    losses, skipped = [], 0
    for _ in range(steps):
        optimizer.zero_grad()
        try:
            beta0, beta1 = model(x, gt_line, True)[:2]
        except RuntimeError:                      # singular normal matrix: the reference skips the batch (main.py:289-292)
            skipped += 1
            continue
        loss = (criterion(beta0, x_gt[:, 0], valid[:, 0])[0] + criterion(beta1, x_gt[:, 1], valid[:, 1])[0]) / 2
        loss.backward()
        optimizer.step()
        losses.append(float(loss))
    return {"steps": steps, "batch": batch, "skipped": skipped, "loss_first": losses[0], "loss_last": losses[-1],
            "loss_min": min(losses), "losses": [round(v, 2) for v in losses]}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--fused-optim", action="store_true", help="step with the library's fused Adam kernel")
    ap.add_argument("--graphed", action="store_true", help="one CUDA graph replay per iteration (implies --fused-optim)")
    a = ap.parse_args()
    print(json.dumps(run(a.steps, a.batch, fused=a.fused_optim, graphed=a.graphed)))
