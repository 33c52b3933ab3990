"""Epoch time of main.py's training loop and validation pass: eager as main.py writes them against engine.train_epoch and
inference.validate (one CUDA-graph replay per batch).  Writes profiles/h100/bench_epoch.json (or --out).

    python tools/bench_epoch.py [--out PATH] [--rounds 3]

Workload: the synthetic 3626-file TuSimple-shaped directory of tests/golden/loader_tusimple.npz (the one
tools/bench_loader.py times; 2,900 training and 726 validation samples), the train.sh model (4 lanes, order 3, --clas 1,
backprojection loss, mask 0.2, xavier init), batch 32, resize 256, loaded by the GPU loader with its device cache filled
before timing.  Arms, alternated --rounds times in one process, each a whole epoch or pass ended by a device synchronise:
  train_eager     BP/main.py:239-359 restated below (tqdm and plotting aside), torch.optim.Adam as define_optim builds it
  train_graphed   engine.train_epoch with define_optim(..., fused=True)
  valid_eager     BP/main.py:419-526 restated below
  valid_graphed   inference.validate
Each arm has its own model and optimizer, so the training arms keep training their own weights round after round."""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

BATCH, RESIZE = 32, 256


class AverageMeter:          # BP/Networks/utils.py AverageMeter
    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def eager_train(loader, model, optimizer, criterion, criterion_seg, criterion_line_class, criterion_horizon, args):
    """BP/main.py:239-340 (end-to-end branch) with main.py's synchronisations: the status check and loss.item()."""
    import torch
    losses = AverageMeter()
    model.train()
    for i, (input, gt, lanes, idx, gt_line, gt_horizon, valid_points) in enumerate(loader):
        input, lanes = input.cuda(), lanes.cuda()
        valid_points = valid_points.cuda()
        gt = gt.cuda().squeeze(1)
        gt0, gt1, gt2, gt3 = lanes[:, 0, :], lanes[:, 1, :], lanes[:, 2, :], lanes[:, 3, :]
        try:
            beta0, beta1, beta2, beta3, weightmap_zeros, \
                output_net, outputs_line, outputs_horizon, output_seg = model(input, gt_line, args.end_to_end, gt=gt)
        except RuntimeError as e:
            print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
            print(e)
            continue
        loss_left, x_cal0 = criterion(beta0, gt0, valid_points[:, 0])
        loss_right, x_cal1 = criterion(beta1, gt1, valid_points[:, 1])
        loss_left1, x_cal2 = criterion(beta2, gt2, valid_points[:, 2])
        loss_right1, x_cal3 = criterion(beta3, gt3, valid_points[:, 3])
        loss_left += loss_left1
        loss_right += loss_right1
        loss = (loss_left + loss_right) / args.nclasses
        gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
        loss_horizon = criterion_horizon(outputs_horizon, gt_horizon).double()
        loss_line = criterion_line_class(outputs_line, gt_line).double()
        loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
    return losses.avg


def eager_validate(loader, model, criterion, criterion_seg, criterion_line_class, criterion_horizon, args):
    """BP/main.py:419-526 (end-to-end --clas branch)."""
    import torch
    import torch.nn as nn
    losses, acc_hor_tot, acc_line_tot = AverageMeter(), AverageMeter(), AverageMeter()
    model.eval()
    with torch.no_grad():
        for i, (input, gt, lanes, idx, gt_line, gt_horizon, index, valid_points) in enumerate(loader):
            input, lanes = input.cuda(), lanes.cuda()
            input = input.float()
            valid_points = valid_points.cuda()
            gt = gt.cuda().squeeze(1)
            gt0, gt1, gt2, gt3 = lanes[:, 0, :], lanes[:, 1, :], lanes[:, 2, :], lanes[:, 3, :]
            try:
                beta0, beta1, beta2, beta3, weightmap_zeros, \
                    output_net, outputs_line, outputs_horizon, output_seg = model(input, gt_line, args.end_to_end, gt=gt)
            except RuntimeError as e:
                print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
                print(e)
                continue
            loss_left, x_cal0 = criterion(beta0, gt0, valid_points[:, 0])
            loss_right, x_cal1 = criterion(beta1, gt1, valid_points[:, 1])
            loss_left1, x_cal2 = criterion(beta2, gt2, valid_points[:, 2])
            loss_right1, x_cal3 = criterion(beta3, gt3, valid_points[:, 3])
            loss_left += loss_left1
            loss_right += loss_right1
            loss = (loss_left + loss_right) / args.nclasses
            losses.update(loss.item(), input.size(0))
            gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
            horizon_pred = torch.round(nn.Sigmoid()(outputs_horizon))
            acc = torch.eq(horizon_pred, gt_horizon)
            acc_hor = torch.sum(acc).float() / (args.resize * args.val_batch_size)
            acc_hor_tot.update(acc_hor.item())
            line_pred = torch.round(nn.Sigmoid()(outputs_line))
            acc = torch.eq(line_pred, gt_line)
            acc_line = torch.sum(acc).float() / (args.nclasses * args.val_batch_size)
            acc_line_tot.update(acc_line.item())
            loss_horizon = criterion_horizon(outputs_horizon, gt_horizon)
            loss_line = criterion_line_class(outputs_line, gt_line)
            loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
    return losses.avg, acc_hor_tot.avg, acc_line_tot.avg, 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_epoch.json"))
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import torch.nn as nn
    from bench_modes import gpu_info
    from oracle import make_loader_golden as mlg
    from lanedetection_end2end_b200 import engine, inference
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    from lanedetection_end2end_b200.Loss_crit import define_loss_crit
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args, define_init_weights, define_optim
    assert torch.cuda.is_available(), "bench_epoch.py times the GPU; there is no CPU fallback"
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--loss_policy", "backproject", "--weight_init",
                                     "xavier", "--split_percentage", "0.2", "--activation_layer", "square", "--nclasses", "4",
                                     "--mask_percentage", "0.20", "--order", "3", "--clas", "1", "--batch_size", str(BATCH),
                                     "--resize", str(RESIZE)])
    args.val_batch_size = BATCH
    rec = {"gpu": gpu_info(), "batch": BATCH, "resize": RESIZE,
           "model": "train.sh: 4 lanes, order 3, --clas 1, backprojection loss, mask 0.2, xavier init",
           "dataset": "synthetic 3626-file TuSimple-shaped directory (tests/golden/loader_tusimple.npz): 2,900 training "
                      "samples (90 batches), 726 validation samples (22 batches), GPU loader with a filled device cache"}
    z = np.load(os.path.join(ROOT, "tests", "golden", "loader_tusimple.npz"))
    with tempfile.TemporaryDirectory() as d:
        paths = mlg.from_fixture(z, d)
        args.save_path = d
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            train, valid, _ = L.get_loader(3626, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"],
                                           True, BATCH, BATCH, True, 0, True, RESIZE, 4, split_percentage=0.2,
                                           line_file=paths["line_file"])
        for loader in (train, valid):             # fill the cache
            for _ in loader:
                pass
        crits = (*define_loss_crit(args), nn.BCEWithLogitsLoss().cuda(), nn.BCEWithLogitsLoss().cuda())

        def model():
            torch.manual_seed(0)
            m = Net(args)
            with contextlib.redirect_stdout(io.StringIO()):
                define_init_weights(m, "xavier")
            return m.cuda()

        m_eager, m_graphed = model(), model()
        opt_eager = define_optim("adam", m_eager.parameters(), args.learning_rate, args.weight_decay, fused=False)
        opt_graphed = define_optim("adam", m_graphed.parameters(), args.learning_rate, args.weight_decay, fused=True)
        arms = {
            "train_eager": lambda e: eager_train(train, m_eager, opt_eager, *crits, args),
            "train_graphed": lambda e: engine.train_epoch(train, m_graphed, opt_graphed, *crits, args, e)[0],
            "valid_eager": lambda e: eager_validate(valid, m_eager, *crits, args)[0],
            "valid_graphed": lambda e: inference.validate(valid, m_graphed, *crits, args, e)[0],
        }
        res = {k: {"seconds": [], "loss_avg": []} for k in arms}
        for r in range(a.rounds):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                loss = fn(r)
                torch.cuda.synchronize()
                res[name]["seconds"].append(round(time.perf_counter() - t0, 3))
                res[name]["loss_avg"].append(loss)
                print(name, r, res[name]["seconds"][-1], loss, flush=True)
        for name, v in res.items():
            n = len(train) if name.startswith("train") else len(valid)
            v["median_s"] = statistics.median(v["seconds"])
            v["batches"] = n
            v["median_ms_per_batch"] = round(1e3 * v["median_s"] / n, 2)
        rec["arms"] = res
        rec["note"] = ("each round's epoch includes building the graphs of the graphed arms (warm-up and capture), as a "
                       "main.py epoch calling them would")
    from lanedetection_end2end_b200 import ops_net
    rec["conv_mode"] = ops_net.CONV_MODE
    rec["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
