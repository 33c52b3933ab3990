"""What --pretrained costs on the library: the per-parameter-step optimizer update against the shared-step one, and a skip
epoch of the segmentation pretraining, graphed against main.py's eager loop.  Writes profiles/h100/bench_pretrain.json
(or --out).

    python tools/bench_pretrain.py [--out PATH] [--rounds 3] [--launches 200]

Update: FusedOptimizer(per_param_step=False) (lf_optim_step, one launch) and (per_param_step=True) (lf_optim_step_pp,
two launches) over every parameter of the model that gets a gradient in an end-to-end step, on the 2-lane model and on
train.sh's --clas model (4 lanes, order 3).  Per round and arm, CUDA events around --launches launches after a warm-up;
the arms alternate --rounds times in one process; the record holds every round and the median.

Skip epoch (BP/main.py:255-282): train.sh's model with --pretrained (4 lanes, order 3, --clas 1), batch 32, resize 256,
on the synthetic 3626-file TuSimple-shaped directory of tests/golden/loader_tusimple.npz that tools/bench_loader.py and
tools/bench_epoch.py time (2,900 training samples, 90 batches), loaded by the GPU loader with its device cache filled
before timing.  Arms, alternated --rounds times, each a whole epoch ended by a device synchronise:
  skip_eager     main.py's skip loop restated below, torch.optim.Adam as define_optim builds it
  skip_graphed   engine.train_epoch(epoch 0) with define_optim(..., fused=True, per_param_step=True)
Each arm has its own model and optimizer.  A graphed epoch includes building its graph, as a main.py epoch would."""
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


def eager_skip(loader, model, optimizer, criterion_seg):
    """BP/main.py:255-282 (the plot at save_freq aside), with its loss.item() per batch."""
    losses_skip = AverageMeter()
    model.train()
    for i, (input, gt, lanes, idx, gt_line, gt_horizon, valid_points) in enumerate(loader):
        input, gt = input.cuda(), gt.cuda().squeeze(1)
        output_net = model(input, gt_line, False, early_return=True)
        loss = criterion_seg(output_net, gt)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        losses_skip.update(loss.item(), input.size(0))
    return losses_skip.avg


def _args(extra):
    from lanedetection_end2end_b200.Networks.utils import define_args
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--loss_policy", "backproject", "--weight_init",
                                     "xavier", "--split_percentage", "0.2", "--activation_layer", "square",
                                     "--mask_percentage", "0.20", "--batch_size", str(BATCH), "--resize", str(RESIZE)]
                                    + extra)
    args.val_batch_size = BATCH
    return args


def _model(args):
    import torch
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    torch.manual_seed(0)
    m = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(m, "xavier")
    return m.cuda()


def bench_update(rounds, launches):
    import torch
    from lanedetection_end2end_b200.optim import FusedOptimizer
    sets = {"2 lanes": ["--nclasses", "2", "--order", "2"],
            "train.sh --clas (4 lanes, order 3)": ["--nclasses", "4", "--order", "3", "--clas", "1"]}
    out = {}
    for name, extra in sets.items():
        model = _model(_args(extra))
        # the parameters an end-to-end step gives a gradient (all but the encoder's unused output_conv)
        params = [p for n, p in model.named_parameters() if not n.startswith("net.encoder.output_conv")]
        g = torch.Generator(device="cuda").manual_seed(1)
        for p in params:
            p.grad = torch.randn(p.shape, device="cuda", generator=g) * 1e-3
        opts = {"shared_step": FusedOptimizer(params, "adam", 1e-3, 0),
                "per_param_step": FusedOptimizer(params, "adam", 1e-3, 0, per_param_step=True)}
        for o in opts.values():
            o.prepare(o.grad_params())
            o.sync_hyperparameters()
            for _ in range(20):
                o.launch()
        torch.cuda.synchronize()
        res = {k: [] for k in opts}
        for _ in range(rounds):
            for k, o in opts.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(launches):
                    o.launch()
                e1.record()
                torch.cuda.synchronize()
                res[k].append(round(1e3 * e0.elapsed_time(e1) / launches, 2))
        nelem = sum(p.numel() for p in params)
        out[name] = {"tensors": len(params), "elements": nelem,
                     "us_per_update": res, "median_us": {k: statistics.median(v) for k, v in res.items()}}
        print(name, out[name], flush=True)
    return out


def bench_skip_epoch(rounds):
    import torch
    import torch.nn as nn
    from oracle import make_loader_golden as mlg
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    from lanedetection_end2end_b200.Loss_crit import define_loss_crit
    from lanedetection_end2end_b200.Networks.utils import define_optim
    args = _args(["--nclasses", "4", "--order", "3", "--clas", "1", "--pretrained", "True", "--pretrain_epochs", "25",
                  "--skip_epochs", "25"])
    z = np.load(os.path.join(ROOT, "tests", "golden", "loader_tusimple.npz"))
    out = {}
    with tempfile.TemporaryDirectory() as d:
        paths = mlg.from_fixture(z, d)
        args.save_path = d
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            train, _, _ = L.get_loader(3626, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"],
                                       True, BATCH, BATCH, True, 0, True, RESIZE, 4, split_percentage=0.2,
                                       line_file=paths["line_file"])
        for _ in train:                  # fill the cache
            pass
        crits = (*define_loss_crit(args), nn.BCEWithLogitsLoss().cuda(), nn.BCEWithLogitsLoss().cuda())
        m_eager, m_graphed = _model(args), _model(args)
        opt_eager = define_optim("adam", m_eager.parameters(), args.learning_rate, args.weight_decay, fused=False)
        opt_graphed = define_optim("adam", m_graphed.parameters(), args.learning_rate, args.weight_decay, fused=True,
                                   per_param_step=True)
        args.end_to_end = False          # get_flags(0) of a pretrained run
        arms = {"skip_eager": lambda: eager_skip(train, m_eager, opt_eager, crits[1]),
                "skip_graphed": lambda: engine.train_epoch(train, m_graphed, opt_graphed, *crits, args, 0)[0]}
        res = {k: {"seconds": [], "loss_avg": []} for k in arms}
        for r in range(rounds):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                loss = fn()
                torch.cuda.synchronize()
                res[name]["seconds"].append(round(time.perf_counter() - t0, 3))
                res[name]["loss_avg"].append(loss)
                print(name, r, res[name]["seconds"][-1], loss, flush=True)
        for v in res.values():
            v["median_s"] = statistics.median(v["seconds"])
            v["batches"] = len(train)
            v["median_ms_per_batch"] = round(1e3 * v["median_s"] / len(train), 2)
        out["arms"] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_pretrain.json"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    a = ap.parse_args()
    import torch
    from bench_modes import gpu_info
    from lanedetection_end2end_b200 import ops_net
    assert torch.cuda.is_available(), "bench_pretrain.py times the GPU; there is no CPU fallback"
    rec = {"gpu": gpu_info(), "conv_mode": ops_net.CONV_MODE}
    rec["update"] = bench_update(a.rounds, a.launches)
    rec["skip_epoch"] = bench_skip_epoch(a.rounds)
    rec["skip_epoch"].update({
        "batch": BATCH, "resize": RESIZE,
        "model": "train.sh with --pretrained: 4 lanes, order 3, --clas 1, mask 0.2, xavier init; skip epoch (epoch 0)",
        "dataset": "synthetic 3626-file TuSimple-shaped directory (tests/golden/loader_tusimple.npz): 2,900 training "
                   "samples (90 batches), GPU loader with a filled device cache"})
    rec["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
