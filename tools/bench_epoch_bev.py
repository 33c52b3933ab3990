"""Epoch time of the bird's-eye-view experiment's training loop and validation pass: eager as Birds_Eye_View_Loss/main.py
writes them against engine.train_epoch_bev and inference.validate_bev (one CUDA-graph replay per batch), and the device
time of lf_area_loss.  Writes profiles/h100/bench_epoch_bev.json (or --out).

    python tools/bench_epoch_bev.py [--out PATH] [--rounds 3]

Workload: the synthetic 2535-file BEV directory of tests/golden/loader_bev.npz (the one tools/bench_loader_bev.py times),
the BEV defaults (2 lanes, order 2, area loss with weight none, mask 0.3, xavier init), the library's default convolution
mode (tf32x3), resize 256, batch 8 (the BEV default) and 32, loaded by the GPU loader with its device cache filled before
timing.  Arms, alternated --rounds times in one process per batch size, each a whole epoch or pass ended by a device
synchronise:
  train_eager     BEV/main.py:199-295 restated below (tqdm and plotting aside), torch.optim.Adam as define_optim builds it,
                  the exact-area metric on the CPU (Loss_crit.polynomial, the reference's arithmetic)
  train_graphed   engine.train_epoch_bev with define_optim(..., fused=True)
  valid_eager     BEV/main.py:362-501 restated below
  valid_graphed   inference.validate_bev
Each arm has its own model and optimizer, so the training arms keep training their own weights round after round.
Kernel: lf_area_loss (loss, gradient and exact-area mean) timed with CUDA events over 2,000 back-to-back launches."""
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

BATCHES, RESIZE, COUNT, KERNEL_LAUNCHES = (8, 32), 256, 2535, 2000


class AverageMeter:          # BEV/Networks/utils.py AverageMeter
    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def exact_cpu(beta0, beta1, gt0, gt1):
    from lanedetection_end2end_b200.Loss_crit import polynomial
    trap_left = polynomial(beta0.cpu()).trapezoidal(polynomial(gt0.cpu()))
    trap_right = polynomial(beta1.cpu()).trapezoidal(polynomial(gt1.cpu()))
    return ((trap_left + trap_right) / 2).mean().item()


def eager_train(loader, model, optimizer, criterion, args):
    """BEV/main.py:199-295 (end-to-end branch, 2 lanes) with main.py's synchronisations."""
    import torch
    losses, exact_area = AverageMeter(), AverageMeter()
    model.train()
    for i, (input, gt, params, idx, gt_line, gt_horizon) in enumerate(loader):
        input, params = input.cuda(), params.cuda()
        gt0, gt1 = params[:, 0, :], params[:, 1, :]
        try:
            beta0, beta1, beta2, beta3, weightmap_zeros, M, output_net, outputs_line, outputs_horizon = \
                model(input, args.end_to_end)
        except RuntimeError as e:
            print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
            print(e)
            continue
        loss = criterion(beta0, gt0) + criterion(beta1, gt1)
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        with torch.no_grad():
            exact_area.update(exact_cpu(beta0, beta1, gt0, gt1), input.size(0))
    return losses.avg, exact_area.avg


def eager_validate(loader, model, criterion, args):
    """BEV/main.py:362-501 (end-to-end branch, 2 lanes)."""
    import torch
    losses, avg_trapezium_rule = AverageMeter(), AverageMeter()
    model.eval()
    with torch.no_grad():
        for i, (input, gt, params, idx, gt_line, gt_horizon, index) in enumerate(loader):
            input, params = input.cuda(), params.cuda()
            gt0, gt1 = params[:, 0, :], params[:, 1, :]
            try:
                beta0, beta1, beta2, beta3, weightmap_zeros, M, output_net, outputs_line, outputs_horizon = \
                    model(input, args.end_to_end)
            except RuntimeError as e:
                print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
                print(e)
                continue
            loss = criterion(beta0, gt0) + criterion(beta1, gt1)
            avg_trapezium_rule.update(exact_cpu(beta0, beta1, gt0, gt1), input.size(0))
            losses.update(loss.item(), input.size(0))
    return losses.avg, avg_trapezium_rule.avg


def kernel_ms(B, L=2):
    """Device time of one lf_area_loss launch (all outputs) over KERNEL_LAUNCHES back-to-back launches."""
    import torch
    from lanedetection_end2end_b200 import _capi
    g = torch.Generator().manual_seed(B)
    beta, params = torch.randn(B, L, 3, generator=g).cuda(), torch.randn(B, 4, 3, generator=g).cuda()
    out = torch.empty(2 + B * L * 3 + B, device="cuda")
    p, s = _capi.ptr, _capi.stream_ptr()
    args = (p(beta), p(params), B, L, 0, p(out[0:1]), p(out[2:2 + B * L * 3]), p(out[2 + B * L * 3:]), p(out[1:2]), s)
    fn = _capi.lib().lf_area_loss
    for _ in range(50):
        fn(*args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(KERNEL_LAUNCHES):
        rc = fn(*args)
    e1.record()
    torch.cuda.synchronize()
    assert rc == 0
    return round(e0.elapsed_time(e1) / KERNEL_LAUNCHES, 5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_epoch_bev.json"))
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    from bench_modes import gpu_info
    from oracle import make_loader_bev_golden as mbg
    from lanedetection_end2end_b200 import engine, inference, ops_net
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    from lanedetection_end2end_b200.bev.Loss_crit import define_loss_crit
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args, define_init_weights, define_optim
    assert torch.cuda.is_available(), "bench_epoch_bev.py times the GPU; there is no CPU fallback"
    rec = {"gpu": gpu_info(), "resize": RESIZE, "conv_mode": ops_net.CONV_MODE,
           "model": "BEV defaults: 2 lanes, order 2, area loss (weight none), mask 0.3, xavier init",
           "dataset": "synthetic 2535-file BEV directory (tests/golden/loader_bev.npz), split 0.2, GPU loader with a filled "
                      "device cache",
           "note": "each round's epoch includes building the graphs of the graphed arms (warm-up and capture), as a "
                   "main.py epoch calling them would",
           "kernel_ms": {}, "by_batch": {}}
    z = np.load(os.path.join(ROOT, "tests", "golden", "loader_bev.npz"))
    with tempfile.TemporaryDirectory() as d:
        paths = mbg.from_fixture(z, d)
        for batch in BATCHES:
            args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--loss_policy", "area", "--weight_init",
                                             "xavier", "--nclasses", "2", "--order", "2", "--weight_funct", "none",
                                             "--mask_percentage", "0.3", "--batch_size", str(batch), "--resize", str(RESIZE)])
            args.save_path = d
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                train, valid, _ = L.get_loader(COUNT, paths["json_file"], paths["image_dir"], paths["gt_dir"], False, batch,
                                               True, 0, True, RESIZE, 0.2, line_file=paths["line_file"])
            for loader in (train, valid):         # fill the cache
                for _ in loader:
                    pass
            crit, crit_seg = define_loss_crit(args)
            crits = (crit, crit_seg, torch.nn.CrossEntropyLoss().cuda(), torch.nn.BCEWithLogitsLoss().cuda())
            M_inv = L.get_homography(RESIZE)

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
                "train_eager": lambda e: eager_train(train, m_eager, opt_eager, crit, args),
                "train_graphed": lambda e: engine.train_epoch_bev(train, m_graphed, opt_graphed, *crits, args, e)[0:3:2],
                "valid_eager": lambda e: eager_validate(valid, m_eager, crit, args),
                "valid_graphed": lambda e: inference.validate_bev(valid, m_graphed, *crits, M_inv, args, e)[0:3:2],
            }
            res = {k: {"seconds": [], "loss_avg": [], "exact_area_avg": []} for k in arms}
            for r in range(a.rounds):
                for name, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    loss, exact = fn(r)
                    torch.cuda.synchronize()
                    res[name]["seconds"].append(round(time.perf_counter() - t0, 3))
                    res[name]["loss_avg"].append(loss)
                    res[name]["exact_area_avg"].append(exact)
                    print(batch, name, r, res[name]["seconds"][-1], loss, exact, flush=True)
            for name, v in res.items():
                n = len(train) if name.startswith("train") else len(valid)
                v["median_s"] = statistics.median(v["seconds"])
                v["batches"] = n
                v["median_ms_per_batch"] = round(1e3 * v["median_s"] / n, 2)
            rec["by_batch"][str(batch)] = res
            rec["kernel_ms"][str(batch)] = kernel_ms(batch)
            print(batch, "lf_area_loss ms", rec["kernel_ms"][str(batch)], flush=True)
            del train, valid, m_eager, m_graphed, opt_eager, opt_graphed
            torch.cuda.empty_cache()
    rec["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
