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
Kernel: lf_area_loss (loss, gradient and exact-area mean) timed with CUDA events over 2,000 back-to-back launches.

    python tools/bench_epoch_bev.py --clas [--out PATH] [--rounds 3]

times the same four arms with --clas (4 lanes, the line-type and horizon heads, BEV/main.py:246-253 and :417-488) and
writes profiles/h100/bench_epoch_bev_clas.json.  The eager training arm adds the heads' losses; the eager validation
arm adds the accuracies, writes validation_set_dst.json once per pass (every batch, see NOTES.md) and then runs the
host write_lsq_results and LaneEval (oracle/tusimple_oracle.py's restatement) over the whole set; the graphed
validation arm scores on the device (lf_bev_lane_score).  validation_set.json holds the validation rows of the
directory's label file, each with a raw_file of its own.  Kernel: lf_bev_lane_score, one launch per batch, timed with
CUDA events over 2,000 back-to-back launches."""
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


def eager_train_clas(loader, model, optimizer, criterion, crit_line, crit_hor, args):
    """BEV/main.py:199-295 with --clas (end to end, 4 lanes) with main.py's synchronisations."""
    import torch
    losses, exact_area = AverageMeter(), AverageMeter()
    model.train()
    for i, (input, gt, params, idx, gt_line, gt_horizon) in enumerate(loader):
        input, params = input.cuda(), params.cuda()
        gt0, gt1, gt2, gt3 = params[:, 0, :], params[:, 1, :], params[:, 2, :], params[:, 3, :]
        try:
            beta0, beta1, beta2, beta3, weightmap_zeros, M, output_net, outputs_line, outputs_horizon = \
                model(input, args.end_to_end)
        except RuntimeError as e:
            print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
            print(e)
            continue
        loss = _clas_loss(criterion, crit_line, crit_hor, args, (beta0, beta1, beta2, beta3), (gt0, gt1, gt2, gt3),
                          outputs_line, outputs_horizon, gt_line, gt_horizon)
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        with torch.no_grad():
            exact_area.update(exact_cpu(beta0, beta1, gt0, gt1), input.size(0))
    return losses.avg, exact_area.avg


def _clas_loss(criterion, crit_line, crit_hor, args, betas, gts, outputs_line, outputs_horizon, gt_line, gt_horizon):
    """BEV/main.py:222-237 (4 lanes, the presence masks) and :246-253."""
    import torch
    beta0, beta1, beta2, beta3 = betas
    gt0, gt1, gt2, gt3 = gts
    loss = criterion(beta0, gt0) + criterion(beta1, gt1)
    mask_llhs = torch.prod(gt2 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta2).type(torch.FloatTensor).cuda()
    mask_rrhs = torch.prod(gt3 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta3).type(torch.FloatTensor).cuda()
    loss += criterion(beta2 * mask_llhs, gt2) + criterion(beta3 * mask_rrhs, gt3)
    gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
    return loss * args.weight_fit + (crit_line(outputs_line, gt_line) + crit_hor(outputs_horizon, gt_horizon)) * \
        args.weight_class


def eager_validate_clas(loader, model, criterion, crit_line, crit_hor, args, valid_set_labels):
    """BEV/main.py:362-501 with --clas, validation_set_dst.json opened once per pass; then the host write_lsq_results
    and LaneEval over the whole set.  Returns (losses.avg, avg_trapezium_rule.avg, ACC_SEG)."""
    import torch
    from oracle import tusimple_oracle as to
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    losses, avg_trapezium_rule = AverageMeter(), AverageMeter()
    acc_hor_tot, acc_line_tot = AverageMeter(), AverageMeter()
    val_set_path = os.path.join(args.save_path, "eager_validation_set_dst.json")
    ls_result_path = os.path.join(args.save_path, "eager_ls_result.json")
    model.eval()
    with torch.no_grad(), open(val_set_path, "w") as jsonFile:
        for i, (input, gt, params, idx, gt_line, gt_horizon, index) in enumerate(loader):
            input, params = input.cuda(), params.cuda()
            gt0, gt1, gt2, gt3 = params[:, 0, :], params[:, 1, :], params[:, 2, :], params[:, 3, :]
            try:
                beta0, beta1, beta2, beta3, weightmap_zeros, M, output_net, outputs_line, outputs_horizon = \
                    model(input, args.end_to_end)
            except RuntimeError as e:
                print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
                print(e)
                continue
            gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
            horizon_pred = torch.round(torch.nn.Sigmoid()(outputs_horizon))
            acc_hor_tot.update((torch.sum(torch.eq(horizon_pred, gt_horizon)).float() /
                                (args.resize * args.batch_size)).item())
            _, line_pred = torch.max(outputs_line, 1)
            acc_line_tot.update((torch.sum(torch.eq(line_pred, gt_line)).float() /
                                 (args.nclasses * args.batch_size)).item())
            loss = _clas_loss(criterion, crit_line, crit_hor, args, (beta0, beta1, beta2, beta3), (gt0, gt1, gt2, gt3),
                              outputs_line, outputs_horizon, gt_line, gt_horizon)
            avg_trapezium_rule.update(exact_cpu(beta0, beta1, gt0, gt1), input.size(0))
            losses.update(loss.item(), input.size(0))
            params_batch = torch.cat((beta0, beta1, beta2, beta3), 2).transpose(1, 2).data.tolist()
            line_type, horizon_list = line_pred.data.tolist(), horizon_pred.data.tolist()
            for j in range(input.size(0)):
                json_line = valid_set_labels[index[j]]
                json_line["params"] = params_batch[j]
                json_line["line_id"] = line_type[j]
                json_line["horizon_est"] = horizon_list[j]
                json.dump(json_line, jsonFile)
                jsonFile.write("\n")
    L.write_lsq_results(val_set_path, ls_result_path, args.nclasses, False, False, args.resize, no_ortho=args.no_ortho)
    acc_seg = to.bench_one_submit(ls_result_path, val_set_path)
    return losses.avg, avg_trapezium_rule.avg, acc_seg[0]


def write_validation_set(paths, valid_idx, target):
    """validation_set.json as load_valid_set_file_all writes it (the rows of the label file for valid_idx), each row
    with a raw_file of its own: the synthetic directory reuses a few label rows for all its files."""
    rows = [json.loads(line) for line in open(paths["json_file"]).readlines()]
    target_idx = [int(i.split(".")[0]) for i in sorted(os.listdir(paths["image_dir"]))]
    with open(target, "w") as f:
        for k, i in enumerate(valid_idx):
            row = dict(rows[target_idx[i] - 1], raw_file="clips/valid/%d.jpg" % k)
            f.write(json.dumps(row) + "\n")
    return [json.loads(line) for line in open(target).readlines()]


def score_kernel_ms(B, gt_file):
    """Device time of one lf_bev_lane_score launch over a batch of B validation rows, KERNEL_LAUNCHES back to back."""
    import torch
    from lanedetection_end2end_b200 import _capi, inference
    s = inference.BevLaneScorer(gt_file)
    s.begin(B, RESIZE)
    g = torch.Generator().manual_seed(B)
    beta = (torch.randn(B, 4, 3, generator=g) * torch.tensor([0.1, 0.1, 0.3]) + torch.tensor([0.0, 0.0, 0.5])).cuda()
    rows = (torch.arange(B) % s.N).cuda()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    p = _capi.ptr
    args = (p(beta), p(rows), p(status), p(s.pos), B, 0, s.warp.ctypes.data, p(s.gt_S), p(s.h_samples), p(s.gt_x),
            p(s.gt_lanes), p(s.thresh), s.N, _capi.TUSIMPLE_MAX_GT, s.V, p(s.lanes), p(s.per_row), p(s.scored),
            _capi.stream_ptr())
    fn = _capi.lib().lf_bev_lane_score
    for _ in range(50):
        fn(*args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(KERNEL_LAUNCHES):
        rc = fn(*args)
    e1.record()
    torch.cuda.synchronize()
    assert rc == 0 and int(s.scored.sum()) == B
    return round(e0.elapsed_time(e1) / KERNEL_LAUNCHES, 5)


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
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--clas", action="store_true", help="time the --clas run (4 lanes, both heads, ACC_SEG)")
    a = ap.parse_args()
    if a.out is None:
        a.out = os.path.join(ROOT, "profiles", "h100", "bench_epoch_bev_clas.json" if a.clas else "bench_epoch_bev.json")
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
           "model": ("--clas: 4 lanes, the line-type and horizon heads, order 2, area loss (weight none), mask 0.3, "
                     "xavier init" if a.clas else
                     "BEV defaults: 2 lanes, order 2, area loss (weight none), mask 0.3, xavier init"),
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
                                             "xavier", "--nclasses", "4" if a.clas else "2", "--order", "2",
                                             "--weight_funct", "none", "--mask_percentage", "0.3", "--batch_size",
                                             str(batch), "--resize", str(RESIZE)] + (["--clas", "True"] if a.clas else []))
            args.save_path = d
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                train, valid, valid_idx = L.get_loader(COUNT, paths["json_file"], paths["image_dir"], paths["gt_dir"], False, batch,
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
            if a.clas:
                gt_file = os.path.join(d, "validation_set.json")
                labels = write_validation_set(paths, valid_idx, gt_file)
                acc_seg = {}

                def valid_graphed_clas(e):
                    out = io.StringIO()
                    with contextlib.redirect_stdout(out):
                        res = inference.validate_bev(valid, m_graphed, *crits, M_inv, args, e)
                    acc_seg["valid_graphed"] = float(out.getvalue().split("ACC_SEG on val is ")[1].split()[0])
                    return res[0:3:2]

                def valid_eager_clas(e):
                    loss, exact, acc_seg["valid_eager"] = eager_validate_clas(valid, m_eager, crit, *crits[2:], args,
                                                                              labels)
                    return loss, exact

                arms = {
                    "train_eager": lambda e: eager_train_clas(train, m_eager, opt_eager, crit, *crits[2:], args),
                    "train_graphed": arms["train_graphed"],
                    "valid_eager": valid_eager_clas,
                    "valid_graphed": valid_graphed_clas,
                }
            res = {k: {"seconds": [], "loss_avg": [], "exact_area_avg": []} for k in arms}
            if a.clas:
                for k in ("valid_eager", "valid_graphed"):
                    res[k]["acc_seg"] = []
            for r in range(a.rounds):
                for name, fn in arms.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    loss, exact = fn(r)
                    torch.cuda.synchronize()
                    res[name]["seconds"].append(round(time.perf_counter() - t0, 3))
                    res[name]["loss_avg"].append(loss)
                    res[name]["exact_area_avg"].append(exact)
                    if "acc_seg" in res[name]:
                        res[name]["acc_seg"].append(acc_seg[name])
                    print(batch, name, r, res[name]["seconds"][-1], loss, exact, flush=True)
            for name, v in res.items():
                n = len(train) if name.startswith("train") else len(valid)
                v["median_s"] = statistics.median(v["seconds"])
                v["batches"] = n
                v["median_ms_per_batch"] = round(1e3 * v["median_s"] / n, 2)
            rec["by_batch"][str(batch)] = res
            if a.clas:
                rec["kernel_ms"][str(batch)] = score_kernel_ms(batch, gt_file)
                print(batch, "lf_bev_lane_score ms", rec["kernel_ms"][str(batch)], flush=True)
            else:
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
