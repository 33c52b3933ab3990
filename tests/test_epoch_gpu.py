"""inference.validate and engine.train_epoch (main.py's validation pass and training epoch as CUDA-graph replays) against
eager restatements of BP/main.py:419-526 and :239-340 on the same model and device batches of the GPU loader over a small
synthetic TuSimple directory; lf_seg_lane_maps_line against the reference's boolean-mask substitution; no host
synchronisation between reporting points."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import GOLDEN
from lanedetection_end2end_b200 import _capi, engine, inference
from lanedetection_end2end_b200.Dataloader import Load_Data_new as Ld
from lanedetection_end2end_b200.Loss_crit import define_loss_crit, fused_backprojection_loss
from lanedetection_end2end_b200.Networks import utils as nu
from lanedetection_end2end_b200.Networks.ERFNet import non_bottleneck_1d
from lanedetection_end2end_b200.Networks.LSQ_layer import Net

pytestmark = pytest.mark.gpu

CASES = {"clas4": (4, True, True), "plain2": (2, False, True), "seg4": (4, False, False)}   # nclasses, clas, end_to_end
BATCH = 4


class AverageMeter:          # BP/Networks/utils.py AverageMeter
    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


@pytest.fixture(scope="module")
def paths(tmp_path_factory):
    """16 files over the fixture's two frames and two label maps, with label files of 16 rows."""
    tmp = str(tmp_path_factory.mktemp("epoch"))
    z = np.load(os.path.join(GOLDEN, "loader_tusimple.npz"))
    for d in ("img", "gt", "Labels"):
        os.makedirs(os.path.join(tmp, d))
    fr = [z["jpeg/0"].tobytes(), z["jpeg/1"].tobytes()]
    mp = [z["png/0"].tobytes(), z["png/1"].tobytes()]
    rows = [json.loads(line) for line in z["lanes_jsonl"].tobytes().decode().splitlines()]
    lines = [json.loads(line) for line in z["lines_jsonl"].tobytes().decode().splitlines()]
    n = 16
    for k in range(1, n + 1):
        open(os.path.join(tmp, "img", "%d.jpg" % k), "wb").write(fr[k % 2])
        open(os.path.join(tmp, "gt", "%d.png" % k), "wb").write(mp[k % 2])
    for name, src in (("lanes.json", rows), ("lines.json", lines)):
        with open(os.path.join(tmp, "Labels", name), "w") as f:
            for k in range(n):
                f.write(json.dumps(src[(3 * k) % len(src)]) + "\n")
    return tmp, n


def make_args(case, tmp):
    L, clas, e2e = CASES[case]
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(L), "--order", "3",
                                        "--batch_size", str(BATCH), "--clas", str(int(clas)), "--end_to_end", str(e2e),
                                        "--loss_policy", "backproject", "--mask_percentage", "0.2"])
    args.val_batch_size, args.save_path = BATCH, tmp
    return args


def loaders(paths, args):
    tmp, n = paths
    lf = os.path.join(tmp, "Labels", "lanes.json")
    torch.manual_seed(0)
    return Ld.get_loader(n, lf, lf, os.path.join(tmp, "img"), os.path.join(tmp, "gt"), True, BATCH, BATCH, True, 0,
                         args.end_to_end, args.resize, args.nclasses, split_percentage=0.5, expected_count=None,
                         line_file=os.path.join(tmp, "Labels", "lines.json"))


def lane_prior(mod, inp, out):
    """--end_to_end False: an untrained decoder's argmax leaves lanes without pixels (singular fits); a constant vertical
    band per lane class on its logits gives every lane map pixels on every row."""
    prior = torch.zeros_like(out[1][:1])
    for k in range(prior.shape[1] - 1):
        prior[:, k + 1, :, 96 * k + 80:96 * k + 112] = 100.0
    return out[0], out[1] + prior, out[2]


def make_model(args, seed=0):
    torch.manual_seed(seed)
    model = Net(args).cuda()
    for m in model.modules():
        if isinstance(m, non_bottleneck_1d):
            m.dropout.p = 0.0                # no RNG draws: eager and graphed runs see the same masks
    if not args.end_to_end:
        model.net.register_forward_hook(lane_prior)
    return model


def criteria(args):
    crit, crit_seg = define_loss_crit(args)
    return crit, crit_seg, nn.BCEWithLogitsLoss().cuda(), nn.BCEWithLogitsLoss().cuda()


def short(batch, n=3):
    return tuple(t[:n] for t in batch)


def eager_validate(loader, model, criterion, criterion_seg, criterion_line_class, criterion_horizon, args):
    """BP/main.py:419-526 as written (args passed in; no tqdm, no plotting)."""
    losses, acc_hor_tot, acc_line_tot, rmse_metric_valid = AverageMeter(), AverageMeter(), AverageMeter(), AverageMeter()
    model.eval()
    model.defer_status_check = False
    skipped = []
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
            except RuntimeError:
                skipped.append(idx.tolist())
                continue
            if args.end_to_end:
                loss_left, x_cal0 = criterion(beta0, gt0, valid_points[:, 0])
                loss_right, x_cal1 = criterion(beta1, gt1, valid_points[:, 1])
                if args.nclasses > 3:
                    loss_left1, x_cal2 = criterion(beta2, gt2, valid_points[:, 2])
                    loss_right1, x_cal3 = criterion(beta3, gt3, valid_points[:, 3])
                    loss_left += loss_left1
                    loss_right += loss_right1
                loss = (loss_left + loss_right) / args.nclasses
            else:
                loss = criterion_seg(output_net, gt)
                loss_left, x_cal0 = criterion(beta0, gt0, valid_points[:, 0])
                loss_right, x_cal1 = criterion(beta1, gt1, valid_points[:, 1])
                if args.nclasses > 3:
                    loss_left1, x_cal2 = criterion(beta2, gt2, valid_points[:, 2])
                    loss_right1, x_cal3 = criterion(beta3, gt3, valid_points[:, 3])
                    loss_left += loss_left1
                    loss_right += loss_right1
                loss_metric = (loss_left + loss_right) / args.nclasses
                rmse_metric_valid.update(loss_metric.item(), input.size(0))
            losses.update(loss.item(), input.size(0))
            if args.clas:
                gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
                horizon_pred = torch.round(nn.Sigmoid()(outputs_horizon))
                acc = torch.eq(horizon_pred, gt_horizon)
                acc_hor = torch.sum(acc).float() / (args.resize * args.val_batch_size)
                acc_hor_tot.update(acc_hor.item())
                line_pred = torch.round(nn.Sigmoid()(outputs_line))
                acc = torch.eq(line_pred, gt_line)
                acc_line = torch.sum(acc).float() / (args.nclasses * args.val_batch_size)
                acc_line_tot.update(acc_line.item())
    return (losses.avg, acc_hor_tot.avg, acc_line_tot.avg, rmse_metric_valid.avg), skipped


def eager_train(loader, model, optimizer, criterion, criterion_seg, criterion_line_class, criterion_horizon, args, lane_loss):
    """BP/main.py:239-340 with the loss of the graph (fused_backprojection_loss); returns losses.avg, rmse_metric.avg, the
    per-step relative gap to main.py's per-lane criterion sum and the skipped batches."""
    losses, rmse_metric = AverageMeter(), AverageMeter()
    model.train()
    model.defer_status_check = False
    gaps, skipped = [], []
    for i, (input, gt, lanes, idx, gt_line, gt_horizon, valid_points) in enumerate(loader):
        input, lanes, valid_points, gt = input.cuda(), lanes.cuda(), valid_points.cuda(), gt.cuda().squeeze(1)
        try:
            out = model(input, gt_line, args.end_to_end, gt=gt)
        except RuntimeError:
            skipped.append(idx.tolist())
            continue
        if args.end_to_end:
            loss, _ = fused_backprojection_loss(criterion, out[:args.nclasses], lanes, valid_points)
            ref, _ = lane_loss(criterion, out, lanes, valid_points, args.nclasses)
            gaps.append(abs(loss.item() - ref.item()) / abs(ref.item()))
        else:
            loss = criterion_seg(out[5], gt)
            with torch.no_grad():
                loss_metric, _ = lane_loss(criterion, out, lanes, valid_points, args.nclasses)
                rmse_metric.update(loss_metric.item(), input.size(0))
        if args.clas:
            gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
            loss_horizon = criterion_horizon(out[7], gt_horizon).double()
            loss_line = criterion_line_class(out[6], gt_line).double()
            loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
    return losses.avg, rmse_metric.avg, gaps, skipped


def per_lane_loss(criterion, out, lanes, vp, L):
    loss_left, _ = criterion(out[0], lanes[:, 0, :], vp[:, 0])
    loss_right, _ = criterion(out[1], lanes[:, 1, :], vp[:, 1])
    if L > 3:
        loss_left = loss_left + criterion(out[2], lanes[:, 2, :], vp[:, 2])[0]
        loss_right = loss_right + criterion(out[3], lanes[:, 3, :], vp[:, 3])[0]
    return (loss_left + loss_right) / L, None


class Singular:
    """Zeroes image 0's decoder output in the batches listed in `which` (an all-zero weight map: a singular system) through
    a forward hook; `wrap` sets the factor on the stream before each batch is handed out, so eager and graphed runs see it."""

    def __init__(self, model, which):
        self.which, self.scale = set(which), torch.ones(BATCH, 1, 1, 1, device="cuda")
        self.h = model.net.register_forward_hook(
            lambda mod, inp, out: (out[0], out[1] * self.scale[:out[1].shape[0]], out[2]))

    def wrap(self, batches):
        for k, b in enumerate(batches):
            self.scale.fill_(1.0)
            if k in self.which:
                self.scale[0].fill_(0.0)
            yield b


class Listed(list):
    """A list of batches handed out through a generator each pass (len() as the loader's)."""

    def __init__(self, batches, wrap=None):
        super().__init__(batches)
        self.wrapper = wrap

    def __iter__(self):
        it = super().__iter__()
        return self.wrapper(it) if self.wrapper else it


@pytest.mark.parametrize("case", sorted(CASES))
def test_validate_equals_eager_main(paths, case, capsys):
    """validate == the restated eager validate, over the valid loader's batches plus a short last batch; then with one
    batch made singular: skipped by both, the same meters, and the skip line names its idx."""
    args = make_args(case, paths[0])
    _, valid, _ = loaders(paths, args)
    batches = list(valid)
    batches.append(short(batches[0]))
    model = make_model(args).eval()
    crits = criteria(args)
    want, _ = eager_validate(batches, model, *crits, args)
    got = inference.validate(Listed(batches), model, *crits, args)
    assert got == want, (got, want)
    assert got[0] != 0 and (got[1] != 0) == args.clas and (got[3] != 0) == (not args.end_to_end)
    sing = Singular(model, [1])
    try:
        want_s, skipped = eager_validate(Listed(batches, sing.wrap), model, *crits, args)
        capsys.readouterr()
        got_s = inference.validate(Listed(batches, sing.wrap), model, *crits, args)
    finally:
        sing.h.remove()
    out = capsys.readouterr().out
    assert skipped == [batches[1][3].tolist()]
    assert got_s == want_s and got_s != got
    assert "Batch with idx {} skipped due to singular matrix".format(batches[1][3].numpy()) in out
    assert out.count("skipped due to singular matrix") == 1


@pytest.mark.parametrize("case", ["clas4", "seg4"])
def test_train_epoch_equals_eager_main(paths, case, capsys):
    """One train_epoch against the restated eager loop driven by the same FusedOptimizer class: parameters, optimizer state
    and losses.avg bit for bit; each step's fused loss within 1e-12 of main.py's per-lane sum; a singular batch leaves the
    parameters untouched in both."""
    args = make_args(case, paths[0])
    train, _, _ = loaders(paths, args)
    batches = list(train)
    assert len(batches) == 2
    batches = batches + batches[:1]                 # three steps; the middle one is made singular below
    crits = criteria(args)
    ma, mb = make_model(args), make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    want_loss, want_rmse, gaps, _ = eager_train(batches, ma, oa, *crits, args, per_lane_loss)
    got_loss, got_rmse = engine.train_epoch(batches, mb, ob, *crits, args, 0)
    assert got_loss == want_loss and got_rmse == want_rmse
    assert (got_rmse != 0) == (not args.end_to_end)
    if args.end_to_end:
        assert len(gaps) == 3 and max(gaps) <= 1e-12, gaps
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    assert sa["param_groups"] == sb["param_groups"] and sa["state"].keys() == sb["state"].keys()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    # a singular batch: skipped by both, parameters untouched
    before = [p.detach().clone() for p in mb.parameters()]
    sings = [Singular(ma, [0]), Singular(mb, [0])]
    try:
        _, _, _, skipped = eager_train(Listed(batches[:1], sings[0].wrap), ma, oa, *crits, args, per_lane_loss)
        capsys.readouterr()
        got = engine.train_epoch(Listed(batches[:1], sings[1].wrap), mb, ob, *crits, args, 1)
    finally:
        for s in sings:
            s.h.remove()
    assert skipped == [batches[0][3].tolist()] and got == (0, 0)
    assert "Batch with idx {} skipped".format(batches[0][3].numpy()) in capsys.readouterr().out
    for a, b, p in zip(ma.parameters(), mb.parameters(), before):
        assert torch.equal(a, p) and torch.equal(b, p)


def _nosync(batches):
    """Yields the batches with torch's sync debug mode at "error" from the second batch until the pass has consumed the
    last one (the first batch builds the graph, which synchronises)."""
    def gen(it):
        for k, b in enumerate(it):
            if k == 1:
                torch.cuda.set_sync_debug_mode("error")
            yield b
        torch.cuda.set_sync_debug_mode(0)
    return Listed(batches, gen)


def test_no_host_synchronisation_between_reporting_points(paths):
    args = make_args("clas4", paths[0])
    args.print_freq = args.save_freq = 1000
    train, valid, _ = loaders(paths, args)
    tb, vb = list(train) * 2, list(valid) * 2
    model = make_model(args)
    opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True)
    crits = criteria(args)
    try:
        engine.train_epoch(_nosync(tb), model, opt, *crits, args, 0)
        inference.validate(_nosync(vb), model, *crits, args)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def _maps_reference(out, gt_line, nl, mask_rows):
    """BP/Networks/LSQ_layer.py:279-293,301,308-311 in torch."""
    activated = torch.max(out, 1)[1].float()
    masked = torch.stack([activated * (activated == k + 1).float() for k in range(nl)], 1)
    masked[:, :, :mask_rows] = 0
    if gt_line.sum() != 0:
        gt_mask = gt_line[:, :, None, None].bool().expand_as(masked)
        masked[gt_mask] = masked[0, 0].unsqueeze(0).repeat(int(gt_line.sum().item()), 1, 1).view(-1)
    return masked


def test_seg_lane_maps_line_equals_boolean_substitution():
    g = torch.Generator().manual_seed(7)
    B, nl, H, W, rows = 5, 4, 48, 80, 9
    out = torch.randn(B, nl + 1, H, W, generator=g).cuda()
    plain = torch.empty(B, nl, H, W, device="cuda")
    _capi.call("lf_seg_lane_maps", _capi.ptr(out), B, nl + 1, H, W, nl, rows, _capi.ptr(plain), _capi.stream_ptr())
    patterns = [torch.zeros(B, nl), torch.ones(B, nl)] + [(torch.rand(B, nl, generator=g) < p).float() for p in (0.2, 0.5, 0.8)]
    patterns.append(torch.tensor([[0, 1, 0, 1]] + [[1, 0, 0, 0]] * (B - 1), dtype=torch.float32))
    for gl in patterns:
        got = torch.full((B, nl, H, W), 7.0, device="cuda")
        gld = gl.cuda()
        _capi.call("lf_seg_lane_maps_line", _capi.ptr(out), B, nl + 1, H, W, nl, rows, _capi.ptr(gld), _capi.ptr(got),
                   _capi.stream_ptr())
        assert torch.equal(got, _maps_reference(out, gld, nl, rows)), gl
        if gl.sum() == 0:
            assert torch.equal(got, plain)
    got = torch.empty_like(plain)
    _capi.call("lf_seg_lane_maps_line", _capi.ptr(out), B, nl + 1, H, W, nl, rows, None, _capi.ptr(got), _capi.stream_ptr())
    assert torch.equal(got, plain)


def test_net_segmentation_branch_takes_device_and_host_gt_line():
    """Net.forward's --end_to_end False maps with gt_line on the device and on the host equal the reference's substitution.
    (That the device gt_line is not read on the host shows in test_validate_equals_eager_main[seg4]: its capture would
    fail on a host read.)"""
    args = make_args("seg4", "/tmp")
    model = make_model(args).eval()
    model.defer_status_check = True
    x = torch.rand(BATCH, 3, 256, 512, generator=torch.Generator().manual_seed(2)).cuda()
    gl = torch.tensor([[1, 0, 1, 1], [0, 0, 0, 0], [1, 1, 1, 1], [0, 1, 0, 0]], dtype=torch.float32)
    with torch.no_grad():
        dev = model(x, gl.cuda(), False)
        host = model(x, gl, False)
        zero = model(x, torch.zeros(BATCH, 4), False)
    want = _maps_reference(dev[5].float(), gl.cuda(), 4, model.zero_rows)
    assert torch.equal(dev[4], want) and torch.equal(host[4], want)
    assert torch.equal(zero[4], _maps_reference(dev[5].float(), torch.zeros(BATCH, 4).cuda(), 4, model.zero_rows))
