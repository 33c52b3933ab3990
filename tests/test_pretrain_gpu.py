"""engine.train_epoch under --pretrained (a skip epoch through output_conv2 without the least-squares layer, the
segmentation epochs, then end to end) on FusedOptimizer(per_param_step=True), against an eager restatement of
BP/main.py:32-43,239-340 on the same model, device batches, fused loss and optimizer class: parameters, optimizer state,
per-parameter steps and returned meters bit for bit; the checkpoint after the switch loads into torch.optim.Adam; no host
synchronisation within a skip epoch.  Setup and dropout treatment as tests/test_epoch_gpu.py."""
import pytest
import torch

from lanedetection_end2end_b200 import engine, inference
from lanedetection_end2end_b200.Networks import utils as nu
from lanedetection_end2end_b200.Networks.ERFNet import non_bottleneck_1d
from lanedetection_end2end_b200.Networks.LSQ_layer import Net
from test_epoch_gpu import (BATCH, AverageMeter, Listed, _nosync, criteria, eager_train, lane_prior, loaders,  # noqa: F401
                            paths, per_lane_loss)

pytestmark = pytest.mark.gpu


def make_args(tmp, clas, skip_epochs, pretrain_epochs):
    """train.sh's model scaled down: 4 lanes, order 3, --pretrained, --clas as given."""
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "3",
                                        "--batch_size", str(BATCH), "--clas", str(int(clas)), "--end_to_end", "True",
                                        "--loss_policy", "backproject", "--mask_percentage", "0.2", "--pretrained",
                                        "True", "--skip_epochs", str(skip_epochs), "--pretrain_epochs",
                                        str(pretrain_epochs)])
    args.val_batch_size, args.save_path = BATCH, tmp
    return args


def make_model(args, seed=0):
    torch.manual_seed(seed)
    model = Net(args).cuda()
    for m in model.modules():
        if isinstance(m, non_bottleneck_1d):
            m.dropout.p = 0.0                # no RNG draws: eager and graphed runs see the same masks

    def prior(mod, inp, out):                # the segmentation head's maps only (see test_epoch_gpu.lane_prior)
        return lane_prior(mod, inp, out) if out[1].shape[1] == args.nclasses + 1 else out
    model.net.register_forward_hook(prior)
    return model


def get_flags(args, epoch):
    """BP/main.py:32-43 (prints left out)."""
    skip = False
    if args.pretrained:
        if epoch < args.pretrain_epochs:
            args.end_to_end = False
            if epoch < args.skip_epochs:
                skip = True
        else:
            args.end_to_end = True
    return skip


def eager_skip(loader, model, optimizer, criterion_seg):
    """BP/main.py:255-282 (no plot)."""
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
    return losses_skip.avg, 0.0


def _state(model, opt):
    out = {n: p.detach().clone() for n, p in model.named_parameters()}
    for n, p in model.named_parameters():
        for k, v in opt.state.get(p, {}).items():
            if k != "step":
                out[n + "." + k] = v.clone()
    return out


def _run(paths, clas, skip_epochs, pretrain_epochs, nepochs):
    args_a = make_args(paths[0], clas, skip_epochs, pretrain_epochs)
    args_b = make_args(paths[0], clas, skip_epochs, pretrain_epochs)
    train, _, _ = loaders(paths, args_a)
    batches = list(train)
    crits = criteria(args_a)
    ma, mb = make_model(args_a), make_model(args_b)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True, per_param_step=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True, per_param_step=True)
    names = [n for n, _ in ma.named_parameters()]
    history = []
    for epoch in range(nepochs):
        skip_a, skip_b = get_flags(args_a, epoch), get_flags(args_b, epoch)
        assert skip_a == skip_b
        if skip_a:
            want = eager_skip(batches, ma, oa, crits[1])
        else:
            w_loss, w_rmse, _, _ = eager_train(batches, ma, oa, *crits, args_a, per_lane_loss)
            want = (w_loss, w_rmse)
        before = vars(args_b).copy()
        got = engine.train_epoch(batches, mb, ob, *crits, args_b, epoch)
        assert vars(args_b) == before                     # train_epoch leaves args alone
        assert got == want, (epoch, got, want)
        a, b = _state(ma, oa), _state(mb, ob)
        assert set(a) == set(b)
        for n in a:
            assert torch.equal(a[n], b[n]), (epoch, n)
        assert oa.step_counts == ob.step_counts, epoch
        history.append((skip_a, bool(args_a.end_to_end), dict(zip(names, ob.step_counts)), b))
    return args_b, mb, ob, batches, crits, history


def test_clas_skip_then_end_to_end(paths):
    """train.sh's schedule (skip_epochs == pretrain_epochs): a skip epoch, then end to end with the heads."""
    args, model, opt, batches, _, hist = _run(paths, True, 1, 1, 2)
    nb = len(batches)
    (skip0, _, steps0, state0), (skip1, e2e1, steps1, state1) = hist
    assert skip0 and not skip1 and e2e1
    heads = [n for n in steps1 if "decoder.output_conv." in n or n.startswith(("line_classification", "horizon_estimation"))]
    seg = [n for n in steps1 if "output_conv2" in n]
    never = [n for n in steps1 if steps1[n] == 0]
    assert len(heads) > 4 and len(seg) == 2 and all(n.startswith("net.encoder") for n in never)
    for n in steps1:
        if n in heads:                          # output_conv and the heads start at step 1 in the end-to-end epoch
            assert steps0[n] == 0 and steps1[n] == nb and n + ".exp_avg" not in state0, n
        elif n in seg:                          # output_conv2 keeps its state, untouched
            assert steps0[n] == steps1[n] == nb, n
            assert torch.equal(state1[n], state0[n]) and torch.equal(state1[n + ".exp_avg"], state0[n + ".exp_avg"]), n
        elif n not in never:                    # the shared layers count on
            assert steps0[n] == nb and steps1[n] == 2 * nb, n
    # the checkpoint after the switch loads into torch.optim.Adam with each parameter's own step
    sd = opt.state_dict()
    tor = torch.optim.Adam(model.parameters(), lr=1e-3)
    tor.load_state_dict(sd)
    params = list(model.parameters())
    for i, p in enumerate(params):
        if i in sd["state"]:
            assert float(tor.state[p]["step"]) == opt.step_counts[i]
            assert torch.equal(tor.state[p]["exp_avg"], opt.state[p]["exp_avg"])
    assert len({float(st["step"]) for st in sd["state"].values()}) == 2


def test_segmentation_phase_then_end_to_end(paths):
    """--clas False with a non-empty segmentation phase: skip, segmentation (--end_to_end False, output_conv2 with the
    least-squares fit for the rmse metric), end to end; then inference.validate on the pretrained model."""
    args, model, opt, batches, crits, hist = _run(paths, False, 1, 2, 3)
    assert [(h[0], h[1]) for h in hist] == [(True, False), (False, False), (False, True)]
    nb = len(batches)
    steps = hist[2][2]
    for n, c in steps.items():
        if "output_conv2" in n:
            assert c == 2 * nb, (n, c)
        elif "decoder.output_conv" in n:
            assert c == nb, (n, c)
        else:
            assert c == 3 * nb or (c == 0 and n.startswith("net.encoder")), (n, c)
    _, valid, _ = loaders(paths, args)
    for e2e in (False, True):
        args.end_to_end = e2e
        got = inference.validate(list(valid), model, *crits, args)
        assert got[0] == got[0] and got[0] != 0 and (got[3] != 0) == (not e2e)


def test_clas_refused_in_a_segmentation_epoch(paths):
    args = make_args(paths[0], True, 1, 2)
    model = make_model(args)
    opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True, per_param_step=True)
    get_flags(args, 1)
    with pytest.raises(ValueError, match="--clas needs --end_to_end True"):
        engine.train_epoch([], model, opt, *criteria(args), args, 1)
    default = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True)
    with pytest.raises(ValueError, match="per_param_step=True"):
        engine.train_epoch([], model, default, *criteria(args), args, 0)


def test_no_host_synchronisation_in_a_skip_epoch(paths):
    args = make_args(paths[0], True, 1, 1)
    train, _, _ = loaders(paths, args)
    tb = list(train) * 2
    model = make_model(args)
    opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True, per_param_step=True)
    get_flags(args, 0)
    try:
        loss, zero = engine.train_epoch(_nosync(tb), model, opt, *criteria(args), args, 0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert loss > 0 and zero == 0.0
