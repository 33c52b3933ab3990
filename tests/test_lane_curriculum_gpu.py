"""--lane_curriculum end to end on the back-projection Net: the status guard sees the fitted lanes only, the graphed
egolane step against the eager K = 2 step and the eager full forward, the step from epoch E on against today's
train_epoch, validation after an egolane epoch, and expand_lanes' warm start."""
import pytest
import torch

import test_epoch_gpu as te
from test_epoch_gpu import paths  # noqa: F401  (the module-scoped fixture of the synthetic TuSimple directory)
from lanedetection_end2end_b200 import engine, inference, ops_net
from lanedetection_end2end_b200.Loss_crit import fused_backprojection_loss
from lanedetection_end2end_b200.Networks import utils as nu

pytestmark = pytest.mark.gpu


def curriculum_args(tmp, E=3):
    args = te.make_args("clas4", tmp)
    args.lane_curriculum = E
    return args


class ZeroLane:
    """Zeroes decoder output channel `lane` of every image through a forward hook: that lane's weight map is all zero, a
    singular system."""

    def __init__(self, model, lane):
        def hook(mod, inp, out):
            keep = torch.ones(1, out[1].shape[1], 1, 1, device=out[1].device)
            keep[:, lane] = 0
            return out[0], out[1] * keep, out[2]
        self.h = model.net.register_forward_hook(hook)


def eager_step(model, opt, batch, crits, args, K):
    """One eager training step of train_epoch's loss with model.fit_lanes = K (None: every lane)."""
    input, gt, lanes, idx, gt_line, gt_horizon, valid = batch
    model.train()
    model.defer_status_check = False
    model.fit_lanes = K
    try:
        out = model(input.cuda().float(), gt_line, True)
    finally:
        model.fit_lanes = None
    k = K or args.nclasses
    loss, _ = fused_backprojection_loss(crits[0], out[:k], lanes.cuda(), valid.cuda())
    loss_horizon = crits[3](out[7], gt_horizon.cuda()).double()
    loss_line = crits[2](out[6], gt_line.cuda()).double()
    loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
    opt.zero_grad()
    loss.backward()
    opt.step()
    return loss.item(), out


def test_guard_sees_the_fitted_lanes_only(paths, capsys):
    """A batch whose lane-2 map is all zeros: with fit_lanes = 2 the status word stays 0 and the graphed step updates
    the parameters; with every lane fitted the same batch is skipped."""
    args = curriculum_args(paths[0])
    batches = list(te.loaders(paths, args)[0])[:1]
    crits = te.criteria(args)
    model = te.make_model(args)
    z = ZeroLane(model, 2)
    try:
        opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True)
        before = [p.detach().clone() for p in model.parameters()]
        capsys.readouterr()
        loss, _ = engine.train_epoch(batches, model, opt, *crits, args, 0)
        assert "skipped" not in capsys.readouterr().out and loss != 0
        assert int(model.lsq_status.item()) == 0 and model.fit_lanes is None
        assert any(not torch.equal(p, q) for p, q in zip(model.parameters(), before))
        before = [p.detach().clone() for p in model.parameters()]
        got = engine.train_epoch(batches, model, opt, *crits, args, 3)
        assert got == (0, 0)
        assert "Batch with idx {} skipped".format(batches[0][3].numpy()) in capsys.readouterr().out
        for p, q in zip(model.parameters(), before):
            assert torch.equal(p, q)
    finally:
        z.h.remove()


def test_egolane_step_against_eager(paths):
    """Epoch 0 of --lane_curriculum 3, one batch: the graphed loss is the fused loss over lanes 0 and 1 of a full eager
    forward (plus the heads' 4-lane losses) to 1e-12 relative, the parameters and Adam state equal the eager K = 2 step's,
    and validation right after, with fit_lanes = 2 left on the model, equals validation with fit_lanes = None."""
    args = curriculum_args(paths[0])
    train, valid, _ = te.loaders(paths, args)
    batch = list(train)[0]
    crits = te.criteria(args)
    ma, mb, mc = te.make_model(args), te.make_model(args), te.make_model(args)
    mb.load_state_dict(ma.state_dict())
    mc.load_state_dict(ma.state_dict())
    # the full forward's lanes 0 and 1 (mc is a copy, so its BatchNorm statistics do not touch ma / mb)
    with torch.no_grad():
        mc.train()
        full = mc(batch[0].cuda().float(), batch[4], True)
        assert full[3] is not None
        want_fit, _ = fused_backprojection_loss(crits[0], full[:2], batch[2].cuda(), batch[6].cuda())
        want_heads = crits[2](full[6], batch[4].cuda()).double() + crits[3](full[7], batch[5].cuda()).double()
    want_loss = (want_fit * args.weight_fit + want_heads * args.weight_class).item()
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    eager_loss, out = eager_step(ma, oa, batch, crits, args, 2)
    assert out[2] is None and out[3] is None and out[4].shape[1] == 2
    got_loss, _ = engine.train_epoch([batch], mb, ob, *crits, args, 0)
    assert mb.fit_lanes is None
    assert abs(got_loss - want_loss) <= 1e-12 * abs(want_loss), (got_loss, want_loss)
    assert got_loss == eager_loss
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    # the outer lanes' output_conv channels got a zero gradient: Adam (weight_decay 0) left them as they were
    w = mb.net.decoder.output_conv.weight
    assert torch.equal(w[:, 2:], mc.net.decoder.output_conv.weight[:, 2:]) and not torch.equal(w[:, :2], mc.net.decoder.output_conv.weight[:, :2])
    # an eval forward fits every lane whatever fit_lanes holds: validation with fit_lanes = 2 left on the model is
    # validation with fit_lanes = None
    vb = list(valid)
    want = inference.validate(te.Listed(vb), mb, *crits, args)
    mb.fit_lanes = 2
    try:
        got = inference.validate(te.Listed(vb), mb, *crits, args)
    finally:
        mb.fit_lanes = None
    assert got == want and got[0] != 0


def test_step_from_epoch_e_on_is_todays_step(paths):
    """At epoch E the curriculum fits every lane: train_epoch is bit-identical to train_epoch without the flag."""
    args = curriculum_args(paths[0])
    plain = te.make_args("clas4", paths[0])
    batches = list(te.loaders(paths, args)[0])
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    assert engine.train_epoch(batches, ma, oa, *crits, args, 3) == engine.train_epoch(batches, mb, ob, *crits, plain, 3)
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k


def test_expand_lanes_warm_start(paths):
    """A 4-lane Net loaded from a 2-lane Net with expand_lanes fits lanes 0 and 1 as the 2-lane Net does (fp32 mode)."""
    default = ops_net.CONV_MODE
    ops_net.set_conv_mode("fp32")
    try:
        a2 = te.make_args("plain2", paths[0])
        a4 = te.make_args("clas4", paths[0])
        m2 = te.make_model(a2, seed=0).eval()
        m4 = te.make_model(a4, seed=1).eval()
        missing = nu.expand_lanes(m2.state_dict(), m4)
        assert missing and all(k.startswith(("line_classification.", "horizon_estimation.")) for k in missing)
        batch = list(te.loaders(paths, a4)[0])[0]
        x, gl = batch[0].cuda().float(), batch[4]
        with torch.no_grad():
            o2 = m2(x, gl, True)
            o4 = m4(x, gl, True)
        for k in (0, 1):
            rel = ((o4[k] - o2[k]).abs().max() / o2[k].abs().max()).item()
            assert rel <= 1e-9, (k, rel)
    finally:
        ops_net.set_conv_mode(default)
