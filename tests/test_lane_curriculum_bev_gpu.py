"""--lane_curriculum on the bird's-eye-view Net with --clas: the graphed egolane epoch against the eager K = 2 loop and the
eager full forward, the epoch from E on against today's train_epoch_bev, and validate_bev after an egolane epoch."""
import os

import numpy as np
import pytest
import torch

import test_bev_clas_gpu as tc
from conftest import GOLDEN
from test_epoch_bev_gpu import paths  # noqa: F401  (the module-scoped fixture of the synthetic BEV directory)
from lanedetection_end2end_b200 import engine, inference
from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
from lanedetection_end2end_b200.bev.Loss_crit import fused_area_loss
from lanedetection_end2end_b200.Networks import utils as nu

pytestmark = pytest.mark.gpu


def eager_train(loader, model, optimizer, crit_line, crit_hor, args, K):
    """test_bev_clas_gpu.eager_train with model.fit_lanes = K and the fit loss over K lanes."""
    losses, exact_area = tc.AverageMeter(), tc.AverageMeter()
    model.train()
    model.defer_status_check = False
    model.fit_lanes = K
    try:
        for input, gt, params, idx, gt_line, gt_horizon in loader:
            input, params = input.cuda().float(), params.cuda()
            out = model(input, True)
            assert out[2] is None and out[3] is None and out[4].shape[1] == K
            loss, exact = fused_area_loss(out[:K], params, args.weight_funct, exact=True)
            loss = loss * args.weight_fit + (crit_line(out[7], gt_line.cuda()) + crit_hor(out[8], gt_horizon.cuda())) \
                * args.weight_class
            losses.update(loss.item(), input.size(0))
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            exact_area.update(exact.item(), input.size(0))
    finally:
        model.fit_lanes = None
    return losses.avg, 0, exact_area.avg


def test_egolane_epoch_bev_with_clas(paths):
    args = tc.make_args(paths[0])
    args.lane_curriculum = 3
    batches = tc.batches_of(paths, args, "train")
    crits = tc.criteria(args)
    ma, mb, mc = tc.make_model(args), tc.make_model(args), tc.make_model(args)
    mb.load_state_dict(ma.state_dict())
    mc.load_state_dict(ma.state_dict())
    # the graphed loss of the first batch is the 2-lane area loss of a full forward's lanes 0 and 1, plus the heads
    with torch.no_grad():
        mc.train()
        x, gt, params, idx, gt_line, gt_horizon = batches[0]
        full = mc(x.cuda().float(), True)
        assert full[3] is not None
        fit, _ = fused_area_loss(full[:2], params.cuda(), args.weight_funct, exact=True)
        want_first = (fit * args.weight_fit + (crits[2](full[7], gt_line.cuda()) + crits[3](full[8], gt_horizon.cuda()))
                      * args.weight_class).item()
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    first = engine.train_epoch_bev(batches[:1], mb, ob, *crits, args, 0)
    assert abs(first[0] - want_first) <= 1e-6 * abs(want_first), (first, want_first)
    want = eager_train(batches[:1], ma, oa, crits[2], crits[3], args, 2)
    assert first == want, (first, want)
    want = eager_train(batches[1:], ma, oa, crits[2], crits[3], args, 2)
    got = engine.train_epoch_bev(batches[1:], mb, ob, *crits, args, 1)
    assert got == want, (got, want)
    assert mb.fit_lanes is None
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    # validation right after: what it returns without the flag
    golden = np.load(os.path.join(GOLDEN, "bev_clas.npz"))
    vb = tc.batches_of(paths, args, "valid")
    tc.write_validation_set(paths[0], golden, max(int(b[6].max()) for b in vb) + 1)
    plain = tc.make_args(paths[0])
    want_v = inference.validate_bev(tc.Listed(vb), mb, *crits, L.get_homography(args.resize), args)
    mb.fit_lanes = 2                    # an eval forward fits every lane whatever fit_lanes holds
    try:
        got_v = inference.validate_bev(tc.Listed(vb), mb, *crits, L.get_homography(args.resize), args)
    finally:
        mb.fit_lanes = None
    assert got_v == want_v and got_v[0] > 0
    # from epoch E on: today's epoch, bit for bit
    mc.load_state_dict(mb.state_dict())
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    oc = nu.define_optim("adam", mc.parameters(), 1e-3, 0, fused=True)
    assert engine.train_epoch_bev(batches, mb, ob, *crits, args, 3) == engine.train_epoch_bev(batches, mc, oc, *crits,
                                                                                              plain, 3)
    for (k, a), b in zip(mb.named_parameters(), mc.parameters()):
        assert torch.equal(a, b), k
