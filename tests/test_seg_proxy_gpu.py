"""The proxy segmentation decoder (--seg_proxy) on the GPU: the joint loss, output_seg, beta and every sampled parameter
gradient against the reference modules' float64 goldens; lf_seg_confusion exact against the numpy restatement;
engine.train_epoch against an eager loop bit for bit; inference.validate's proxy metrics against eager restatements; the
weight packer, the eval-mode BatchNorm fold and the bf16 / fp8 modes on the branch."""
import json
import os

import numpy as np
import pytest
import torch

import test_epoch_gpu as te
from conftest import GOLDEN
from test_epoch_gpu import paths  # noqa: F401  (the synthetic TuSimple directory fixture)
from test_seg_proxy_cpu import confusion_restated
from lanedetection_end2end_b200 import engine, inference, ops_net
from lanedetection_end2end_b200.Loss_crit import (define_loss_crit, fused_backprojection_loss, seg_confusion,
                                                  seg_proxy_loss)
from lanedetection_end2end_b200.Networks import ERFNet
from lanedetection_end2end_b200.Networks import utils as nu
from lanedetection_end2end_b200.Networks.LSQ_layer import Net
from oracle import inputs
from oracle import make_seg_proxy_golden as msg

pytestmark = pytest.mark.gpu
WEIGHT = 0.5


# ---------------------------------------------------------------------------------------------------------------------
# against the reference modules (goldens)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c[0] for c in msg.CASES])
def test_against_reference_goldens(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(g["meta"]))
    L, B, H, W, clas = meta["L"], meta["B"], meta["H"], meta["W"], meta["clas"]
    assert ops_net.CONV_MODE == "tf32x3"
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(L), "--order", str(meta["order"]),
                                        "--batch_size", str(B), "--mask_percentage", str(meta["mask_pct"]),
                                        "--loss_policy", "backproject", "--clas", str(int(clas)), "--seg_proxy", "1",
                                        "--weight_seg_proxy", str(meta["weight_seg_proxy"])])
    model = Net(args)
    sd = model.state_dict()
    P = msg.case_params(sd, L, clas)
    assert inputs.sha256_of(*[P[k] for k in sorted(P)]) == str(g["param_sha"])
    ref_sd = {k: (torch.from_numpy(P[k]) if k in P else v) for k, v in sd.items()}     # the reference's float32 state
    assert [(k, list(v.shape)) for k, v in ref_sd.items()] == [tuple(e) for e in json.loads(str(g["state_dict_keys"]))]
    model.load_state_dict(ref_sd, strict=True)
    model = model.cuda().train()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0
    x_np = inputs.make_images(B, H, W, seed=meta["image_seed"])
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=meta["target_seed"])
    gt = torch.from_numpy(g["gt"].astype(np.int64)).cuda()
    line, hor = torch.from_numpy(g["gt_line"]).cuda(), torch.from_numpy(g["gt_horizon"]).cuda()
    xgt, valid = torch.from_numpy(xgt_np).cuda(), torch.from_numpy(valid_np).cuda()
    crit, crit_seg = define_loss_crit(args)
    out = model(torch.from_numpy(x_np).cuda(), line, True)
    betas = [b for b in out[:4] if b is not None]
    loss = sum(crit(betas[l], xgt[:, l], valid[:, l])[0] for l in range(L)) / L
    if clas:
        bce = torch.nn.BCEWithLogitsLoss()
        loss = loss * args.weight_fit + (bce(out[6], line).double() + bce(out[7], hor).double()) * args.weight_class
    total, ce = seg_proxy_loss(loss, crit_seg, out[8], gt, args.weight_seg_proxy)
    total.backward()
    torch.cuda.synchronize()

    # output_seg (sampled), relative to its largest magnitude
    seg = out[8].detach().double().cpu().contiguous().numpy().reshape(-1)
    e = gate_rel(seg, g, "act_%s/output_seg", 1e-4)
    assert e[2], ("output_seg", e)
    ours_b = torch.stack([b.squeeze(-1) for b in betas], 1).detach().cpu().numpy()
    nw = lambda a, b: float((np.abs(a - b).max(-1) / np.abs(b).max(-1)).max())
    eb, rb = nw(ours_b, g["beta_f64"]), nw(g["beta_f32"], g["beta_f64"])
    assert eb <= 4 * rb + 1e-4, ("beta", eb, rb)
    l64, l32 = float(g["loss_f64"]), float(g["loss_f32"])
    el, rl = abs(float(total.detach()) - l64) / abs(l64), abs(l32 - l64) / abs(l64)
    assert el <= 4 * rl + 1e-4, ("loss", el, rl)
    assert abs(float(ce) - float(g["ce_f64"])) / float(g["ce_f64"]) <= 1e-4
    gscale = max(g[k][2] for k in g.files if k.startswith("grad_f64/") and k.endswith("/stat"))
    no_grad = set(json.loads(str(g["params_without_grad"])))
    seen = set()
    for n, p in model.named_parameters():
        if n in no_grad:
            assert p.grad is None, n
            continue
        got = p.grad.double().cpu().numpy().reshape(-1)
        r = gate_rel(got, g, "grad_%s/" + n, 1e-3, floor=1e-6 * gscale)
        assert r[2], ("gradient", n, r)
        seen.add(n.split(".")[1] if n.startswith("net.") else n.split(".")[0])
    assert {"encoder", "decoder"} <= seen
    assert any(n.startswith("net.decoder.layers1.") for n, p in model.named_parameters() if p.grad is not None)


def gate_rel(flat, g, key, tol, floor=0.0):
    """(|ours - fp64|, |ref fp32 - fp64|, passes) over the sampled entries of ``flat``, relative to the fp64 tensor's
    largest magnitude (golden_check's norm-wise gate)."""
    k64, k32 = key % "f64", key % "f32"
    scale = max(g[k64 + "/stat"][2], floor)
    got = flat[g[k64 + "/idx"]]
    e_ours = float(np.abs(got - g[k64 + "/val"]).max() / scale)
    e_ref = float(np.abs(g[k32 + "/val"] - g[k64 + "/val"]).max() / scale)
    return e_ours, e_ref, e_ours <= 4 * e_ref + tol


# ---------------------------------------------------------------------------------------------------------------------
# lf_seg_confusion
# ---------------------------------------------------------------------------------------------------------------------
def _confusion(x, t, status=None, counts=None):
    C = x.shape[1]
    if counts is None:
        counts = torch.zeros(C * C, dtype=torch.int64, device="cuda")
    return seg_confusion(x, t, counts, status)


@pytest.mark.parametrize("C", [3, 5])
@pytest.mark.parametrize("B,H,W", [(1, 7, 13), (4, 64, 96), (32, 256, 512)])
def test_confusion_exact_against_restatement(C, B, H, W):
    rng = np.random.default_rng(C * 1000 + B)
    x = rng.integers(-3, 4, size=(B, C, H, W)).astype(np.float32)        # small integers: many ties
    x[rng.random(x.shape) < 0.05] = np.nan
    t = rng.integers(-1, C + 3, size=(B, H, W))                          # out-of-range targets on both sides
    t[rng.random(t.shape) < 0.02] = -100
    want = confusion_restated(x, t)
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    got = _confusion(xd, td)
    np.testing.assert_array_equal(got.cpu().numpy(), want)
    again = _confusion(xd, td)
    assert torch.equal(again, got)                                      # repeated launches are identical
    _confusion(xd, td, counts=again)
    assert torch.equal(again, 2 * got)                                  # counts accumulate
    st = torch.full((1,), 3, dtype=torch.int32, device="cuda")
    _confusion(xd, td, status=st, counts=again)
    assert torch.equal(again, 2 * got)                                  # a nonzero status word counts nothing
    st.zero_()
    _confusion(xd, td, status=st, counts=again)
    assert torch.equal(again, 3 * got)


def test_confusion_in_a_graph():
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.standard_normal((2, 3, 32, 64)).astype(np.float32)).cuda()
    t = torch.from_numpy(rng.integers(0, 3, size=(2, 32, 64))).cuda()
    counts = torch.zeros(9, dtype=torch.int64, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _confusion(x, t, st, counts)
    torch.cuda.current_stream().wait_stream(s)
    counts.zero_()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        _confusion(x, t, st, counts)
    counts.zero_()
    gr.replay()
    gr.replay()
    want = confusion_restated(x.cpu().numpy(), t.cpu().numpy())
    np.testing.assert_array_equal(counts.cpu().numpy(), 2 * want)


# ---------------------------------------------------------------------------------------------------------------------
# engine.train_epoch and inference.validate
# ---------------------------------------------------------------------------------------------------------------------
def _proxy_args(case, tmp, *extra):
    args = te.make_args(case, tmp)
    args.seg_proxy, args.weight_seg_proxy = True, WEIGHT
    for k, v in extra:
        setattr(args, k, v)
    return args


def eager_train_proxy(loader, model, optimizer, criterion, criterion_seg, criterion_line_class, criterion_horizon, args):
    """main.py's training loop with the fused fit loss and the proxy term: the joint loss of seg_proxy_loss."""
    losses, ces = te.AverageMeter(), te.AverageMeter()
    model.train()
    model.defer_status_check = False
    for i, (input, gt, lanes, idx, gt_line, gt_horizon, valid_points) in enumerate(loader):
        input, lanes, valid_points, gt = input.cuda(), lanes.cuda(), valid_points.cuda(), gt.cuda().squeeze(1)
        out = model(input, gt_line, True, gt=gt)
        loss, _ = fused_backprojection_loss(criterion, out[:args.nclasses], lanes, valid_points)
        if args.clas:
            gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
            loss_horizon = criterion_horizon(out[7], gt_horizon).double()
            loss_line = criterion_line_class(out[6], gt_line).double()
            loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        loss, ce = seg_proxy_loss(loss, criterion_seg, out[8], gt.long(), args.weight_seg_proxy)
        losses.update(loss.item(), input.size(0))
        ces.update(ce.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
    return losses.avg, ces.avg


@pytest.mark.parametrize("case,extra", [("plain2", ()), ("clas4", ()), ("clas4", (("learn_homography", True),))],
                         ids=["plain2", "clas4", "clas4_homography"])
def test_train_epoch_equals_eager_loop(paths, case, extra):
    """One graphed train_epoch against the eager loop on the joint loss and the same FusedOptimizer class: parameters
    (layers1 among them), optimizer state, losses.avg and the proxy term's average bit for bit."""
    args = _proxy_args(case, paths[0], *extra)
    train, _, _ = te.loaders(paths, args)
    batches = list(train)
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    mb.load_state_dict(ma.state_dict())
    assert ma.seg_proxy and any(".layers1." in n for n, _ in ma.named_parameters())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    if args.learn_homography:
        crits[0].bind(ma)
    # the branch's weights (its conv biases in front of a training-mode BatchNorm get exactly zero gradient)
    b0 = [p.detach().clone() for n, p in ma.named_parameters() if ".layers1." in n and p.dim() == 4]
    want_loss, want_ce = eager_train_proxy(batches, ma, oa, *crits, args)
    seg = {}
    got_loss, _ = engine.train_epoch(batches, mb, ob, *crits, args, 0, seg_metrics=seg)
    assert got_loss == want_loss and seg["ce"] == want_ce, (got_loss, want_loss, seg, want_ce)
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    after = [p for n, p in ma.named_parameters() if ".layers1." in n and p.dim() == 4]
    assert len(after) == 19 and all(not torch.equal(p, q) for p, q in zip(after, b0))
    sa, sb = oa.state_dict(), ob.state_dict()
    assert sa["state"].keys() == sb["state"].keys()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)


@pytest.mark.parametrize("case", ["plain2", "clas4"])
def test_validate_proxy_metrics(paths, case, capsys):
    args = _proxy_args(case, paths[0])
    L = args.nclasses
    _, valid, _ = te.loaders(paths, args)
    batches = list(valid)
    batches.append(te.short(batches[0]))
    model = te.make_model(args).eval()
    crits = te.criteria(args)
    want, _ = te.eager_validate(batches, model, *crits, args)
    # eager restatement of the proxy metrics
    counts, ce = np.zeros((L + 1) ** 2, np.int64), te.AverageMeter()
    model.defer_status_check = False
    per_batch = []
    with torch.no_grad():
        for b in batches:
            gt = b[1].cuda().squeeze(1).long()
            out = model(b[0].cuda().float(), b[4], True, gt=gt)
            c = confusion_restated(out[8].cpu().numpy(), gt.cpu().numpy())
            per_batch.append(c)
            counts += c
            ce.update(crits[1](out[8], gt).item(), b[0].shape[0])
    plain = inference.validate(te.Listed(batches), model, *crits, args)
    capsys.readouterr()
    seg = {}
    got = inference.validate(te.Listed(batches), model, *crits, args, seg_metrics=seg)
    printed = capsys.readouterr().out
    assert got == plain == want
    assert seg["confusion"] == counts.reshape(L + 1, L + 1).tolist()
    assert seg["ce"] == ce.avg
    n = counts.reshape(L + 1, L + 1)
    assert seg["pixel_acc"] == float(np.trace(n)) / float(n.sum())
    den = n.sum(0) + n.sum(1) - np.diag(n)
    iou = [float(n[c, c]) / float(den[c]) for c in range(L + 1) if den[c]]
    assert [v for v in seg["iou"] if v == v] == iou and seg["miou"] == sum(iou) / len(iou)
    assert "Proxy segmentation" in printed
    # a batch with a singular system counts nothing
    sing = te.Singular(model, [1])
    try:
        seg_s = {}
        inference.validate(te.Listed(batches, sing.wrap), model, *crits, args, seg_metrics=seg_s)
    finally:
        sing.h.remove()
    assert seg_s["confusion"] == (counts - per_batch[1]).reshape(L + 1, L + 1).tolist()


# ---------------------------------------------------------------------------------------------------------------------
# the library's paths on the branch
# ---------------------------------------------------------------------------------------------------------------------
def test_branch_runs_on_the_library_paths():
    args = te.make_args("plain2", "/tmp")
    args.seg_proxy = True
    torch.manual_seed(0)
    model = Net(args).cuda()
    nu.define_init_weights(model, "kaiming")
    x = torch.rand(2, 3, 256, 512, device="cuda")
    branch = [p for n, p in model.named_parameters() if ".layers1." in n]
    # dropout: the branch's blocks have p = 0 (as the reference's), so the fused mask draw leaves them out
    assert all(m.dropout.p == 0 for m in model.net.decoder.layers1 if isinstance(m, ERFNet.non_bottleneck_1d))
    model.train()
    model(x, torch.zeros(2, 4), True)
    model(x, torch.zeros(2, 4), True)
    packs = model.net._weight_packs
    ptrs = {k[0] for k in packs.entries}
    assert all(p.data_ptr() in packs.by_ptr for p in branch)
    served = [p for p in branch if p.dim() == 4 and p.data_ptr() in ptrs]
    assert len(served) >= 8, len(served)              # the branch's GEMM-layout operands come from the one-launch packer
    # with the main decoder's stage weights copied into the branch, both see the same encoder output: in every mode the
    # branch's last stage must equal the main decoder's bit for bit (the same eval fold, bf16 and fp8 paths)
    for a, b in zip(model.net.decoder.layers, model.net.decoder.layers1):
        b.load_state_dict(a.state_dict())
    taps = {}
    hooks = [model.net.decoder.layers[5].register_forward_hook(lambda m, i, o: taps.__setitem__("main", o.clone())),
             model.net.decoder.layers1[5].register_forward_hook(lambda m, i, o: taps.__setitem__("branch", o.clone()))]
    prev = ops_net.CONV_MODE
    try:
        model.train()
        model(x, torch.zeros(2, 4), True)
        assert torch.equal(taps["main"], taps["branch"]), "train"
        model.eval()
        with torch.no_grad():
            for mode, fused in (("tf32x3", True), ("tf32x3", False), ("bf16", True), ("fp8", True)):
                ops_net.set_conv_mode(mode)
                ERFNet.EVAL_FUSED = fused
                taps.clear()
                out = model(x, torch.zeros(2, 4), True)
                assert torch.isfinite(out[8]).all(), mode
                assert torch.equal(taps["main"], taps["branch"]), (mode, fused)
    finally:
        ERFNet.EVAL_FUSED = True
        ops_net.set_conv_mode(prev)
        for h in hooks:
            h.remove()
