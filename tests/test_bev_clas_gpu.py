"""The bird's-eye-view --clas run on the GPU: the BEV heads against the reference's own (tests/golden/bev_clas.npz,
oracle/make_bev_clas_golden.py) in both fp32-accurate convolution modes; lf_bev_lane_score against write_lsq_results and
LaneEval column for column and bit for bit, eagerly and from a captured graph; validate_bev and train_epoch_bev with --clas
against eager restatements of Birds_Eye_View_Loss/main.py:362-501 and :186-295."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from lanedetection_end2end_b200 import engine, inference
from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
from lanedetection_end2end_b200.bev.Loss_crit import fused_area_loss
from lanedetection_end2end_b200.Networks import utils as nu
from oracle import inputs
from oracle import tusimple_oracle as to
from oracle.make_bev_clas_golden import bev_head_params
from test_epoch_bev_gpu import AverageMeter, Listed, Singular, batches_of, criteria, make_model, paths  # noqa: F401

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "bev_clas.npz"))


@pytest.fixture(params=["tf32x3", "fp32"])
def conv_mode(request):
    from lanedetection_end2end_b200 import ops_net
    ops_net.set_conv_mode(request.param)
    yield request.param


@pytest.mark.parametrize("kind", ["line", "horizon"])
def test_head_matches_reference_golden(golden, kind, conv_mode):
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Classification
    meta = json.loads(str(golden["meta"]))
    m = Classification(kind, size=(32, 64), channels_in=128, resize=256)
    sd = m.state_dict()
    for k, v in bev_head_params(kind, meta["param_seeds"][kind]).items():
        sd[k] = torch.from_numpy(v)
    m.load_state_dict(sd)
    m = m.cuda().train()
    x = torch.from_numpy(inputs.make_encoder_map(2, seed=meta["map_seed"])).cuda().requires_grad_(True)
    y = m(x)
    pre = "heads/%s/" % kind
    assert y.shape == golden[pre + "out_f64"].shape and y.dtype == torch.float32
    (y * torch.from_numpy(golden[pre + "g"]).float().cuda()).sum().backward()
    torch.cuda.synchronize()
    ref64, ref32 = golden[pre + "out_f64"], golden[pre + "out_f32"]
    scale = float(np.abs(ref64).max())
    e_ours = float(np.abs(y.detach().double().cpu().numpy() - ref64).max() / scale)
    assert e_ours <= 4 * float(np.abs(ref32 - ref64).max() / scale) + TOL, (kind, conv_mode, e_ours)
    k = pre + "dx_f64"
    got = x.grad.double().cpu().numpy().reshape(-1)[golden[k + "/idx"]]
    e_ours = float(np.abs(got - golden[k + "/val"]).max() / golden[k + "/stat"][2])
    e_ref = float(np.abs(golden[pre + "dx_f32/val"] - golden[k + "/val"]).max() / golden[k + "/stat"][2])
    assert e_ours <= 4 * e_ref + 10 * TOL, (kind, "dx", e_ours, e_ref)
    gscale = max(golden[q][2] for q in golden.files if q.startswith(pre + "grad_f64/") and q.endswith("/stat"))
    for n, p in m.named_parameters():
        k64, k32 = pre + "grad_f64/" + n, pre + "grad_f32/" + n
        got = p.grad.double().cpu().numpy().reshape(-1)[golden[k64 + "/idx"]]
        scale = max(golden[k64 + "/stat"][2], 1e-6 * gscale)
        e_ours = float(np.abs(got - golden[k64 + "/val"]).max() / scale)
        e_ref = float(np.abs(golden[k32 + "/val"] - golden[k64 + "/val"]).max() / scale)
        assert e_ours <= 4 * e_ref + 10 * TOL, (kind, conv_mode, n, e_ours, e_ref)


def test_net_returns_the_heads_with_the_reference_shapes():
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "2",
                                        "--batch_size", "2", "--loss_policy", "area", "--clas", "True"])
    torch.manual_seed(0)
    model = Net(args).cuda().train()
    out = model(torch.from_numpy(inputs.make_images(2, 256, 512, seed=3)).cuda(), True)
    assert out[7].shape == (2, 3, 4) and out[8].shape == (2, 256)
    (out[7].sum() + out[8].sum()).backward()
    torch.cuda.synchronize()
    for fc in (model.line_classification.fully_connected_line1, model.line_classification.fully_connected_line4):
        assert fc.weight.grad is not None and float(fc.weight.grad.abs().max()) > 0
    assert model(torch.zeros(2, 3, 256, 512, device="cuda"), False)[7] is None


def test_net_with_clas_matches_reference_golden(golden, conv_mode):
    """The 4-lane --clas Net, forward and backward of main.py:222-253's combined loss (the fit loss of the graphed step,
    engine.clas_loss), against the reference's own Net in float32 and float64: beta, line, horizon, the loss and the
    sampled gradients of both heads, the encoder's first and the decoder's last layer."""
    from oracle.make_bev_clas_golden import net_all_params, net_params, net_targets, net_grad_sampled
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    meta = json.loads(str(golden["meta"]))
    B = meta["B"]
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "2",
                                        "--batch_size", str(B), "--loss_policy", "area", "--clas", "True"])
    torch.manual_seed(0)
    model = Net(args)
    sd = model.state_dict()
    for k, v in net_all_params().items():
        if k in sd:
            sd[k] = torch.from_numpy(v)
    model.load_state_dict(sd)
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0.0
    model = model.cuda().train()
    gt_line, gt_horizon = net_targets(B, 256, meta["net_target_seed"])
    st = {"gt_line": torch.from_numpy(gt_line).cuda(), "gt_horizon": torch.from_numpy(gt_horizon).cuda()}
    params = torch.from_numpy(net_params(meta["net_target_seed"])).cuda()
    out = model(torch.from_numpy(inputs.make_images(B, 256, 512, seed=meta["net_image_seed"])).cuda(), True)
    loss, _ = fused_area_loss(out[:4], params, args.weight_funct)
    _, _, crit_line, crit_hor = criteria(args)
    loss = engine.clas_loss(loss, out, st, crit_line, crit_hor, args)
    loss.backward()
    torch.cuda.synchronize()
    got = {"beta": torch.cat(out[:4], 2).transpose(1, 2), "line": out[7], "horizon": out[8], "loss": loss}
    for name, t in got.items():
        ref64, ref32 = golden["net/f64/" + name], golden["net/f32/" + name]
        scale = float(np.abs(ref64).max())
        e_ours = float(np.abs(t.detach().double().cpu().numpy() - ref64).max() / scale)
        e_ref = float(np.abs(ref32 - ref64).max() / scale)
        assert e_ours <= 4 * e_ref + TOL, (name, conv_mode, e_ours, e_ref)
    gkeys = [k[len("net/f64/grad/"):-len("/stat")] for k in golden.files
             if k.startswith("net/f64/grad/") and k.endswith("/stat")]
    assert sorted(gkeys) == sorted(n for n, _ in model.named_parameters() if net_grad_sampled(n))
    gscale = max(golden["net/f64/grad/%s/stat" % n][2] for n in gkeys)
    for n, p in model.named_parameters():
        if n not in gkeys:
            continue
        k64, k32 = "net/f64/grad/" + n, "net/f32/grad/" + n
        g = p.grad.double().cpu().numpy().reshape(-1)[golden[k64 + "/idx"]]
        scale = max(golden[k64 + "/stat"][2], 1e-6 * gscale)
        e_ours = float(np.abs(g - golden[k64 + "/val"]).max() / scale)
        e_ref = float(np.abs(golden[k32 + "/val"] - golden[k64 + "/val"]).max() / scale)
        assert e_ours <= 4 * e_ref + 10 * TOL, (n, conv_mode, e_ours, e_ref)


def _rows(golden):
    return [json.loads(line) for line in golden["score/rows_jsonl"].tobytes().decode().splitlines()]


def _ls_lanes(golden, tag):
    return [json.loads(line)["lanes"] for line in golden[tag + "/ls_bytes"].tobytes().decode().splitlines()]


@pytest.mark.parametrize("no_ortho", [False, True])
@pytest.mark.parametrize("graphed", [False, True])
def test_kernel_equals_write_lsq_results_and_lane_eval(golden, no_ortho, graphed, tmp_path):
    rows, params = _rows(golden), golden["score/params"]
    tag = "score/no_ortho%d" % int(no_ortho)
    N = len(rows)
    s = inference.BevLaneScorer(rows)
    B = 4
    s.begin(N, 256)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    beta = torch.zeros(B, 4, 3, device="cuda")
    idx = torch.zeros(B, dtype=torch.int64, device="cuda")
    line = torch.ones(B, 4, dtype=torch.int64, device="cuda")
    hor = torch.zeros(B, 256, device="cuda")
    run = lambda: s.score(beta, line, hor, idx, status, no_ortho)
    if graphed:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run()                 # recorded only: the slot position and the results stay as begin() left them
        run = g.replay
    for b0 in range(0, N, B):
        beta.copy_(torch.from_numpy(params[b0:b0 + B]))
        idx.copy_(torch.arange(b0, b0 + B))
        run()
    torch.cuda.synchronize()
    lanes = s.lanes.cpu().numpy()
    want = _ls_lanes(golden, tag)
    for i, r in enumerate(rows):
        assert lanes[i, :, :len(r["h_samples"])].tolist() == want[i], i
    assert s.per_row.cpu().numpy().tobytes() == golden[tag + "/per_row"].tobytes()
    acc = s.finish(str(tmp_path / "dst.json"), str(tmp_path / "ls.json"))
    assert acc == golden[tag + "/file"].tolist()
    assert open(tmp_path / "dst.json", "rb").read() == golden["score/dst_bytes"].tobytes()
    assert open(tmp_path / "ls.json", "rb").read() == golden[tag + "/ls_bytes"].tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# the loops

def make_args(tmp):
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "2",
                                        "--batch_size", "2", "--loss_policy", "area", "--clas", "True"])
    args.save_path = tmp
    return args


def write_validation_set(tmp, golden, n):
    """validation_set.json: one row per validation index, the fixture's Curve_parameters rows."""
    rows = _rows(golden)
    with open(os.path.join(tmp, "validation_set.json"), "w") as f:
        for k in range(n):
            r = dict(rows[k % len(rows)], raw_file="clips/%d.jpg" % k)
            f.write(json.dumps(r) + "\n")
    return [json.loads(line) for line in open(os.path.join(tmp, "validation_set.json"))]


def eager_validate(loader, model, criterion, crit_line, crit_hor, args, valid_set_labels):
    """BEV/main.py:362-501 with --clas as written, except that validation_set_dst.json is opened once before the loop."""
    losses, avg_area, avg_trapezium_rule = AverageMeter(), AverageMeter(), AverageMeter()
    acc_hor_tot, acc_line_tot = AverageMeter(), AverageMeter()
    model.eval()
    model.defer_status_check = False
    val_set_path = os.path.join(args.save_path, "eager_dst.json")
    ls_result_path = os.path.join(args.save_path, "eager_ls.json")
    with torch.no_grad(), open(val_set_path, "w") as jsonFile:
        for i, (input, gt, params, idx, gt_line, gt_horizon, index) in enumerate(loader):
            input, params = input.cuda().float(), params.cuda()
            try:
                beta0, beta1, beta2, beta3, _, M, output_net, outputs_line, outputs_horizon = model(input, True)
            except RuntimeError:
                continue
            loss, exact = fused_area_loss([beta0, beta1, beta2, beta3], params, args.weight_funct, exact=True)
            gt_horizon, gt_line = gt_horizon.cuda(), gt_line.cuda()
            horizon_pred = torch.round(torch.nn.Sigmoid()(outputs_horizon))
            acc_hor = torch.sum(torch.eq(horizon_pred, gt_horizon)).float() / (args.resize * args.batch_size)
            acc_hor_tot.update(acc_hor.item())
            _, line_pred = torch.max(outputs_line, 1)
            acc_line = torch.sum(torch.eq(line_pred, gt_line)).float() / (args.nclasses * args.batch_size)
            acc_line_tot.update(acc_line.item())
            loss = loss * args.weight_fit + (crit_line(outputs_line, gt_line) + crit_hor(outputs_horizon, gt_horizon)) \
                * args.weight_class
            avg_trapezium_rule.update(exact.item(), input.size(0))
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
    return (losses.avg, avg_area.avg, avg_trapezium_rule.avg, acc_hor_tot.avg, acc_line_tot.avg), acc_seg


def test_validate_bev_with_clas_equals_eager_main(paths, golden, capsys):
    tmp = paths[0]
    args = make_args(tmp)
    batches = batches_of(paths, args, "valid")
    n_valid = max(int(b[6].max()) for b in batches) + 1
    model = make_model(args).eval()
    crits = criteria(args)
    for which in ([], [1]):
        labels = write_validation_set(tmp, golden, n_valid)
        sing = Singular(model, which)
        try:
            want, acc_seg = eager_validate(Listed(batches, sing.wrap), model, crits[0], crits[2], crits[3], args, labels)
            capsys.readouterr()
            got = inference.validate_bev(Listed(batches, sing.wrap), model, *crits, L.get_homography(args.resize), args)
        finally:
            sing.h.remove()
        out = capsys.readouterr().out
        assert got == want, (got, want)
        assert got[3] > 0 and got[4] > 0
        for a, b in (("validation_set_dst.json", "eager_dst.json"), ("ls_result.json", "eager_ls.json")):
            assert open(os.path.join(tmp, a), "rb").read() == open(os.path.join(tmp, b), "rb").read(), a
        n_rows = len(open(os.path.join(tmp, "validation_set_dst.json")).readlines())
        assert n_rows == sum(b[0].shape[0] for k, b in enumerate(batches) if k not in which)
        assert "===> Average ACC_SEG on val is {:.8}".format(acc_seg[0]) in out


def eager_train(loader, model, optimizer, crit_line, crit_hor, args):
    """BEV/main.py:199-295 with --clas, the fit loss of the graph (fused_area_loss)."""
    losses, avg_area, exact_area = AverageMeter(), AverageMeter(), AverageMeter()
    model.train()
    model.defer_status_check = False
    for i, (input, gt, params, idx, gt_line, gt_horizon) in enumerate(loader):
        input, params = input.cuda().float(), params.cuda()
        out = model(input, True)
        loss, exact = fused_area_loss(out[:4], params, args.weight_funct, exact=True)
        loss = loss * args.weight_fit + (crit_line(out[7], gt_line.cuda()) + crit_hor(out[8], gt_horizon.cuda())) \
            * args.weight_class
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        exact_area.update(exact.item(), input.size(0))
    return losses.avg, avg_area.avg, exact_area.avg


def test_train_epoch_bev_with_clas_equals_eager_main(paths):
    args = make_args(paths[0])
    batches = batches_of(paths, args, "train")
    crits = criteria(args)
    ma, mb = make_model(args), make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    want = eager_train(batches, ma, oa, crits[2], crits[3], args)
    got = engine.train_epoch_bev(batches, mb, ob, *crits, args, 0)
    assert got == want, (got, want)
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)


def test_no_host_synchronisation_between_reporting_points(paths, golden):
    args = make_args(paths[0])
    args.print_freq = args.save_freq = 1000
    tb, vb = batches_of(paths, args, "train"), batches_of(paths, args, "valid")
    write_validation_set(paths[0], golden, max(int(b[6].max()) for b in vb) + 1)
    model = make_model(args)
    opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True)
    crits = criteria(args)

    def nosync(batches):
        def gen(it):
            for k, b in enumerate(it):
                if k == 1:
                    torch.cuda.set_sync_debug_mode("error")
                yield b
            torch.cuda.set_sync_debug_mode(0)
        return Listed(batches, gen)
    try:
        engine.train_epoch_bev(nosync(tb), model, opt, *crits, args, 0)
        inference.validate_bev(nosync(vb * 2), model, *crits, L.get_homography(args.resize), args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
