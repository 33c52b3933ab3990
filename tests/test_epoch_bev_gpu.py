"""The bird's-eye-view loop on the GPU: lf_area_loss against its host twin (bit for bit) and float64 autograd of the oracle;
the 4-lane masks of BEV/main.py:226-234 changing nothing; inference.validate_bev and engine.train_epoch_bev against eager
restatements of Birds_Eye_View_Loss/main.py:362-501 and :186-295 on device batches of the BEV loader over a small
synthetic directory; no host synchronisation between reporting points."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import GOLDEN
from lanedetection_end2end_b200 import _capi, engine, inference
from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
from lanedetection_end2end_b200.bev.Loss_crit import define_loss_crit, fused_area_loss, polynomial
from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
from lanedetection_end2end_b200.Loss_crit import AREA_WEIGHTS
from lanedetection_end2end_b200.Networks import utils as nu
from oracle import lsq_oracle as lo

pytestmark = pytest.mark.gpu
BATCH = 2
CASES = {"l2": (2, True), "l4": (4, True), "seg2": (2, False)}       # nclasses, end_to_end


class AverageMeter:          # BEV/Networks/utils.py AverageMeter
    def __init__(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _inputs(B, seed, absent=True):
    g = np.random.default_rng(seed)
    beta = (g.normal(size=(B, 4, 3)) * 0.5).astype(np.float32)
    params = (g.normal(size=(B, 4, 3)) * 0.5).astype(np.float32)
    if absent and B > 1:
        params[0, 2:] = 0.0                 # lanes 2 and 3 absent in image 0
        params[B - 1, 1, 1] = 0.0           # one zero coefficient: lane 1 absent in the last image
    return beta, params


def _run(beta, params, L, wf, device):
    B = beta.shape[0]
    beta = np.ascontiguousarray(beta[:, :L])
    if device:
        b, p = torch.from_numpy(beta).cuda(), torch.from_numpy(params).cuda()
        out = torch.full((2 + B * L * 3 + B,), 7.0, device="cuda")
        ptr = _capi.ptr
        _capi.call("lf_area_loss", ptr(b), ptr(p), B, L, AREA_WEIGHTS[wf], ptr(out[0:1]), ptr(out[2:2 + B * L * 3]),
                   ptr(out[2 + B * L * 3:]), ptr(out[1:2]), _capi.stream_ptr())
        return out.cpu().numpy()
    out = np.full(2 + B * L * 3 + B, 7.0, np.float32)
    a = lambda k: out[k:].ctypes.data
    rc = _capi.lib().lf_area_loss_host(beta.ctypes.data, params.ctypes.data, B, L, AREA_WEIGHTS[wf], a(0), a(2),
                                       a(2 + B * L * 3), a(1))
    assert rc == 0
    return out


@pytest.mark.parametrize("wf", sorted(AREA_WEIGHTS))
@pytest.mark.parametrize("L", [2, 4])
@pytest.mark.parametrize("B", [1, 3, 32, 300])
def test_kernel_bit_identical_to_host_twin(B, L, wf):
    """loss, dbeta, exact and exact_mean: the same bits from the kernel and the host twin (B = 300 > the CTA's threads)."""
    beta, params = _inputs(B, 10 * B + L)
    assert _run(beta, params, L, wf, True).tobytes() == _run(beta, params, L, wf, False).tobytes()
    params[:] = 0.0                         # no lane present anywhere: loss and gradient 0
    got = _run(beta, params, L, wf, True)
    assert got.tobytes() == _run(beta, params, L, wf, False).tobytes()
    assert got[0] == 0.0 and not got[2:2 + B * L * 3].any()


def test_kernel_exact_bit_identical_to_reference_golden():
    z = np.load(os.path.join(GOLDEN, "bev_exact_area.npz"))
    for case in sorted({k.split("/")[0] for k in z.files}):
        beta, params = z[case + "/beta"], z[case + "/params"]
        B = beta.shape[0]
        got = _run(beta, params, 2, "none", True)
        assert got[2 + B * 6:].tobytes() == z[case + "/exact"].tobytes(), case
        mean = float(z[case + "/mean"])
        assert abs(float(got[1]) - mean) <= B * 2 ** -24 * abs(mean), case


@pytest.mark.parametrize("wf", sorted(AREA_WEIGHTS))
@pytest.mark.parametrize("L", [2, 4])
def test_gradient_matches_float64_autograd_of_the_oracle(L, wf):
    beta, params = _inputs(8, L)
    bt = [torch.from_numpy(beta[:, l, :, None].copy()).cuda().requires_grad_(True) for l in range(L)]
    p = torch.from_numpy(params).cuda()
    loss, exact = fused_area_loss(bt, p, wf)
    assert exact is None
    loss.backward()
    b64 = [torch.from_numpy(beta[:, l, :, None].astype(np.float64)).requires_grad_(True) for l in range(L)]
    ref = sum(lo.area_loss(b64[l], torch.from_numpy(params[:, l].astype(np.float64)), 2, wf) for l in range(L))
    ref.backward()
    ref = float(ref.detach())
    assert abs(float(loss) - ref) <= 2 ** -24 * abs(ref) + 1e-12, (float(loss), ref)
    for l in range(L):
        g, gr = bt[l].grad.double().cpu(), b64[l].grad
        assert float((g - gr).abs().max()) <= 2 ** -24 * float(gr.abs().max()) + 1e-12, l


def test_four_lane_mask_product_changes_nothing():
    """main.py:226-234 multiply beta2 / beta3 by the images' presence masks before the criterion; Area_Loss selects the
    same images, so the value and the gradient stay the same (eager Area_Loss and the fused loss alike)."""
    beta, params = _inputs(6, 5)
    params[2, 2] = 0.0
    params[4, 3, 0] = 0.0
    p = torch.from_numpy(params).cuda()
    crit = define_loss_crit(nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y"]))[0]
    res = []
    for masked in (False, True):
        bt = [torch.from_numpy(beta[:, l, :, None].copy()).cuda().requires_grad_(True) for l in range(4)]
        use = list(bt)
        if masked:
            for l in (2, 3):
                mask = torch.prod(p[:, l] != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(bt[l]).type(torch.FloatTensor).cuda()
                use[l] = bt[l] * mask
        fused, _ = fused_area_loss(use, p, "none")
        eager = sum(crit(use[l], p[:, l]) for l in range(4))
        (fused + eager).backward()
        res.append((float(fused), float(eager), [b.grad.clone() for b in bt]))
    (f0, e0, g0), (f1, e1, g1) = res
    assert f0 == f1 and e0 == e1
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# the loops

@pytest.fixture(scope="module")
def paths(tmp_path_factory):
    """16 files over the BEV fixture's two frames and two labelled maps, label files of 16 rows."""
    tmp = str(tmp_path_factory.mktemp("bev_epoch"))
    z = np.load(os.path.join(GOLDEN, "loader_bev.npz"))
    for d in ("img", "gt", "Labels"):
        os.makedirs(os.path.join(tmp, d))
    rows = [json.loads(line) for line in z["params_jsonl"].tobytes().decode().splitlines()]
    lines = [json.loads(line) for line in z["lines_jsonl"].tobytes().decode().splitlines()]
    n = 16
    for k in range(1, n + 1):
        open(os.path.join(tmp, "img", "%d.jpg" % k), "wb").write(z["jpeg/%d" % (k % 2)].tobytes())
        open(os.path.join(tmp, "gt", "%d.png" % k), "wb").write(z["png/%d" % (k % 2)].tobytes())
    for name, src in (("params.json", rows), ("lines.json", lines)):
        with open(os.path.join(tmp, "Labels", name), "w") as f:
            for k in range(n):
                f.write(json.dumps(src[k % len(src)]) + "\n")
    return tmp, n


def make_args(case, tmp):
    nl, e2e = CASES[case]
    args = nu.define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(nl), "--order", "2",
                                        "--batch_size", str(BATCH), "--end_to_end", str(e2e), "--loss_policy", "area"])
    args.save_path = tmp
    return args


def batches_of(paths, args, split):
    tmp, n = paths
    torch.manual_seed(0)
    train, valid, _ = L.get_loader(n, os.path.join(tmp, "Labels", "params.json"), os.path.join(tmp, "img"),
                                   os.path.join(tmp, "gt"), False, BATCH, True, 0, args.end_to_end, args.resize, 0.25,
                                   expected_count=None, line_file=os.path.join(tmp, "Labels", "lines.json"))
    loader = train if split == "train" else valid
    return [tuple(t.clone() for t in b) for b in loader]


def lane_prior(mod, inp, out):
    """--end_to_end False: a constant vertical band per lane class on the untrained decoder's logits gives both lane maps
    pixels on every row (no singular fit)."""
    prior = torch.zeros_like(out[1][:1])
    for k in range(prior.shape[1] - 1):
        prior[:, k + 1, :, 128 * k + 160:128 * k + 200] = 100.0
    return out[0], out[1] + prior


def make_model(args, seed=0):
    torch.manual_seed(seed)
    model = Net(args).cuda()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0.0                # no RNG draws: eager and graphed runs see the same masks
    if not args.end_to_end:
        model.net.register_forward_hook(lane_prior)
    return model


def criteria(args):
    crit, crit_seg = define_loss_crit(args)
    return crit, crit_seg, nn.CrossEntropyLoss().cuda(), nn.BCEWithLogitsLoss().cuda()


class Singular:
    """Zeroes image 0's decoder output in the batches listed in `which` (an all-zero weight map: a singular system)."""

    def __init__(self, model, which):
        self.which, self.scale = set(which), torch.ones(BATCH, 1, 1, 1, device="cuda")
        self.h = model.net.register_forward_hook(lambda mod, inp, out: (out[0], out[1] * self.scale[:out[1].shape[0]]))

    def wrap(self, batches):
        for k, b in enumerate(batches):
            self.scale.fill_(1.0)
            if k in self.which:
                self.scale[0].fill_(0.0)
            yield b


class Listed(list):
    def __init__(self, batches, wrap=None):
        super().__init__(batches)
        self.wrapper = wrap

    def __iter__(self):
        it = super().__iter__()
        return self.wrapper(it) if self.wrapper else it


def exact_cpu(beta0, beta1, gt0, gt1):
    """BEV/main.py:274-280 as written: the reference's polynomial on the CPU."""
    trap_left = polynomial(beta0.cpu()).trapezoidal(polynomial(gt0.cpu()))
    trap_right = polynomial(beta1.cpu()).trapezoidal(polynomial(gt1.cpu()))
    return ((trap_left + trap_right) / 2).mean().item()


def eager_validate(loader, model, criterion, criterion_seg, args):
    """BEV/main.py:362-501 as written (no --clas; no tqdm, no plotting)."""
    losses, avg_area, avg_trapezium_rule = AverageMeter(), AverageMeter(), AverageMeter()
    model.eval()
    model.defer_status_check = False
    skipped = []
    with torch.no_grad():
        for i, (input, gt, params, idx, gt_line, gt_horizon, index) in enumerate(loader):
            input, params = input.cuda(), params.cuda()
            input = input.float()
            gt0, gt1, gt2, gt3 = params[:, 0, :], params[:, 1, :], params[:, 2, :], params[:, 3, :]
            try:
                beta0, beta1, beta2, beta3, weightmap_zeros, M, output_net, outputs_line, outputs_horizon = \
                    model(input, args.end_to_end)
            except RuntimeError:
                skipped.append(idx.tolist())
                continue
            if args.end_to_end:
                loss = criterion(beta0, gt0) + criterion(beta1, gt1)
                if args.nclasses > 3:
                    mask_llhs = torch.prod(gt2 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta2).type(torch.FloatTensor)
                    mask_rrhs = torch.prod(gt3 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta3).type(torch.FloatTensor)
                    beta2 = beta2 * mask_llhs.cuda()
                    beta3 = beta3 * mask_rrhs.cuda()
                    loss += criterion(beta2, gt2) + criterion(beta3, gt3)
            else:
                gt = gt.cuda()
                loss = criterion_seg(output_net, gt)
                area = criterion(beta0, gt0) + criterion(beta1, gt1)
                avg_area.update(area.item(), input.size(0))
            avg_trapezium_rule.update(exact_cpu(beta0, beta1, gt0, gt1), input.size(0))
            losses.update(loss.item(), input.size(0))
    return (losses.avg, avg_area.avg, avg_trapezium_rule.avg, 0, 0), skipped


def _close_to_rounding(got, want, rel):
    return abs(got - want) <= rel * abs(want)


@pytest.mark.parametrize("case", sorted(CASES))
def test_validate_bev_equals_eager_main(paths, case, capsys):
    """validate_bev against the restated eager pass, over the valid loader's batches plus a short last batch: the
    exact-area average within B 2^-24 of it (summation order of the batch means), the loss and area averages within
    float32 rounding of the reference's float32 closed forms, the same skipped batch."""
    args = make_args(case, paths[0])
    batches = batches_of(paths, args, "valid")
    assert len(batches) == 2
    batches.append(tuple(t[:1] for t in batches[0]))
    model = make_model(args).eval()
    crits = criteria(args)
    M_inv = L.get_homography(args.resize)
    for which in ([], [1]):
        sing = Singular(model, which)
        try:
            want, skipped = eager_validate(Listed(batches, sing.wrap), model, crits[0], crits[1], args)
            capsys.readouterr()
            got = inference.validate_bev(Listed(batches, sing.wrap), model, *crits, M_inv, args)
        finally:
            sing.h.remove()
        out = capsys.readouterr().out
        assert skipped == [batches[k][3].tolist() for k in which]
        assert out.count("skipped due to singular matrix") == len(which)
        for k in which:
            assert "Batch with idx {} skipped due to singular matrix".format(batches[k][3].numpy()) in out
        assert got[3:] == (0, 0) and got[2] > 0 and got[0] > 0
        assert abs(got[2] - want[2]) <= BATCH * 2 ** -24 * want[2], (got, want)
        assert _close_to_rounding(got[0], want[0], 1e-5), (got, want)
        assert _close_to_rounding(got[1], want[1], 1e-5) and (got[1] != 0) == (not args.end_to_end), (got, want)


def eager_train(loader, model, optimizer, criterion_seg, args):
    """BEV/main.py:199-295 with the loss of the graph (fused_area_loss) and the exact-area metric of its launch."""
    losses, avg_area, exact_area = AverageMeter(), AverageMeter(), AverageMeter()
    model.train()
    model.defer_status_check = False
    skipped = []
    for i, (input, gt, params, idx, gt_line, gt_horizon) in enumerate(loader):
        input, params = input.cuda().float(), params.cuda()
        try:
            out = model(input, args.end_to_end)
        except RuntimeError:
            skipped.append(idx.tolist())
            continue
        if args.end_to_end:
            loss, exact = fused_area_loss(out[:args.nclasses], params, args.weight_funct, exact=True)
        else:
            loss = criterion_seg(out[6], gt.cuda())
            with torch.no_grad():
                area, exact = fused_area_loss(out[:2], params, args.weight_funct, exact=True)
                avg_area.update(area.item(), input.size(0))
        losses.update(loss.item(), input.size(0))
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        exact_area.update(exact.item(), input.size(0))
    return (losses.avg, avg_area.avg, exact_area.avg), skipped


@pytest.mark.parametrize("case", sorted(CASES))
def test_train_epoch_bev_equals_eager_main(paths, case, capsys):
    """One train_epoch_bev against the restated eager loop driven by the same FusedOptimizer class: parameters, optimizer
    state and the three averages bit for bit; then a singular batch leaves the parameters untouched in both."""
    args = make_args(case, paths[0])
    batches = batches_of(paths, args, "train")
    assert len(batches) == 6
    crits = criteria(args)
    ma, mb = make_model(args), make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    want, _ = eager_train(batches, ma, oa, crits[1], args)
    got = engine.train_epoch_bev(batches, mb, ob, *crits, args, 0)
    assert got == want, (got, want)
    assert got[0] > 0 and got[2] > 0 and (got[1] != 0) == (not args.end_to_end)
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    assert sa["param_groups"] == sb["param_groups"] and sa["state"].keys() == sb["state"].keys()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    before = [p.detach().clone() for p in mb.parameters()]
    sings = [Singular(ma, [0]), Singular(mb, [0])]
    try:
        _, skipped = eager_train(Listed(batches[:1], sings[0].wrap), ma, oa, crits[1], args)
        capsys.readouterr()
        got = engine.train_epoch_bev(Listed(batches[:1], sings[1].wrap), mb, ob, *crits, args, 1)
    finally:
        for s in sings:
            s.h.remove()
    assert skipped == [batches[0][3].tolist()] and got == (0, 0, 0)
    assert "Batch with idx {} skipped".format(batches[0][3].numpy()) in capsys.readouterr().out
    for a, b, p in zip(ma.parameters(), mb.parameters(), before):
        assert torch.equal(a, p) and torch.equal(b, p)


def _nosync(batches):
    """The batches with torch's sync debug mode at "error" from the second batch until the pass has consumed the last one
    (the first batch builds the graph, which synchronises)."""
    def gen(it):
        for k, b in enumerate(it):
            if k == 1:
                torch.cuda.set_sync_debug_mode("error")
            yield b
        torch.cuda.set_sync_debug_mode(0)
    return Listed(batches, gen)


def test_no_host_synchronisation_between_reporting_points(paths):
    args = make_args("l4", paths[0])
    args.print_freq = args.save_freq = 1000
    tb, vb = batches_of(paths, args, "train"), batches_of(paths, args, "valid") * 2
    model = make_model(args)
    opt = nu.define_optim("adam", model.parameters(), 1e-3, 0, fused=True)
    crits = criteria(args)
    try:
        engine.train_epoch_bev(_nosync(tb), model, opt, *crits, args, 0)
        inference.validate_bev(_nosync(vb), model, *crits, L.get_homography(args.resize), args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
