"""--trapezium_mask on the H100: the masked least-squares layer against the reference modules' float64 fixtures
(tests/golden/trapezium_*.npz, oracle/make_trapezium_golden.py), the *_keep entry points entry by entry against the
fp64 / exact contract of tests/lsq_contract.py over every kernel instantiation, an all-ones keep map against the plain
entry points bit for bit, and the flag through the graphed training epoch, validation, the eval-mode forward in every
convolution mode and test_model."""
import json
import os
import numpy as np
import pytest
import torch

import lsq_contract as lc
import lsq_tables_contract as tc
from conftest import GOLDEN
from test_epoch_gpu import paths  # noqa: F401  (the synthetic TuSimple directory fixture)
from test_lsq_contract_gpu import GUARD, SENT, SENT64, Workspace, _check, _guarded
from oracle.make_trapezium_golden import CASES, case_dict, case_inputs

from lanedetection_end2end_b200 import _capi, ops_lsq
from lanedetection_end2end_b200.Networks.utils import define_args

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _args(*extra, L=4, B=2):
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", str(L), "--batch_size", str(B),
                                     "--trapezium_mask", "True"] + list(extra))


def normwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float((np.abs(a - b).max(-1) / np.abs(b).max(-1)).max())


# ---------------------------------------------------------------------------------------------------------------------
# the reference modules' fixtures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_masked_fit_matches_reference_golden(case):
    """beta, masked, the loss, d_o and (warp case) dL/dtheta through the Net's own keep map and least-squares call, under
    the gates of the lsq_*.npz fixtures: |ours - fp64| <= 1e-4 max|fp64| and within the reference fp32's own error."""
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net as BevNet
    c = case_dict(case)
    z = np.load(os.path.join(GOLDEN, c["name"] + ".npz"))
    o_np, g_np = case_inputs(c)
    assert lc_sha(o_np, g_np) == str(z["input_sha"])
    bp = c["variant"] == "Backprojection_Loss"
    extra = ["--resize", str(c["resize"]), "--mask_percentage", str(c["mask_pct"]), "--order", str(c["order"]),
             "--activation_layer", c["act"], "--reg_ls", str(c["reg_ls"])] + list(c["flags"])
    if c["warp"]:
        extra += ["--learn_homography", "True", "--loss_policy", "backproject"]
    torch.manual_seed(0)
    net = (Net if bp else BevNet)(_args(*extra, L=c["L"])).cuda()
    np.testing.assert_array_equal(net.keep.cpu().numpy(), z["keep"])
    o = torch.from_numpy(o_np).cuda().requires_grad_(True)
    keep = net.keep
    if c["warp"]:
        with torch.no_grad():
            net.homography.offsets.copy_(torch.from_numpy(z["theta"]))
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        beta, masked = net._lsq_warp(o, net.homography(st), net.zero_rows, c["act"], True, st, True, keep)
    elif bp:
        beta, masked = net.ls_layer.forward_all(o, net.grid[:o.shape[0]], mask_rows=net.zero_rows, act=c["act"],
                                                want_masked=True, keep=keep)
    else:
        grid = net.project_layer(net.M.cuda())[:o.shape[0]]
        beta, masked = net.ls_layer.forward_all(o, grid, mask_rows=net.zero_rows, act=c["act"], want_masked=True,
                                                keep=keep)
    ours = beta.detach().cpu().numpy()
    b64, b32 = z["beta_f64"], z["beta_f32"]
    e_ours, e_ref = normwise(ours, b64), normwise(b32, b64)
    print("%s: beta |ours - f64| %.2e, |ref32 - f64| %.2e" % (c["name"], e_ours, e_ref))
    assert e_ours <= 1e-4, (e_ours, e_ref)
    assert normwise(ours, b32) <= e_ref + 1e-4
    # masked: act(o) * keep, +0.0 at every masked pixel
    m = masked.cpu().numpy()
    assert not m[..., z["keep"] == 0].any()
    got = m.reshape(-1).astype(np.float64)[z["masked_f64/idx"]]
    np.testing.assert_allclose(got, z["masked_f64/val"], rtol=2e-6, atol=1e-7 * z["masked_f64/stat"][2])
    loss = (beta * torch.from_numpy(g_np).cuda()).sum()
    l64, l32 = float(z["loss_f64"]), float(z["loss_f32"])
    assert abs(loss.item() - l64) <= 4 * abs(l32 - l64) + 1e-6 * abs(l64), (loss.item(), l64, l32)
    loss.backward()
    d_o = o.grad.cpu().numpy()
    assert not d_o[..., z["keep"] == 0].any()
    flat = d_o.reshape(-1).astype(np.float64)
    idx, val, stat = z["grad_f64/idx"], z["grad_f64/val"], z["grad_f64/stat"]
    assert np.abs(flat[idx] - val).max() <= 1e-4 * stat[2]
    # (the learned warp's fp32 device tables against the reference's float64 warp: 1.3e-5 measured on the norm)
    assert abs(np.sqrt((flat * flat).sum()) - stat[3]) <= (1e-4 if c["warp"] else 1e-5) * stat[3]
    if c["warp"]:
        # the reference fp32 chain's own distance from fp64 sets the scale, as for beta
        gt = net.homography.offsets.grad.double().cpu().numpy()
        ref, ref32 = z["gtheta_f64"], z["gtheta_f32"]
        err, err32 = np.linalg.norm(gt - ref), np.linalg.norm(ref32 - ref)
        print("%s: theta.grad |ours - f64| %.2e, |ref32 - f64| %.2e, |f64| %.2e" % (c["name"], err, err32,
                                                                                      np.linalg.norm(ref)))
        assert err <= max(1e-4 * np.linalg.norm(ref), 4 * err32), (gt, ref, ref32)


def lc_sha(o, g):
    from oracle import inputs
    return inputs.sha256_of(o, g)


# ---------------------------------------------------------------------------------------------------------------------
# the entry points against the fp64 / exact contract
# ---------------------------------------------------------------------------------------------------------------------
def _keep(H, W, seed):
    """A keep map with isolated holes, whole masked columns and a masked corner: about 30 % of the pixels zeroed."""
    rng = np.random.default_rng(seed)
    k = (rng.uniform(size=(H, W)) > 0.2).astype(np.uint8)
    k[:, 1:min(3, W)] = 0
    k[:H // 3, W - W // 4:] = 0
    k[k != 0] = rng.integers(1, 256, size=int((k != 0).sum()))         # any nonzero byte keeps the pixel
    return k


def _zeroed(o, keep, act):
    """o with the masked pixels replaced by a value whose activation is exactly 0 in the contract's fp64 act64."""
    fill = -np.inf if lc.ACTS[act] in ("sigmoid", "softplus") else 0.0
    return np.where(keep[None, None] != 0, o, fill)


def _fwd_keep(o_t, c, xt, ytt, yrt, keep_t, rowsums=False):
    B, L, H, W, n = c["B"], c["L"], c["H"], c["W"], c["order"] + 1
    beta = _guarded(B * L * n, torch.float64, SENT64)
    zinv = _guarded(B * L * n * n, torch.float64, SENT64)
    masked = _guarded(B * L * H * W, torch.float32, SENT)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    h = _capi.lib()
    need = h.lf_lsq_workspace_bytes(B, L, H, W, c["order"])
    ws = Workspace(need)
    p = lambda t: None if t is None else t.data_ptr()
    if rowsums:
        rs = torch.full((B, L, H, 3), SENT, dtype=torch.float32, device=DEV)
        rc = h.lf_lsq_fwd_rowsums_keep(p(o_t), c["dtype"], p(xt), p(yrt), p(keep_t), B, L, H, W, c["order"],
                                       c["mask_rows"], c["act"], c["reg_ls"], c["solver"], beta[GUARD:].data_ptr(),
                                       zinv[GUARD:].data_ptr(), masked[GUARD:].data_ptr(), status.data_ptr(), rs.data_ptr(),
                                       ws.ptr(), need, _capi.stream_ptr())
    else:
        rc = h.lf_lsq_fwd_keep(p(o_t), c["dtype"], p(xt), p(ytt), p(yrt), p(keep_t), B, L, H, W, c["order"],
                               c["mask_rows"], c["act"], c["reg_ls"], c["solver"], beta[GUARD:].data_ptr(),
                               zinv[GUARD:].data_ptr(), masked[GUARD:].data_ptr(), status.data_ptr(), ws.ptr(), need,
                               _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (c["name"], rc)
    for buf, sent, what in ((beta, SENT64, "beta"), (zinv, SENT64, "zinv"), (masked, SENT, "masked")):
        _check(buf, sent, c["name"], what)
    ws.check(c["name"])
    out = (beta[GUARD:-GUARD].cpu().numpy().reshape(B, L, n), zinv[GUARD:-GUARD].cpu().numpy().reshape(B, L, n, n),
           masked[GUARD:-GUARD].cpu().view(B, L, H, W), int(status.item()))
    return out + ((rs.cpu(),) if rowsums else ())


def _bwd_keep(o_t, c, xt, ytt, yrt, keep_t, beta, zinv, g):
    B, L, H, W = c["B"], c["L"], c["H"], c["W"]
    odt = torch.bfloat16 if c["dtype"] == lc.LF_BF16 else torch.float32
    d_o = _guarded(B * L * H * W, odt, SENT)
    bt, zt, gt = (torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(DEV) for v in (beta, zinv, g))
    p = lambda t: None if t is None else t.data_ptr()
    rc = _capi.lib().lf_lsq_bwd_keep(p(o_t), c["dtype"], p(xt), p(ytt), p(yrt), p(keep_t), B, L, H, W, c["order"],
                                     c["mask_rows"], c["act"], bt.data_ptr(), zt.data_ptr(), gt.data_ptr(),
                                     d_o[GUARD:].data_ptr(), _capi.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0, (c["name"], rc)
    _check(d_o, SENT, c["name"], "d_o")
    return d_o[GUARD:-GUARD].float().cpu().numpy().reshape(B, L, H, W).astype(np.float64)


def _operands(c, seed=0):
    o, xtab, ytab, yrow = lc.case_operands(c, seed)
    o_t = torch.from_numpy(np.ascontiguousarray(o, np.float32)).to(DEV)
    if c["dtype"] == lc.LF_BF16:
        o_t = o_t.bfloat16()
    xt, ytt = torch.from_numpy(xtab).to(DEV), torch.from_numpy(ytab).to(DEV)
    yrt = torch.from_numpy(yrow).to(DEV) if c["yrow"] else None
    return o_t, xt, ytt, yrt, xtab, ytab, yrow


@pytest.mark.parametrize("case", lc.COVERAGE, ids=[c[0] for c in lc.COVERAGE])
def test_keep_entry_points_against_fp64(case):
    c = lc.case_dict(case)
    o_t, xt, ytt, yrt, xtab, ytab, yrow = _operands(c)
    H, W = c["H"], c["W"]
    keep = _keep(H, W, sum(map(ord, c["name"])))
    keep_t = torch.from_numpy(keep).to(DEV)
    plan = lc.query_plan(0, c["dtype"], c["yrow"], True, c["B"], c["L"], H, W, c["order"], c["mask_rows"], c["act"])[1]
    bplan = lc.query_plan(1, c["dtype"], c["yrow"], True, c["B"], c["L"], H, W, c["order"], c["mask_rows"], c["act"])[1]
    beta, zinv, masked, st = _fwd_keep(o_t, c, xt, ytt, yrt, keep_t)
    assert st == 0, (c["name"], st)
    o_exact = o_t.float().cpu().numpy().astype(np.float64)
    ref = lc.forward_reference(_zeroed(o_exact, keep, c["act"]), xtab, yrow if plan["rowsep"] else ytab, H, W,
                               c["order"], c["mask_rows"], c["act"], c["reg_ls"], plan["rowsep"], plan["nchunks"],
                               c["dtype"])
    assert float(ref["rho"].max()) <= lc.RHO_MAX
    exc = lc.forward_excess(beta, zinv, ref)
    assert exc <= 1.0, "%s: beta / Z^-1 outside the gate (%.3g)" % (c["name"], exc)
    # the fit must see the keep map: the unmasked fit is outside the gate
    ref_open = lc.forward_reference(o_exact, xtab, yrow if plan["rowsep"] else ytab, H, W, c["order"], c["mask_rows"],
                                    c["act"], c["reg_ls"], plan["rowsep"], plan["nchunks"], c["dtype"])
    if c["mask_rows"] < H:
        assert lc.forward_excess(beta, zinv, dict(ref_open, bound_beta=ref["bound_beta"],
                                                  bound_zinv=ref["bound_zinv"])) > 1.0
    # masked: +0.0 at every masked pixel and row, the activation elsewhere
    live = np.zeros((H, W), bool)
    live[c["mask_rows"]:] = keep[c["mask_rows"]:] != 0
    mk = masked.numpy()
    assert (mk[..., ~live].view(np.int32) == 0).all()
    want = lc.act_f32_torch(o_t.float().cpu(), c["act"]).numpy()
    if lc.ACTS[c["act"]] in ("sigmoid", "softplus"):
        ea, _ = lc.act_err(o_exact, c["act"])
        a64, _ = lc.act64(o_exact, c["act"])
        assert (np.abs(mk - a64)[..., live] <= ea[..., live]).all()
    else:
        np.testing.assert_array_equal(mk[..., live], want[..., live])
    if plan["rowsep"]:
        # the row-sum instantiation: beta in the same gate, the same masked, and (A_r, B_r, C_r) over the kept pixels
        b2, z2, m2, st2, rs = _fwd_keep(o_t, c, xt, ytt, yrt, keep_t, rowsums=True)
        assert st2 == 0 and lc.forward_excess(b2, z2, ref) <= 1.0 and torch.equal(m2, masked)
        mr = c["mask_rows"]
        ref_rs, bound_rs = tc.rowsums_reference(o_exact, xtab, H, W, mr, c["act"], c["dtype"], keep)
        exc = lc.excess(rs[..., mr:, :].double().numpy(), ref_rs, bound_rs)
        assert exc <= 1.0, "%s: row sums outside the gate (%.3g)" % (c["name"], exc)
    # backward: the contract's reference with d_o = 0 demanded exactly at the masked pixels
    beta_b, zinv_b, g = lc.nonsymmetric_backward_inputs(c["B"], c["L"], c["order"], float(np.abs(yrow).max()), 0)
    got = _bwd_keep(o_t, c, xt, ytt, yrt, keep_t, beta_b, zinv_b, g)
    yv = (yrt if bplan["rowsep"] else ytt).cpu().numpy()
    rb, bound = lc.backward_reference(o_exact, xtab, yv, H, W, c["order"], c["mask_rows"], c["act"], beta_b, zinv_b, g,
                                      bplan["rowsep"], c["dtype"], got)
    rb[..., keep == 0] = 0.0
    bound[..., keep == 0] = 0.0
    exc = lc.excess(got, rb, bound)
    assert exc <= 1.0, "%s: d_o outside the gate (%.3g)" % (c["name"], exc)


@pytest.mark.parametrize("case", lc.COVERAGE, ids=[c[0] for c in lc.COVERAGE])
def test_all_ones_keep_gives_the_plain_bits(case):
    c = lc.case_dict(case)
    o_t, xt, ytt, yrt, _, _, yrow = _operands(c, seed=1)
    B, L, H, W, d = c["B"], c["L"], c["H"], c["W"], c["order"]
    ones = torch.ones(H, W, dtype=torch.uint8, device=DEV)
    from test_lsq_contract_gpu import bwd, fwd
    want = fwd(o_t, c["dtype"], xt, ytt, yrt, B, L, H, W, d, c["mask_rows"], c["act"], c["reg_ls"], c["solver"])
    got = _fwd_keep(o_t, c, xt, ytt, yrt, ones)
    assert torch.equal(got[2].view(torch.int32), want[2].view(torch.int32)) and got[3] == want[3]
    plan = lc.query_plan(0, c["dtype"], c["yrow"], True, B, L, H, W, d, c["mask_rows"], c["act"])[1]
    if plan["rowsep"] and plan["act_t"] == lc.ACT_RUNTIME:
        # the run-time-activation row-separable forward compiles its row sums differently with the map (measured: beta
        # up to 1e-8 relative apart); held to 1e-6 here and to the fp64 contract by test_keep_entry_points_against_fp64
        for g_, w_ in ((got[0], want[0]), (got[1].reshape(B, L, -1), want[1].reshape(B, L, -1))):
            assert np.array_equal(g_, w_) or normwise(g_, w_) <= 1e-6
    else:
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    beta_b, zinv_b, g = lc.nonsymmetric_backward_inputs(B, L, d, float(np.abs(yrow).max()), 1)
    a = bwd(o_t, c["dtype"], xt, ytt, yrt, B, L, H, W, d, c["mask_rows"], c["act"], beta_b, zinv_b, g)
    b = _bwd_keep(o_t, c, xt, ytt, yrt, ones, beta_b, zinv_b, g)
    assert np.array_equal(a.view(np.int64), b.view(np.int64))


def test_all_ones_keep_rowsums_and_op_level_bits():
    """The row-sum entry point and the autograd op: an all-ones bool map gives the unmasked bits, forward and backward."""
    from lanedetection_end2end_b200 import homography as hg
    R, B, L, mask, order = 256, 2, 4, 52, 3
    o = torch.randn(B, L, R, 2 * R, generator=torch.Generator().manual_seed(5)).cuda()
    gb = torch.randn(B, L, order + 1, generator=torch.Generator().manual_seed(6), dtype=torch.float64).cuda()
    ones = torch.ones(R, 2 * R, dtype=torch.bool, device=DEV)
    res = []
    for keep in (None, ones):
        mod = hg.LearnedHomography(R, mask).cuda()
        with torch.no_grad():
            mod.offsets.copy_(torch.tensor([0.004, -0.003, 0.006, -0.005, 0.01]))
        st = torch.zeros(1, dtype=torch.int32, device=DEV)
        oc = o.clone().requires_grad_(True)
        beta, masked = ops_lsq.lsq_warp(oc, mod(st), order, mask, "square", want_masked=True, status_out=st, keep=keep)
        (beta * gb).sum().backward()
        res.append((beta.detach(), masked, oc.grad, mod.offsets.grad))
    for a, b in zip(*res):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# the flag through the training epoch, validation, eval modes and test_model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("learn_homography", [False, True])
def test_train_epoch_equals_eager_loop(paths, learn_homography):
    """engine.train_epoch with --trapezium_mask against the eager loop on the same fused functions: parameters,
    optimizer state and losses.avg bit for bit."""
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    args = te.make_args("clas4", paths[0])
    args.trapezium_mask = True
    args.learn_homography = learn_homography
    train, _, _ = te.loaders(paths, args)
    batches = list(train)
    crits = te.criteria(args)
    ma, mb = te.make_model(args), te.make_model(args)
    assert ma.keep is not None
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True)
    if learn_homography:
        crits[0].bind(ma)
    want_loss, _, _, skipped = te.eager_train(batches, ma, oa, *crits, args, te.per_lane_loss)
    got_loss, _ = engine.train_epoch(batches, mb, ob, *crits, args, 0)
    assert not skipped and got_loss == want_loss
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    # and the mask changed the training: the same epoch without it ends elsewhere
    args.trapezium_mask = False
    mc = te.make_model(args)
    mc.load_state_dict(te.make_model(args).state_dict())
    oc = nu.define_optim("adam", mc.parameters(), 1e-3, 0, fused=True)
    crits = te.criteria(args)
    if learn_homography:
        crits[0].bind(mc)
    other, _ = engine.train_epoch(batches, mc, oc, *crits, args, 0)
    assert other != got_loss


def test_validate_equals_eager_with_mask(paths):
    import test_epoch_gpu as te
    from lanedetection_end2end_b200 import inference
    args = te.make_args("clas4", paths[0])
    args.trapezium_mask = True
    _, valid, _ = te.loaders(paths, args)
    batches = list(valid)
    model = te.make_model(args).eval()
    crits = te.criteria(args)
    want, _ = te.eager_validate(batches, model, *crits, args)
    got = inference.validate(te.Listed(batches), model, *crits, args)
    assert got == want and got[0] != 0


@pytest.mark.parametrize("mode", ["tf32x3", "bf16", "fp8"])
def test_eval_forward_applies_the_mask(mode):
    """The eval-mode (BatchNorm-folded) forward in each convolution mode: masked is act(output) * keep, and beta is the
    masked fit of the returned output."""
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    torch.manual_seed(0)
    args = _args("--order", "3", "--clas", "True", "--mask_percentage", "0.2", B=4)
    model = Net(args).cuda().eval()
    x = torch.rand(4, 3, 256, 512, device=DEV)
    old = ops_net.CONV_MODE
    try:
        ops_net.set_conv_mode(mode)
        with torch.no_grad():
            out = model(x, torch.zeros(4, 4), True)
    finally:
        ops_net.set_conv_mode(old)
    masked, output = out[4], out[5]
    keep = model.keep.bool()
    want = (output.float() ** 2) * keep
    assert torch.equal(masked, want)
    with torch.no_grad():
        beta, _ = ops_lsq.lsq(output, model.grid[:4], 3, 255.0, model.zero_rows, "square", keep=model.keep)
    got = torch.stack([b.squeeze(-1) for b in out[:4]], 1)
    assert torch.equal(got, beta)


def test_test_model_runs_with_mask(tmp_path):
    """inference.test_model with --trapezium_mask: the written predictions are the eager host path's on the masked model."""
    import io
    from test_tusimple_gpu import _eager_host_path, _ground_truth
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from oracle import inputs
    N, B = 40, 32
    args = _args("--order", "3", "--clas", "1", B=B)
    torch.manual_seed(0)
    model = Net(args).cuda().eval()
    images = torch.from_numpy(inputs.make_images(N, 256, 512, seed=31))
    batches = [images[i:i + B] for i in range(0, N, B)]
    lanes = _eager_host_path(model, args, batches)
    rows = _ground_truth(lanes, 5)
    with open(tmp_path / "test_label.json", "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    want = io.StringIO()
    inference.write_tusimple_predictions(want, rows, lanes, 0)
    args.test_dir = args.save_path = str(tmp_path)
    inference.test_model(batches, model, None, None, None, None, args)
    assert (tmp_path / "test_set_predictions.json").read_text() == want.getvalue()
