"""GPU tests of the inference-only fp8 convolution mode (ops_net.set_conv_mode("fp8")): lf_conv1d_tc_fp8 (csrc/conv_tc.cu),
lf_amax_per_image (csrc/net_misc.cu) and the fp8 eval path of ops_eval.

  * Operand level, entry by entry, one launch per shape family: the kernel against the fp64 sum of the exactly quantised
    operands (oracle/fp8_oracle.py), within the fp32-accumulation bound of the other operand-level tests plus the fp8
    tensor core's own accumulation bound (MMA_GATE); out_amax must be exactly the per-image max of the stored output.
  * Full eval path on the golden inputs: beta within 3e-2 of the fp64 eval forward and within 4x of the CPU emulation's
    error either way; the H100 figures are recorded in tests/golden/fp8_accuracy_<case>.json.
  * Batch invariance, graph replay, and switching modes back and forth.
"""
import functools
import json
import os

import numpy as np
import pytest
import torch

from oracle import inputs, fp8_oracle as fo
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

# fp32 accumulation of exact products, as the TF32-exact / bf16-exact cases of test_conv_tc_gpu.py / test_bf16_gpu.py
EXACT_GATE = 2e-6
# The H100's e4m3 wgmma sums the 32 products of one k32 step with fewer mantissa bits than fp32 (measured on these cases:
# up to 7.3e-5, about 2^-13.7, of an output's sum of |products|): each output is also allowed 2^-11 of its sum of
# |products| (dequantised).  A fragment,
# descriptor or quantisation bug moves a result by whole products.
MMA_GATE = 2.0 ** -11

CASES = ([(2, 64, 64, 128, v, 1) for v in (True, False)]
         + [(2, 128, 32, 64, v, d) for d in (1, 2, 4, 8, 16) for v in (True, False)]
         + [(2, 16, 128, 256, v, 1) for v in (True, False)])


def ops():
    from lanedetection_end2end_b200 import ops_net
    return ops_net


@pytest.fixture
def fp8_mode():
    o = ops()
    prev = o.CONV_MODE
    o.set_conv_mode("fp8")
    yield o
    o.set_conv_mode(prev)


@pytest.mark.parametrize("N,C,H,W,vertical,dil", CASES)
@pytest.mark.parametrize("in_bf16", [False, True], ids=["f32_in", "bf16_in"])
@pytest.mark.parametrize("residual", [False, True], ids=["relu", "residual"])
def test_fp8_conv_against_fp64_of_quantised_operands(N, C, H, W, vertical, dil, in_bf16, residual, fp8_mode):
    from lanedetection_end2end_b200 import ops_eval
    o = fp8_mode
    g = torch.Generator().manual_seed(N * 1000 + C * 10 + dil + 7 * vertical)
    x = torch.randn(N, H, W, C, generator=g)
    x[1] *= 3.0                                     # the images have different scales
    x = x.bfloat16() if in_bf16 else x
    kh, kw = (3, 1) if vertical else (1, 3)
    w = torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5
    w[3] = 0.0                                      # an all-zero output channel: q_w = 0, s_w = 0
    b = torch.randn(C, generator=g)
    add = torch.randn(N, H, W, C, generator=g) if residual else None
    xd = x.cuda()
    sup = C == 16
    assert (o.super_ok(xd, 1) if sup else o.tc_supported(xd, vertical, dil))
    wp, s_w = ops_eval._fp8_operand(w.cuda(), vertical, sup)
    # the block-input scale: lf_amax_per_image, exactly the per-image max
    ax = ops_eval.block_input_amax(xd)
    torch.cuda.synchronize()
    assert torch.equal(ax.cpu(), fo.image_amax(x))
    am = torch.zeros(N, device="cuda")
    epi = dict(relu=2, add_src=add.cuda()) if residual else dict(relu=True)
    out_dtype = torch.bfloat16 if (in_bf16 and not residual) else torch.float32
    got = o.conv3(xd, None, vertical, dil, False, wp=wp, bias=b.cuda(), dtype=out_dtype, fp8=(ax, s_w, am), **epi)
    torch.cuda.synchronize()
    got, am = got.float().cpu(), am.cpu()
    # oracle: fp64 sum of the exactly quantised operands, the fp32 dequantisation factors, then the epilogue in fp64
    xn = x.float().permute(0, 3, 1, 2)
    qw, sw = fo.quantize_weight(w)
    assert torch.equal(s_w.cpu()[:C], sw)
    qx = fo.quantize_act(xn, ax.cpu())
    acc = fo.conv3_fp64(qx, qw, vertical, dil)
    dq = fo.scale(ax.cpu()).view(-1, 1, 1, 1) * sw.view(1, -1, 1, 1)        # fp32, as the kernel
    abssum = (fo.conv3_fp64(qx.abs(), qw.abs(), vertical, dil) * dq.double()).permute(0, 2, 3, 1)
    ref = acc * dq.double() + b.double().view(1, -1, 1, 1)
    ref = ref.clamp_min(0) if not residual else (ref + add.double().permute(0, 3, 1, 2)).clamp_min(0)
    ref = ref.permute(0, 2, 3, 1)
    scale = float(ref.abs().max())
    tol = EXACT_GATE * scale + MMA_GATE * abssum + (2.0 ** -8 * ref.abs() if out_dtype == torch.bfloat16 else 0.0)
    err = (got.double() - ref).abs()
    nz = abssum > 0
    print("max |err| %.3e, max |err| / sum|products| %.3e" % (float(err.max()), float((err[nz] / abssum[nz]).max())))
    assert bool((err <= tol).all()), (float(err.max()), float((err - tol).max()), scale)
    # out_amax: exactly the per-image max |stored value|
    assert torch.equal(am, got.abs().flatten(1).amax(1)), (am, got.abs().flatten(1).amax(1))


def _golden_model(name, P32, batch=None):
    from oracle import golden_check
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = json.loads(str(g["meta"]))
    L, order, B = meta["L"], meta["order"], meta["B"]
    model, _ = golden_check.build_net(L, order, meta["mask_pct"], batch or B)
    sd = model.state_dict()
    for k, v in P32.items():
        if "net." + k in sd:
            sd["net." + k] = v
    model.load_state_dict(sd)
    return model.cuda().eval(), meta


@pytest.mark.parametrize("name", ["net_l2_d2", "net_l4_d3"])
def test_full_eval_path_fp8_accuracy(name, fp8_mode):
    """beta of the graphed-able eval forward in fp8 mode vs the fp64 eval forward of the same model (running statistics
    from one training-mode forward of the golden input)."""
    rec, P32, beta64 = fo.emulate_golden_case(name)
    model, meta = _golden_model(name, P32)
    L, B = meta["L"], meta["B"]
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=meta["image_seed"])).cuda()
    with torch.no_grad():
        out = model(x, torch.zeros(B, 4), True)
    torch.cuda.synchronize()
    ours = torch.stack([out[l].squeeze(-1) for l in range(L)], 1).cpu().numpy()
    err = fo.normwise(ours, beta64)
    emu = rec["beta_normwise_err_fp8"]
    res = {"case": name, "beta_normwise_err_fp8": err, "beta_normwise_err_fp8_emulation": emu,
           "beta_normwise_err_bf16_emulation": rec["beta_normwise_err_bf16"], "gpu": torch.cuda.get_device_name()}
    print(res)
    outdir = os.environ.get("LANEFIT_ACCURACY_OUT")   # optional: where to write the measured record
    if outdir and os.path.isdir(outdir):
        with open(os.path.join(outdir, "fp8_accuracy_%s.json" % name), "w") as f:
            json.dump(res, f)
    assert err < 3e-2, res
    assert emu / 4 <= err <= 4 * emu, res


@functools.lru_cache(maxsize=None)
def _golden_statistics():
    return fo.emulate_golden_case("net_l2_d2")[1]


def _net_with_stats(batch):
    """net_l2_d2's model in eval mode, running statistics from one training-mode forward of its golden input."""
    return _golden_model("net_l2_d2", _golden_statistics(), batch)[0]


def test_fp8_batch_invariance(fp8_mode):
    """Image i's beta and decoder output are bit-identical at batch 1 and inside a batch of 8: every scale is per image."""
    model = _net_with_stats(8)
    x = torch.from_numpy(inputs.make_images(8, 256, 512, seed=21)).cuda()
    with torch.no_grad():
        full = model(x, torch.zeros(8, 4), True)
        for i in (0, 5):
            one = model(x[i:i + 1].contiguous(), torch.zeros(1, 4), True)
            for k in (0, 1, 5):       # beta0, beta1, decoder output
                assert torch.equal(one[k][0], full[k][i]), (i, k, float((one[k][0] - full[k][i]).abs().max()))


def test_fp8_graph_replay_and_mode_switches():
    """A GraphedInference replay in fp8 mode == the eager fp8 eval forward, bit for bit; bf16 and tf32x3 give their
    earlier bits after it."""
    from lanedetection_end2end_b200 import _capi
    from lanedetection_end2end_b200.engine import GraphedInference
    o = ops()
    model = _net_with_stats(4)
    x = torch.from_numpy(inputs.make_images(4, 256, 512, seed=22)).cuda()

    def eager(mode):
        o.set_conv_mode(mode)
        with torch.no_grad():
            out = model(x, torch.zeros(4, 4), True)
        torch.cuda.synchronize()
        return [t.clone() for t in (out[0], out[1], out[5])]

    prev = o.CONV_MODE
    try:
        before = {m: eager(m) for m in ("bf16", "tf32x3")}
        _capi.TRACE = []
        ref = eager("fp8")
        names = [t[0] for t in _capi.TRACE]
        _capi.TRACE = None
        assert names.count("lf_conv1d_tc_fp8") == 4 * 13 + 4 * 4, names      # every 3-tap conv of the 17 blocks
        assert "lf_conv1d_tc_bf16" not in names and "lf_amax_per_image" in names and "lf_conv_tcg" in names
        gi = GraphedInference(model, x)
        got = gi.infer(x)
        torch.cuda.synchronize()
        for a, b in zip(ref, (got[0], got[1], got[5])):
            assert torch.equal(a, b)
        assert not torch.equal(ref[2], before["bf16"][2])
        del gi
        for m in ("bf16", "tf32x3", "fp8"):
            again = eager(m)
            want = ref if m == "fp8" else before[m]
            for a, b in zip(want, again):
                assert torch.equal(a, b), m
    finally:
        _capi.TRACE = None
        o.set_conv_mode(prev)
        o.ACTIVE_PACKS = None
