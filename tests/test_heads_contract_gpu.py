"""The heads' kernels driven directly through their C entry points, entry by entry against the fp64 restatements of
tests/heads_contract.py: lf_linear_fwd / _bwd_data / _bwd_weight, lf_rowmean_fwd / _bwd, lf_ce2d_fwd / _bwd and
lf_seg_lane_maps / _line.

Every case launches into sentinel-filled buffers with a guard tail and holds every entry the contract writes to its
gate (or to its exact value), and every other entry to the sentinel:
  * linear: every batch tile BT = 8 / 16 / 32 / 64, one to three 64-row passes and a final pass of each BT, K tails from
    1 to 32768 columns, with and without ReLU / bias / db, normal, heavy-tailed and ReLU-output operands; the production
    layers at B = 2, 8, 32; the ReLU gate bit for bit at +0.0, -0.0 and the smallest subnormal; the backward's
    shared-memory refusal at its boundary;
  * row mean: C from 1 to 256 against W from 1 to 1000 (the forward's lane split and its IEEE division), the gradient bit
    for bit, the horizon head's shape past the gradient's grid-stride cap;
  * cross entropy: C = 1..8, weight NULL / positive / with a zero class, targets in range / mixed with misses / none
    counted, gout NULL / 1 / -3.5 / 0, five logit classes (ties, expf underflow, a class at 1e4), sizes from one pixel to
    past the grid-stride cap and the production ones; two forwards give the same bits; a pixel whose target is not a
    class gets +0.0, also when no pixel is counted;
  * lane maps: exact past the grid-stride cap, with ties, mask_rows 0 and >= H, nl < C - 1 and gt_line none / some / all.
The largest |err| / gate per kernel is printed at the end (pytest -s)."""
import math

import pytest
import torch

import heads_contract as hc

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -1.2345e30                     # sentinel: a value no kernel here produces
GUARD = 1024                          # entries of sentinel after every output
MEASURED = {}                         # kernel -> largest |err| / gate seen


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(MEASURED.items()):
        print("%-36s max |err| / gate %.3f" % (k, v))


def _hold(kern, what, got, ref, bound):
    x = hc.excess(got, ref, bound)
    MEASURED[kern] = max(MEASURED.get(kern, 0.0), x)
    assert x <= 1.0, "%s: |err| reaches %.3g x the gate" % (what, x)


def _exact(kern, what, got, ref):
    MEASURED.setdefault(kern + " (bit-exact)", 0.0)
    assert torch.equal(got, ref), what + ": not bit-exact"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _buf(n, dtype=torch.float32):
    return torch.full((n + GUARD,), SENT, dtype=dtype, device=DEV)


def _guarded(buf, n):
    return bool((buf[n:] == SENT).all())


def _p(t):
    return None if t is None else t.data_ptr()


def grid_stride_cap():
    """Items one launch of a grid-stride kernel covers before a thread takes a second: 8 CTAs per SM of 256 threads."""
    return 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256


# =====================================================================================================================
# lf_linear_*
# =====================================================================================================================
def _relu_out(y):
    """The forward's ReLU output with +0.0, -0.0 and the smallest subnormal written over its first entries."""
    r = y.clone().view(-1)
    sp = torch.tensor([0.0, -0.0, 1e-45], device=DEV)
    r[:min(3, r.numel())] = sp[:min(3, r.numel())]
    return r.view_as(y)


def _by_pass(kern, what, got, ref, bound, B):
    for b0, bt in hc.lin_passes(B):
        r = slice(b0, min(B, b0 + 64))
        _hold("%s BT=%d" % (kern, bt), "%s rows %d.. (BT %d)" % (what, b0, bt), got[r], ref[r], bound[r])


def run_linear(B, K, O, relu, bias, has_db, cls, seed):
    c = _capi()
    g = _gen(seed)
    x = hc.operand((B, K), cls, g, DEV)
    W = torch.randn(O, K, generator=g, device=DEV) / math.sqrt(K)
    b = torch.randn(O, generator=g, device=DEV) if bias else None
    dy = torch.randn(B, O, generator=g, device=DEV)
    what = "linear B %d K %d O %d relu %d bias %d %s" % (B, K, O, relu, bias, cls)
    nch = hc.lin_chunks(K)
    partial, y = _buf(nch * B * O), _buf(B * O)
    c.call("lf_linear_fwd", _p(x), _p(W), _p(b), B, K, O, int(relu), _p(partial), _p(y), c.stream_ptr())
    assert _guarded(partial, nch * B * O) and _guarded(y, B * O), what + ": wrote past its output"
    assert bool((partial[:nch * B * O] != SENT).all()), what + ": a partial was not written"
    yv = y[:B * O].view(B, O)
    ref, S = hc.linear_fwd(x, W, b, relu)
    _by_pass("lf_linear_fwd", what, yv, ref, hc.gate(hc.linear_fwd_k(K), S), B)

    relu_out = _relu_out(yv) if relu else None
    dx = _buf(B * K)
    c.call("lf_linear_bwd_data", _p(dy), _p(relu_out), _p(W), B, K, O, _p(dx), c.stream_ptr())
    assert _guarded(dx, B * K), what + ": dx past its end"
    dref, dS = hc.linear_bwd_data(dy, relu_out, W)
    _by_pass("lf_linear_bwd_data", what, dx[:B * K].view(B, K), dref, hc.gate(O, dS), B)

    dW, db = _buf(O * K), (_buf(O) if has_db else None)
    c.call("lf_linear_bwd_weight", _p(dy), _p(relu_out), _p(x), B, K, O, _p(dW), _p(db), c.stream_ptr())
    assert _guarded(dW, O * K) and (db is None or _guarded(db, O)), what + ": dW / db past its end"
    wref, wS, bref, bS = hc.linear_bwd_weight(dy, relu_out, x)
    bts = "+".join(str(bt) for _, bt in hc.lin_passes(B))
    _hold("lf_linear_bwd_weight dW BT=" + bts, what + " dW", dW[:O * K].view(O, K), wref, hc.gate(B, wS))
    if has_db:
        _hold("lf_linear_bwd_weight db BT=" + bts, what + " db", db[:O], bref, hc.gate(B, bS))


LIN_CASES = hc.linear_cases()


@pytest.mark.parametrize("case", LIN_CASES, ids=["B%d_K%d_O%d_relu%d_bias%d_db%d_%s" % c for c in LIN_CASES])
def test_linear_every_batch_tile_and_k_tail(case):
    run_linear(*case, seed=sum(case[:3]))


@pytest.mark.parametrize("B", [2, 8, 32])
@pytest.mark.parametrize("layer", hc.LIN_PRODUCTION, ids=["K%d_O%d_relu%d" % l for l in hc.LIN_PRODUCTION])
def test_linear_production_layers(layer, B):
    """The heads' layers: line head 32768->128 (+ReLU) and 128->4, bird's-eye-view 128->12, DLT branch 128->3 / 128->5,
    horizon head 2048->256 / 2048->320."""
    K, O, relu = layer
    run_linear(B, K, O, relu, True, True, "relu" if K == 32768 else "randn", seed=B + K + O)


@pytest.mark.parametrize("B", [1, 9, 17, 33, 65])
def test_linear_relu_gate_bit_for_bit(B):
    """W = [I 0] and x with one-hot rows make dx = g and dW[:, :B] = g^T exact, g = dy * (relu_out > 0): -0.0 and +0.0
    and NaN gate, the smallest subnormal and 1.0 pass, in every batch tile."""
    c = _capi()
    O, K = 6, 300
    g = _gen(B)
    dy = torch.randn(B, O, generator=g, device=DEV)
    pat = torch.tensor([0.0, -0.0, 1e-45, 1.0, -1.0, float("nan")], device=DEV)
    relu_out = torch.stack([pat.roll(b) for b in range(B)])
    W = torch.eye(O, K, device=DEV)
    x = torch.eye(B, K, device=DEV)
    gated = hc.relu_gate(dy, relu_out)
    assert int((gated == 0).sum()) == 4 * B                  # +0.0, -0.0, -1.0 and NaN gate
    dx = _buf(B * K)
    c.call("lf_linear_bwd_data", _p(dy), _p(relu_out), _p(W), B, K, O, _p(dx), c.stream_ptr())
    want = torch.zeros(B, K, device=DEV)
    want[:, :O] = gated
    _exact("lf_linear_bwd_data relu gate", "dx B %d" % B, dx[:B * K].view(B, K), want)
    assert _guarded(dx, B * K)
    dW, db = _buf(O * K), _buf(O)
    c.call("lf_linear_bwd_weight", _p(dy), _p(relu_out), _p(x), B, K, O, _p(dW), _p(db), c.stream_ptr())
    want = torch.zeros(O, K, device=DEV)
    want[:, :B] = gated.T
    _exact("lf_linear_bwd_weight relu gate", "dW B %d" % B, dW[:O * K].view(O, K), want)
    _, _, bref, bS = hc.linear_bwd_weight(dy, relu_out, x)
    _hold("lf_linear_bwd_weight db relu gate", "db B %d" % B, db[:O], bref, hc.gate(B, bS))
    assert _guarded(dW, O * K) and _guarded(db, O)


@pytest.mark.parametrize("B,O", [(64, 384), (32, 385), (33, 385), (64, 385), (65, 385), (130, 385)])
def test_linear_backward_shared_memory_boundary(B, O):
    """The backward stages dy as [O][BT] floats in at most 96 KiB: O = 384 fits BT = 64, O = 385 fits BT = 32 but not 64,
    and a refused call returns LF_ERR_INVALID_ARGUMENT with nothing written."""
    c = _capi()
    K = 300
    if hc.lin_bwd_accepts(B, O):
        run_linear(B, K, O, True, True, True, "randn", seed=B * O)
        return
    g = _gen(B + O)
    dy, x = torch.randn(B, O, generator=g, device=DEV), torch.randn(B, K, generator=g, device=DEV)
    W = torch.randn(O, K, generator=g, device=DEV)
    dx, dW, db = _buf(B * K), _buf(O * K), _buf(O)
    h = c.lib()
    assert h.lf_linear_bwd_data(_p(dy), None, _p(W), B, K, O, _p(dx), c.stream_ptr()) == -1
    assert h.lf_linear_bwd_weight(_p(dy), None, _p(x), B, K, O, _p(dW), _p(db), c.stream_ptr()) == -1
    torch.cuda.synchronize()
    assert all(bool((t == SENT).all()) for t in (dx, dW, db)), "a refused call wrote"


# =====================================================================================================================
# lf_rowmean_*
# =====================================================================================================================
def run_rowmean(B, H, W, C, seed, cls="randn"):
    c = _capi()
    g = _gen(seed)
    x = hc.operand((B, H, W, C), cls, g, DEV)
    what = "rowmean B %d H %d W %d C %d %s" % (B, H, W, C, cls)
    out = _buf(B * C * H)
    c.call("lf_rowmean_fwd", _p(x), B, H, W, C, _p(out), c.stream_ptr())
    assert _guarded(out, B * C * H), what + ": wrote past out"
    ref, S = hc.rowmean_fwd(x)
    _hold("lf_rowmean_fwd", what, out[:B * C * H].view(B, C * H), ref, hc.gate(hc.rowmean_k(W, C), S))
    dout = torch.randn(B, C * H, generator=g, device=DEV)
    n = B * H * W * C
    dx = _buf(n)
    c.call("lf_rowmean_bwd", _p(dout), B, H, W, C, _p(dx), c.stream_ptr())
    assert _guarded(dx, n), what + ": wrote past dx"
    _exact("lf_rowmean_bwd", what, dx[:n].view(B, H, W, C), hc.rowmean_bwd(dout, B, H, W, C))
    return n


@pytest.mark.parametrize("W", hc.ROWMEAN_W)
@pytest.mark.parametrize("C", hc.ROWMEAN_C)
def test_rowmean_lane_splits_and_widths(C, W):
    for H in hc.ROWMEAN_H:
        run_rowmean(2, H, W, C, seed=C * 7 + W + H, cls=("randn", "heavy", "relu")[(C + W + H) % 3])


@pytest.mark.parametrize("B", [2, 8, 32])
def test_rowmean_horizon_head_past_the_grid_stride_cap(B):
    H, W, C = hc.HORIZON
    n = run_rowmean(B, H, W, C, seed=B)
    if B >= 8:
        assert n > 3 * grid_stride_cap(), "the gradient's threads each take several items"


def test_rowmean_refuses_more_than_256_channels():
    c = _capi()
    x = torch.randn(2 * 4 * 3 * 257, device=DEV)
    out = _buf(2 * 257 * 4)
    assert c.lib().lf_rowmean_fwd(_p(x), 2, 4, 3, 257, _p(out), c.stream_ptr()) == -1
    torch.cuda.synchronize()
    assert bool((out == SENT).all())
    run_rowmean(2, 4, 3, 256, seed=256)


# =====================================================================================================================
# lf_ce2d_*
# =====================================================================================================================
def _bits(t):
    return t.view(torch.int64)


def run_ce(B, C, H, W, wmode, tmode, gout, logits, seed):
    c = _capi()
    g = _gen(seed)
    x = hc.ce_logits((B, C, H, W), logits, g, DEV).contiguous()
    t = hc.ce_targets((B, H, W), C, tmode, g, DEV).contiguous()
    w = hc.ce_weight(C, wmode, g, DEV)
    what = "ce B %d C %d %dx%d weight %s targets %s gout %s %s" % (B, C, H, W, wmode, tmode, gout, logits)
    nblk = int(c.lib().lf_ce2d_blocks(B, H, W))
    f64 = torch.float64
    runs = []
    for _ in range(2):
        partial, sums, loss = _buf(2 * nblk, f64), _buf(2, f64), _buf(1, f64)
        c.call("lf_ce2d_fwd", _p(x), _p(t), _p(w), B, C, H, W, _p(partial), _p(sums), _p(loss), c.stream_ptr())
        assert _guarded(partial, 2 * nblk) and _guarded(sums, 2) and _guarded(loss, 1), what + ": wrote past its outputs"
        runs.append((sums, loss))
    (sums, loss), (sums2, loss2) = runs
    assert torch.equal(_bits(loss[:1]), _bits(loss2[:1])) and torch.equal(_bits(sums[:2]), _bits(sums2[:2])), \
        what + ": two forwards differ"
    ref, bound, den = hc.ce2d_fwd(x, t, w)
    got = float(loss[0])
    N = B * H * W
    assert abs(float(sums[1]) - den) <= N * 2.0 ** -53 * den, what + ": weight sum"
    if den == 0:
        assert math.isnan(got), what + ": no pixel counted, loss must be NaN as torch's"
    else:
        err = abs(got - ref) / bound if got != ref else 0.0
        MEASURED["lf_ce2d_fwd"] = max(MEASURED.get("lf_ce2d_fwd", 0.0), err)
        assert err <= 1.0, "%s: loss |err| reaches %.3g x the gate" % (what, err)
        assert abs(float(sums[0]) / float(sums[1]) - got) <= 2.0 ** -52 * abs(got)

    gbuf = None if gout is None else torch.tensor([gout], dtype=f64, device=DEV)
    n = B * C * H * W
    dx = _buf(n)
    c.call("lf_ce2d_bwd", _p(x), _p(t), _p(w), B, C, H, W, _p(sums), _p(gbuf), _p(dx), c.stream_ptr())
    assert _guarded(dx, n), what + ": wrote past dx"
    dxv = dx[:n].view(B, C, H, W)
    counted = ((t >= 0) & (t < C))[:, None].expand_as(dxv)
    un = dxv[~counted]
    assert bool((un == 0).all()) and not bool(torch.signbit(un).any()), what + ": an uncounted pixel's gradient is not +0.0"
    dref, dbound = hc.ce2d_bwd(x, t, w, gout)
    if den == 0:
        assert bool(torch.isnan(dxv[counted]).all()), what + ": counted pixels of zero weight sum are NaN, as torch's"
    else:
        _hold("lf_ce2d_bwd", what, dxv, dref, dbound)
    return n


CE_CASES = hc.ce_cases()
CE_ODD = (3, 37, 41)                  # 4551 pixels: not a multiple of 256


@pytest.mark.parametrize("case", CE_CASES, ids=["C%d_%s_%s_g%s_%s" % c for c in CE_CASES])
def test_ce_classes_weights_targets_gout_and_logits(case):
    C, wmode, tmode, gout, logits = case
    B, H, W = CE_ODD
    run_ce(B, C, H, W, wmode, tmode, gout, logits, seed=C * 31 + len(wmode) + 7 * len(tmode))


def _ce_size(name):
    cap = grid_stride_cap()
    return {"1x1x1": (1, 1, 1), "under_cap": (2, 1, cap // 2 - 1), "over_cap": (2, 1, cap // 2 + 3),
            "odd": CE_ODD, "prod_c3": (8, 256, 512), "prod_c5": (8, 256, 512)}[name]


CE_SIZES = [("1x1x1", 4, "positive", "in_range", None, "randn"), ("1x1x1", 3, "none", "none", 1.0, "randn"),
            ("under_cap", 5, "positive", "mixed", -3.5, "spread80"), ("over_cap", 5, "zero_class", "mixed", 1.0, "randn30"),
            ("over_cap", 8, "none", "in_range", None, "ties"), ("over_cap", 5, "positive", "none", -3.5, "randn"),
            ("odd", 7, "positive", "mixed", 0.0, "big1e4"),
            ("prod_c3", 3, "positive", "mixed", None, "randn"), ("prod_c5", 5, "positive", "in_range", -3.5, "randn30")]


@pytest.mark.parametrize("case", CE_SIZES, ids=["%s_C%d_%s_%s_g%s_%s" % c for c in CE_SIZES])
def test_ce_sizes_past_the_grid_stride_cap_and_production(case):
    name, C, wmode, tmode, gout, logits = case
    B, H, W = _ce_size(name)
    n = run_ce(B, C, H, W, wmode, tmode, gout, logits, seed=len(name) * C)
    pixels = B * H * W
    if name == "under_cap":
        assert pixels < grid_stride_cap()
    if name in ("over_cap", "prod_c3", "prod_c5"):
        assert pixels > grid_stride_cap() and n > pixels


def test_ce_no_counted_pixel_gives_nan_loss_and_zero_gradient():
    """Every target outside [0, C): torch's cross_entropy gives a NaN loss and an all-zero gradient, and so do the
    kernels -- the gradient of an uncounted pixel is +0.0 whatever gout / sum w is."""
    cap = grid_stride_cap()
    for gout in (None, -3.5, 0.0):
        run_ce(2, 5, 1, cap // 2 + 3, "positive", "none", gout, "randn", seed=11)


def test_ce_refuses_more_than_eight_classes():
    c = _capi()
    x = torch.randn(1 * 9 * 4 * 4, device=DEV)
    t = torch.zeros(16, dtype=torch.long, device=DEV)
    f64 = torch.float64
    partial, sums, loss, dx = _buf(64, f64), _buf(2, f64), _buf(1, f64), _buf(9 * 16)
    h = c.lib()
    assert h.lf_ce2d_fwd(_p(x), _p(t), None, 1, 9, 4, 4, _p(partial), _p(sums), _p(loss), c.stream_ptr()) == -1
    assert h.lf_ce2d_bwd(_p(x), _p(t), None, 1, 9, 4, 4, _p(sums), None, _p(dx), c.stream_ptr()) == -1
    torch.cuda.synchronize()
    assert all(bool((b == SENT).all()) for b in (partial, sums, loss, dx))


# =====================================================================================================================
# lf_seg_lane_maps / _line
# =====================================================================================================================
LANE_CASES = [(5, 4, 0, "randn"), (5, 4, 300, "ties"), (5, 2, 17, "ties"), (3, 2, 64, "randn"), (8, 1, 5, "ties")]


@pytest.mark.parametrize("case", LANE_CASES, ids=["C%d_nl%d_mask%d_%s" % c for c in LANE_CASES])
def test_lane_maps_exact_past_the_grid_stride_cap(case):
    """mask_rows 0, inside the map and >= H; nl = C - 1 and nl < C - 1; ties everywhere in the 'ties' cases."""
    C, nl, mask_rows, kind = case
    c = _capi()
    B, H = 3, 64
    W = grid_stride_cap() // (B * H) + 7
    assert B * H * W > grid_stride_cap()
    g = _gen(C * 100 + nl + mask_rows)
    out = (torch.randint(-1, 2, (B, C, H, W), generator=g, device=DEV).float() if kind == "ties"
           else torch.randn(B, C, H, W, generator=g, device=DEV))
    n = B * nl * H * W
    lines = [None, torch.zeros(B, nl, device=DEV), torch.ones(B, nl, device=DEV)]
    some = torch.zeros(B, nl, device=DEV)
    some[1:, 0] = 1.0
    some[0, -1] = 2.5
    lines.append(some)
    for gl in lines:
        maps = _buf(n)
        c.call("lf_seg_lane_maps_line", _p(out), B, C, H, W, nl, mask_rows, _p(gl), _p(maps), c.stream_ptr())
        assert _guarded(maps, n)
        want = hc.lane_maps(out, nl, mask_rows, gl)
        _exact("lf_seg_lane_maps_line", "lane maps C %d nl %d mask %d gt_line %s" % (C, nl, mask_rows, gl is not None),
               maps[:n].view(B, nl, H, W), want)
    maps = _buf(n)
    c.call("lf_seg_lane_maps", _p(out), B, C, H, W, nl, mask_rows, _p(maps), c.stream_ptr())
    assert _guarded(maps, n)
    _exact("lf_seg_lane_maps", "lane maps C %d nl %d mask %d" % (C, nl, mask_rows), maps[:n].view(B, nl, H, W),
           hc.lane_maps(out, nl, mask_rows))
