"""The fp64 restatements of tests/heads_contract.py checked without a GPU: against torch float64's F.linear and autograd,
F.avg_pool2d, F.cross_entropy and the reference's torch.max formulation of the lane maps; the fp32 emulations of the
kernels pass their gates with headroom, and every seeded mutation fails its gate on the shapes the GPU tests use; the
ctypes prototypes of the seven heads entry points match the header, and the host-side checks refuse what they guard
before any launch."""
import ctypes
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

import heads_contract as hc

F64 = torch.float64
TOL = 1e-12
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADROOM = 0.5                      # a correct fp32 emulation stays below this fraction of its gate
# except the cross-entropy gradient of widely spread logits: there the rounding of d_c = v_c - m, u |d_c| relative in
# exp(d_c), is the one first-order term of the gate a correct kernel attains in full (|d_c| just above a power of two),
# so such an entry sits near |d_c| / (|d_c| + 2C + 29) of its gate -- 0.69 at d_c = -67.6, C = 4
HEADROOM_CE_BWD = 0.75


def _g(seed):
    return torch.Generator().manual_seed(seed)


# =====================================================================================================================
# restatements against torch
# =====================================================================================================================
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("bias", [False, True])
def test_linear_restatement_matches_torch_linear_and_autograd(relu, bias):
    g = _g(3 + 2 * relu + bias)
    B, K, O = 7, 300, 9
    x = torch.randn(B, K, generator=g, dtype=F64).requires_grad_()
    W = torch.randn(O, K, generator=g, dtype=F64).requires_grad_()
    b = torch.randn(O, generator=g, dtype=F64).requires_grad_() if bias else None
    y = F.linear(x, W, b)
    y = y.relu() if relu else y
    dy = torch.randn(B, O, generator=g, dtype=F64)
    grads = torch.autograd.grad(y, [x, W] + ([b] if bias else []), dy)
    ref, S = hc.linear_fwd(x.detach(), W.detach(), None if b is None else b.detach(), relu)
    assert (ref - y.detach()).abs().max() < TOL
    assert (S >= ref.abs() - TOL).all()
    relu_out = y.detach() if relu else None
    dx, _ = hc.linear_bwd_data(dy, relu_out, W.detach())
    dW, _, db, _ = hc.linear_bwd_weight(dy, relu_out, x.detach())
    assert (dx - grads[0]).abs().max() < TOL and (dW - grads[1]).abs().max() < TOL
    if bias:
        assert (db - grads[2]).abs().max() < TOL


def test_relu_gate_is_exact_at_signed_zeros_subnormals_and_nan():
    tiny = torch.tensor(1e-45, dtype=torch.float32)
    assert float(tiny) > 0                                  # the smallest positive subnormal survives as itself
    relu_out = torch.tensor([[0.0, -0.0, float(tiny), 1.0, -1.0, float("nan")]], dtype=torch.float32)
    dy = torch.full((1, 6), 3.0)
    got = hc.relu_gate(dy, relu_out)
    assert got.tolist() == [[0.0, 0.0, 3.0, 3.0, 0.0, 0.0]]
    assert not torch.signbit(got).any(), "a gated entry is +0.0"
    assert hc.relu_gate(dy, relu_out, ge=True).tolist() == [[3.0, 3.0, 3.0, 3.0, 0.0, 0.0]]


@pytest.mark.parametrize("C,H,W", [(1, 1, 1), (3, 2, 63), (100, 3, 65), (64, 32, 64)])
def test_rowmean_restatement_matches_avg_pool_and_nchw_flatten(C, H, W):
    g = _g(C + H + W)
    x = torch.randn(2, C, H, W, generator=g, dtype=F64).requires_grad_()
    y = F.avg_pool2d(x, (1, W)).reshape(2, -1)
    ref, S = hc.rowmean_fwd(x.detach().permute(0, 2, 3, 1))
    assert ref.shape == (2, C * H) and (ref - y.detach()).abs().max() < TOL
    assert (S >= ref.abs() - TOL).all()
    dout = torch.randn(2, C * H, generator=g, dtype=F64)
    dx, = torch.autograd.grad(y, x, dout)
    got = hc.rowmean_bwd(dout.float(), 2, H, W, C)                          # fp32: dout * fl32(1/W)
    assert got.dtype == torch.float32 and got.shape == (2, H, W, C)
    assert (got.double() - dx.permute(0, 2, 3, 1)).abs().max() <= 2 * hc.U * dx.abs().max()
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(W), dtype=torch.float32)
    assert torch.equal(got[1, H - 1, W - 1], dout.float()[1].view(C, H)[:, H - 1] * inv)


@pytest.mark.parametrize("C", [1, 2, 5, 8])
@pytest.mark.parametrize("tmode", ["in_range", "mixed", "none"])
@pytest.mark.parametrize("wmode", ["none", "positive", "zero_class"])
def test_ce_restatement_matches_torch_cross_entropy(C, tmode, wmode):
    g = _g(10 * C + len(tmode) + len(wmode))
    shape = (2, 5, 7)
    x = torch.randn((2, C) + shape[1:], generator=g, dtype=F64).requires_grad_()
    t = hc.ce_targets(shape, C, tmode, g)
    w = hc.ce_weight(C, wmode, g)
    tt = torch.where((t >= 0) & (t < C), t, torch.full_like(t, -100))       # torch takes only ignore_index as a miss
    ref = F.cross_entropy(x, tt, weight=None if w is None else w.double(), ignore_index=-100)
    gout = -3.5
    dx, = torch.autograd.grad(ref, x, torch.tensor(gout, dtype=F64))
    loss, bound, den = hc.ce2d_fwd(x.detach(), t, w)
    got, gb = hc.ce2d_bwd(x.detach(), t, w, gout)
    if tmode == "none" or (wmode == "zero_class" and C == 1):
        assert den == 0 and math.isnan(loss) and math.isnan(float(ref.detach()))
    else:
        assert abs(loss - float(ref.detach())) < TOL and bound > 0
    if tmode == "none":
        assert torch.equal(dx, torch.zeros_like(dx)) and torch.equal(got, torch.zeros_like(got))
        assert not torch.signbit(got).any()
    elif den > 0:
        assert (got - dx).abs().max() < TOL
        assert (gb > 0).all()


def test_ce_counted_pixels_with_zero_weight_sum_are_nan_in_torch_too():
    """Where every counted pixel has class weight 0 the sum is 0 and torch's gradient is NaN on them: that case is not
    the uncounted one, and the kernel's NaN there agrees with torch."""
    x = torch.randn(1, 3, 2, 2, dtype=F64).requires_grad_()
    t = torch.ones(1, 2, 2, dtype=torch.long)
    w = torch.tensor([1.0, 0.0, 1.0], dtype=F64)
    dx, = torch.autograd.grad(F.cross_entropy(x, t, weight=w), x)
    assert torch.isnan(dx).all()


def _reference_lane_maps(out, nl, mask_rows, gt_line):
    """BP/Networks/LSQ_layer.py's non-end-to-end branch: torch.max(., 1)[1], label * (label == k), index_fill of the top
    rows, then masked[gt_mask] = masked[0, 0] repeated."""
    _, act = torch.max(out, 1)
    act = act.float()
    masked = torch.stack([act * (act == k + 1).float() for k in range(nl)], 1)
    masked = masked.index_fill(2, torch.arange(mask_rows), 0) if mask_rows else masked
    if gt_line is not None and gt_line.sum() != 0:
        gt_mask = gt_line[:, :, None, None].bool().expand_as(masked)
        masked[gt_mask] = masked[0, 0].unsqueeze(0).repeat(int(gt_line.sum().item()), 1, 1).view(-1)
    return masked


@pytest.mark.parametrize("C,nl", [(3, 2), (5, 4), (5, 2), (8, 7)])
@pytest.mark.parametrize("mask_rows", [0, 3, 9])
def test_lane_maps_restatement_matches_reference_formulation(C, nl, mask_rows):
    g = _g(C * 10 + nl + mask_rows)
    B, H, W = 3, 9, 11
    out = torch.randint(-1, 2, (B, C, H, W), generator=g).float()            # ties everywhere: the first maximum wins
    for gl in (None, torch.zeros(B, nl), torch.tensor([[0.0] * nl, [1.0] + [0.0] * (nl - 1), [1.0] * nl]), torch.ones(B, nl)):
        got = hc.lane_maps(out, nl, mask_rows, gl)
        assert torch.equal(got, _reference_lane_maps(out, nl, min(mask_rows, H), gl)), gl
    first = torch.zeros(B, H, W, dtype=torch.long)
    best = out[:, 0].clone()
    for c in range(1, C):
        first = torch.where(out[:, c] > best, torch.full_like(first, c), first)
        best = torch.maximum(best, out[:, c])
    assert torch.equal(torch.max(out, 1)[1], first)


# =====================================================================================================================
# the fp32 emulations pass with headroom; the mutations fail
# =====================================================================================================================
def _small(case):
    B, K, O = case[:3]
    return B * K * O <= 3_000_000


LIN_CPU = [c for c in hc.linear_cases() if _small(c)]


def test_linear_cases_cover_every_batch_tile_with_a_k_tail():
    cases = hc.linear_cases()
    assert {c[0] for c in cases} == set(hc.LIN_B) and {c[1] for c in cases} == set(hc.LIN_K)
    tails = {bt for B, K, *_ in cases if K % hc.LIN_KC for _, bt in hc.lin_passes(B)}
    assert tails == {8, 16, 32, 64}
    assert {len(hc.lin_passes(c[0])) for c in cases} == {1, 2, 3}
    assert {hc.lin_passes(c[0])[-1][1] for c in cases if c[0] > 64} == {8, 32}
    for flag in (3, 4, 5):
        assert {c[flag] for c in cases} == {False, True}
    assert all(hc.lin_bwd_accepts(B, O) for B, _, O, *_ in cases)
    assert len(LIN_CPU) >= 20 and {c[0] for c in LIN_CPU} == set(hc.LIN_B)


def _linear_operands(case, seed):
    B, K, O, relu, bias, _, cls = case
    g = _g(seed)
    x = hc.operand((B, K), cls, g)
    W = torch.randn(O, K, generator=g) / math.sqrt(K)
    b = torch.randn(O, generator=g) if bias else None
    dy = torch.randn(B, O, generator=g)
    return x, W, b, dy


def _relu_out(y):
    r = y.clone().view(-1)
    specials = torch.tensor([0.0, -0.0, 1e-45])
    r[:min(3, r.numel())] = specials[:min(3, r.numel())]
    return r.view_as(y)


@pytest.mark.parametrize("case", LIN_CPU, ids=["B%d_K%d_O%d" % c[:3] for c in LIN_CPU])
def test_linear_emulation_passes_and_mutations_fail(case):
    B, K, O, relu, bias, _, cls = case
    x, W, b, dy = _linear_operands(case, B * 7 + K + O)
    y = hc.emulate_linear_fwd(x, W, b, relu)
    ref, S = hc.linear_fwd(x, W, b, relu)
    bound = hc.gate(hc.linear_fwd_k(K), S)
    assert hc.excess(y, ref, bound) <= HEADROOM
    if hc.lin_chunks(K) > 1:
        assert hc.excess(hc.emulate_linear_fwd(x, W, b, relu, mutate="drop_last_chunk"), ref, bound) > 1.0
    relu_out = _relu_out(y) if relu else None
    dref, dS = hc.linear_bwd_data(dy, relu_out, W)
    dbound = hc.gate(O, dS)
    assert hc.excess(hc.emulate_linear_bwd_data(dy, relu_out, W), dref, dbound) <= HEADROOM
    if relu:
        assert hc.excess(hc.emulate_linear_bwd_data(dy, relu_out, W, mutate="relu_ge"), dref, dbound) > 1.0
    wref, wS, bref, bS = hc.linear_bwd_weight(dy, relu_out, x)
    dW, db = hc.emulate_linear_bwd_weight(dy, relu_out, x)
    wb, bb = hc.gate(B, wS), hc.gate(B, bS)
    assert hc.excess(dW, wref, wb) <= HEADROOM and hc.excess(db, bref, bb) <= HEADROOM
    b_last = hc.lin_passes(B)[-1][0]
    leak = bool((hc.relu_gate(dy, relu_out)[b_last] != 0).any())          # the row a padded row would repeat is not all zero
    for m, applies in (("pad_leak", sum(bt for _, bt in hc.lin_passes(B)) > B and leak),
                       ("no_accumulate", B > 64)):
        if applies:
            mW, mb = hc.emulate_linear_bwd_weight(dy, relu_out, x, mutate=m)
            assert hc.excess(mW, wref, wb) > 1.0 and hc.excess(mb, bref, bb) > 1.0, m


def test_linear_mutations_cover_the_gpu_shapes():
    """Each linear mutation has GPU cases it applies to: a K tail past one chunk, a padded last tile, several passes."""
    cases = hc.linear_cases()
    assert sum(1 for c in cases if hc.lin_chunks(c[1]) > 1) >= 10
    assert sum(1 for c in cases if sum(bt for _, bt in hc.lin_passes(c[0])) > c[0]) >= 10
    assert sum(1 for c in cases if c[0] > 64) >= 6
    assert sum(1 for c in cases if c[3]) >= 10


@pytest.mark.parametrize("C", hc.ROWMEAN_C)
@pytest.mark.parametrize("W", hc.ROWMEAN_W)
def test_rowmean_emulation_passes_and_mutations_fail(C, W):
    g = _g(C * 1000 + W)
    for H in hc.ROWMEAN_H:
        x = hc.operand((2, H, W, C), ("randn", "heavy", "relu")[(C + W + H) % 3], g) + 0.25
        ref, S = hc.rowmean_fwd(x)
        bound = hc.gate(hc.rowmean_k(W, C), S)
        assert hc.excess(hc.emulate_rowmean_fwd(x), ref, bound) <= HEADROOM
        if W >= 2:
            assert hc.excess(hc.emulate_rowmean_fwd(x, mutate="div_w_minus_1"), ref, bound) > 1.0
        if hc.rowmean_lpc(C) > 1 and W >= hc.rowmean_lpc(C):
            assert hc.excess(hc.emulate_rowmean_fwd(x, mutate="drop_last_lane"), ref, bound) > 1.0


CE_CPU_SHAPE = (2, 13, 21)          # the GPU cases' odd size at a CPU-friendly scale: 546 pixels, not a multiple of 256


@pytest.mark.parametrize("case", hc.ce_cases(), ids=["C%d_%s_%s_g%s_%s" % c for c in hc.ce_cases()])
def test_ce_emulation_passes_and_mutations_fail(case):
    C, wmode, tmode, gout, logits = case
    g = _g(C * 100 + len(wmode) + len(tmode) + len(logits))
    shape = CE_CPU_SHAPE
    x = hc.ce_logits((shape[0], C) + shape[1:], logits, g)
    t = hc.ce_targets(shape, C, tmode, g)
    w = hc.ce_weight(C, wmode, g)
    loss, bound, den = hc.ce2d_fwd(x, t, w)
    eloss, eden = hc.emulate_ce2d_fwd(x, t, w)
    dref, dbound = hc.ce2d_bwd(x, t, w, gout)
    dx = hc.emulate_ce2d_bwd(x, t, w, gout)
    if den == 0:
        assert math.isnan(loss) and math.isnan(eloss) and eden == 0
        counted = ((t >= 0) & (t < C))[:, None].expand_as(dx)
        assert torch.equal(dx[~counted], torch.zeros_like(dx[~counted])) and not torch.signbit(dx[~counted]).any()
        assert torch.isnan(dx[counted]).all() and torch.isnan(dref[counted]).all()
        return
    assert abs(eloss - loss) <= HEADROOM * bound, (eloss, loss, bound)
    assert hc.excess(dx, dref, dbound) <= (HEADROOM_CE_BWD if logits in ("spread80", "randn30") else HEADROOM)
    muts = ce_mutations(C, wmode, tmode, gout, logits)
    for m in muts:
        ml, _ = hc.emulate_ce2d_fwd(x, t, w, mutate=m)
        mdx = hc.emulate_ce2d_bwd(x, t, w, gout, mutate=m)
        fwd_caught = not (abs(ml - loss) <= bound)
        bwd_caught = hc.excess(mdx, dref, dbound) > 1.0
        assert fwd_caught or bwd_caught, m
        if m == "count_uncounted":
            assert fwd_caught, m
    if shape[0] > 1 and gout != 0.0 and C > 1 and logits != "big1e4":      # else every image's softmax is the same
        assert hc.excess(hc.emulate_ce2d_bwd(x, t, w, gout, mutate="next_image"), dref, dbound) > 1.0


def ce_mutations(C, wmode, tmode, gout, logits):
    """The cross-entropy mutations a case can see: uncounted pixels in the weight sum need uncounted pixels; the argmax
    weight needs unequal weights; the missing max subtraction needs a logit past expf's range."""
    out = []
    if tmode == "mixed":
        out.append("count_uncounted")
    if wmode != "none" and C > 1:
        out.append("argmax_weight")
    if logits in ("randn30", "big1e4"):
        out.append("no_max")
    return out


def test_every_ce_mutation_has_cases():
    seen = set()
    for case in hc.ce_cases():
        seen.update(ce_mutations(*case))
    assert seen == {"count_uncounted", "argmax_weight", "no_max"}
    assert {c[2] for c in hc.ce_cases()} == set(hc.CE_TARGETS) and {c[0] for c in hc.ce_cases()} == set(range(1, 9))
    assert {c[1] for c in hc.ce_cases()} == set(hc.CE_WEIGHTS) and {c[4] for c in hc.ce_cases()} == set(hc.CE_LOGITS)
    assert set(map(str, (c[3] for c in hc.ce_cases()))) == set(map(str, hc.CE_GOUT))


def test_ce_logit_classes_reach_their_edges():
    g = _g(1)
    x = hc.ce_logits((2, 5, 8, 8), "spread80", g)
    assert float(x.max() - x.min()) > 150 and float(torch.exp((x - x.max(1, keepdim=True).values).float()).min()) == 0.0
    x = hc.ce_logits((2, 5, 8, 8), "big1e4", g)
    assert float(x.max()) == 1e4 and not torch.isfinite(torch.exp(x.float())).all()
    x = hc.ce_logits((2, 5, 8, 8), "ties", g)
    assert (x == x.max(1, keepdim=True).values).sum(1).max() > 1


# =====================================================================================================================
# the C ABI of the seven entry points
# =====================================================================================================================
ENTRY_POINTS = ["lf_linear_fwd", "lf_linear_bwd_data", "lf_linear_bwd_weight", "lf_rowmean_fwd", "lf_rowmean_bwd",
                "lf_ce2d_fwd", "lf_ce2d_bwd", "lf_linear_chunks", "lf_ce2d_blocks", "lf_seg_lane_maps", "lf_seg_lane_maps_line"]
_CTYPE = {"int": ctypes.c_int, "lf_stream_t": ctypes.c_void_p}


def test_prototypes_match_the_header():
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    for name in ENTRY_POINTS:
        m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
        assert m, name
        want = []
        for p in m.group(1).split(","):
            p = " ".join(p.split())
            want.append(ctypes.c_void_p if "*" in p else _CTYPE[p.rsplit(" ", 1)[0]])
        res, args = _capi.PROTOTYPES[name]
        assert res is ctypes.c_int and list(args) == want, name


P_ = ctypes.c_void_p(4096)            # a non-NULL pointer that is never dereferenced (every call below is refused first)


def test_refusals_before_any_launch():
    from lanedetection_end2end_b200 import _capi
    h = _capi.lib()
    assert h.lf_linear_chunks(0) == 0 and h.lf_linear_chunks(1) == 1 and h.lf_linear_chunks(257) == 2
    for args in ((None, P_, None, 2, 8, 4, 0, P_, P_), (P_, None, None, 2, 8, 4, 0, P_, P_), (P_, P_, None, 2, 8, 4, 0, None, P_),
                 (P_, P_, None, 2, 8, 4, 0, P_, None), (P_, P_, None, 0, 8, 4, 0, P_, P_), (P_, P_, None, 2, 0, 4, 0, P_, P_),
                 (P_, P_, None, 2, 8, 0, 0, P_, P_)):
        assert h.lf_linear_fwd(*args, None) == -1, args
    for B, O in ((33, 385), (64, 385), (65, 385), (130, 385), (17, 769), (9, 1537), (1, 3073)):
        assert not hc.lin_bwd_accepts(B, O)
        assert h.lf_linear_bwd_data(P_, None, P_, B, 8, O, P_, None) == -1, (B, O)
        assert h.lf_linear_bwd_weight(P_, None, P_, B, 8, O, P_, P_, None) == -1, (B, O)
    assert hc.lin_bwd_accepts(64, 384) and hc.lin_bwd_accepts(32, 385) and hc.lin_bwd_accepts(8, 3072)
    for args in ((None, None, P_, 2, 8, 4), (P_, None, None, 2, 8, 4), (P_, None, P_, 0, 8, 4), (P_, None, P_, 2, 0, 4),
                 (P_, None, P_, 2, 8, 0)):
        assert h.lf_linear_bwd_data(*args, P_, None) == -1, args
    assert h.lf_linear_bwd_data(P_, None, P_, 2, 8, 4, None, None) == -1
    assert h.lf_linear_bwd_weight(P_, None, P_, 2, 8, 4, None, None, None) == -1
    assert h.lf_linear_bwd_weight(None, None, P_, 2, 8, 4, P_, None, None) == -1
    assert h.lf_linear_bwd_weight(P_, None, None, 2, 8, 4, P_, None, None) == -1
    for B, H, W, C in ((0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0), (1, 1, 1, 257)):
        assert h.lf_rowmean_fwd(P_, B, H, W, C, P_, None) == -1, (B, H, W, C)
    assert h.lf_rowmean_fwd(None, 1, 1, 1, 1, P_, None) == -1 and h.lf_rowmean_fwd(P_, 1, 1, 1, 1, None, None) == -1
    for B, H, W, C in ((0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, 0)):
        assert h.lf_rowmean_bwd(P_, B, H, W, C, P_, None) == -1, (B, H, W, C)
    assert h.lf_rowmean_bwd(None, 1, 1, 1, 1, P_, None) == -1 and h.lf_rowmean_bwd(P_, 1, 1, 1, 1, None, None) == -1
    for C in (0, 9, 12):
        assert h.lf_ce2d_fwd(P_, P_, None, 1, C, 4, 4, P_, P_, P_, None) == -1, C
        assert h.lf_ce2d_bwd(P_, P_, None, 1, C, 4, 4, P_, None, P_, None) == -1, C
    for B, H, W in ((0, 4, 4), (1, 0, 4), (1, 4, 0)):
        assert h.lf_ce2d_fwd(P_, P_, None, B, 3, H, W, P_, P_, P_, None) == -1
        assert h.lf_ce2d_bwd(P_, P_, None, B, 3, H, W, P_, None, P_, None) == -1
    for i in (0, 1, 7, 8, 9):
        a = [P_, P_, None, 1, 3, 4, 4, P_, P_, P_]
        a[i] = None
        assert h.lf_ce2d_fwd(*a, None) == -1, i
    for i in (0, 1, 7, 9):
        a = [P_, P_, None, 1, 3, 4, 4, P_, None, P_]
        a[i] = None
        assert h.lf_ce2d_bwd(*a, None) == -1, i
    for C, nl, mr in ((1, 1, 0), (3, 3, 0), (3, 0, 0), (3, 2, -1)):
        assert h.lf_seg_lane_maps(P_, 1, C, 4, 4, nl, mr, P_, None) == -1, (C, nl, mr)
        assert h.lf_seg_lane_maps_line(P_, 1, C, 4, 4, nl, mr, None, P_, None) == -1, (C, nl, mr)
