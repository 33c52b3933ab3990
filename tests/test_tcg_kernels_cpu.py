"""Checks of the gate and quantisers in tests/tcg_contract.py, without a GPU.

A kernel-faithful fp32 emulation of lf_wgrad_tcg's summation order (every 32-pixel stage summed from zero, added into
the CTA's running sum with one fp32 add, partials reduced in fixed order) must pass the per-entry gate at every
precision; seeded bugs -- a dropped or duplicated patch, a block with the wrong tap, swapped channel blocks, RNE
instead of RNA, a missing partial -- must each fail it.  The quantisers must match ops_net.split_tf32 and torch's bf16
cast bit for bit."""
import pytest
import torch

import tcg_contract as tc
from lanedetection_end2end_b200 import ops_net

N, HS, WS, KA, NN, NCTAS = 2, 8, 32, 96, 32, 3
BLOCKS = [(0, 0, 1, 2), (0, -1, 0, 0), (0, 1, 3, 1)]        # (view, dy, dx, cblk)


def _operands(kind, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(N, HS, WS, KA, generator=g)
    B = torch.randn(N, HS, WS, NN, generator=g)
    if kind == "ties":
        A = tc.with_low_bits(A.abs() + 2.0 ** -20, 0x1000, 13)
        B = tc.with_low_bits(B.abs() + 2.0 ** -20, 0x1000, 13)
    return A, B


def _columns(A, B, blocks):
    """raw fp64 A columns [pix, nb*32] and B rows [pix, NN] in patch order"""
    bx, by = tc.wgt_pick_patch(HS, WS)
    n, y, x = tc.patch_pixels(N, HS, WS, bx, by)
    fa, fb = A.reshape(-1).double(), B.reshape(-1).double()
    cols = [tc.gather(fa, 0, HS, WS, HS * WS * KA, WS * KA, KA, n, y + dy, x + dx, 32 * cb, 32) for _m, dy, dx, cb in blocks]
    return torch.cat(cols, 1), tc.gather(fb, 0, HS, WS, HS * WS * NN, WS * NN, NN, n, y, x, 0, NN)


def _split(t, prec, rounding):
    """fp32 operand -> (large-term operand, correction operands or None), as the kernel feeds the tensor core"""
    if prec == tc.TC_X3:
        hi, lo = tc.split_tf32(t)
        return hi, lo
    return (rounding or (tc.tf32_rna if prec == tc.TC_TF32 else tc.bf16_rne))(t), None


def _emulate(A, B, prec, blocks=BLOCKS, rounding=None, drop=None, dup=None, skip_partial=None):
    """fp32 emulation of lf_wgrad_tcg + lf_wgrad_reduce in the kernel's order -> (partials [NCTAS][nb*32][NN], reduced).
    drop / dup: a patch index left out / taken twice; skip_partial: a partial the reduction leaves out."""
    Ga, Gb = _columns(A, B, blocks)
    ah, al = _split(Ga.float(), prec, rounding)
    bh, bl = _split(Gb.float(), prec, rounding)
    total = Ga.shape[0] // 32
    ranges, _ = tc.cta_patch_ranges(total, NCTAS)
    parts = []
    for p0, p1 in ranges:
        acc = torch.zeros(Ga.shape[1], NN, dtype=torch.float32)
        acs = torch.zeros_like(acc)
        for p in list(range(p0, p1)) + ([dup] if dup is not None and p0 <= dup < p1 else []):
            if p == drop:
                continue
            r = slice(32 * p, 32 * p + 32)
            acc = acc + (ah[r].double().t() @ bh[r].double()).float()          # the stage, summed from zero
            if al is not None:
                acs = acs + (ah[r].double().t() @ bl[r].double() + al[r].double().t() @ bh[r].double()).float()
        parts.append(acs + acc if al is not None else acc)
    red = torch.zeros_like(parts[0])
    for i, pt in enumerate(parts):
        if i != skip_partial:
            red = red + pt
    return torch.stack(parts), red


def _reference(A, B, prec, blocks=BLOCKS):
    Ga, Gb = _columns(A, B, blocks)
    qa, qb = tc.quantise(Ga.float(), prec), tc.quantise(Gb.float(), prec)
    total = Ga.shape[0] // 32
    ranges, per = tc.cta_patch_ranges(total, NCTAS)
    parts = [tc.exact_and_abs(qa[32 * p0:32 * p1], qb[32 * p0:32 * p1]) for p0, p1 in ranges]
    return tc.exact_and_abs(qa, qb), parts, per


def _excess(got, prec, A, B):
    """(max over the partials, reduced) of |err| / gate"""
    parts, red = got
    (ref, S), pref, per = _reference(A, B, prec)
    xp = max(tc.gate_excess(parts[i], r, s, per + 1, prec) for i, (r, s) in enumerate(pref))
    return xp, tc.gate_excess(red, ref, S, per + 1 + NCTAS, prec)


@pytest.mark.parametrize("prec", [0, 1, 2])
@pytest.mark.parametrize("kind", ["randn", "ties"])
def test_kernel_order_emulation_passes_the_gate(prec, kind):
    A, B = _operands(kind, 1 + prec)
    xp, xr = _excess(_emulate(A, B, prec), prec, A, B)
    assert xp <= 1.0 and xr <= 1.0, (xp, xr)


@pytest.mark.parametrize("prec", [0, 1, 2])
@pytest.mark.parametrize("bug", ["dropped_patch", "duplicated_patch", "wrong_tap", "swapped_cblk", "missing_partial"])
def test_seeded_bugs_fail_the_gate(prec, bug):
    A, B = _operands("randn", 10 + prec)
    total = N * HS * WS // 32
    ranges, _ = tc.cta_patch_ranges(total, NCTAS)
    kw = {}
    if bug == "dropped_patch":
        kw["drop"] = ranges[-1][1] - 1
    elif bug == "duplicated_patch":
        kw["dup"] = ranges[1][0]
    elif bug == "wrong_tap":
        kw["blocks"] = [BLOCKS[0], (0, -1, 1, 0), BLOCKS[2]]
    elif bug == "swapped_cblk":
        kw["blocks"] = [BLOCKS[0][:3] + (BLOCKS[1][3],), BLOCKS[1][:3] + (BLOCKS[0][3],), BLOCKS[2]]
    else:
        kw["skip_partial"] = NCTAS - 1
    xp, xr = _excess(_emulate(A, B, prec, **kw), prec, A, B)
    assert xr > 1.0, (bug, xr)
    if bug != "missing_partial":
        assert xp > 1.0, (bug, xp)


@pytest.mark.parametrize("prec,rounding", [(0, tc.tf32_rne), (2, tc.bf16_rna)])
def test_other_tie_rounding_fails_the_gate(prec, rounding):
    A, B = _operands("ties", 20 + prec)
    if prec == 2:
        A = tc.with_low_bits(A, 0x8000, 16)
        B = tc.with_low_bits(B, 0x8000, 16)
    assert _excess(_emulate(A, B, prec), prec, A, B)[1] <= 1.0
    xp, xr = _excess(_emulate(A, B, prec, rounding=rounding), prec, A, B)
    assert xp > 1.0 and xr > 1.0, (xp, xr)


def _values():
    g = torch.Generator().manual_seed(3)
    v = torch.randn(4096, generator=g) * torch.exp(3 * torch.randn(4096, generator=g))
    ties13 = tc.with_low_bits(v[:512], 0x1000, 13)
    ties16 = tc.with_low_bits(v[512:1024], 0x8000, 16)
    edges = torch.tensor([0.0, -0.0, 1.0, -1.0, 3.4e38, -3.4e38, 1e-38, 1e-40, -1e-45, float("inf"), float("-inf")])
    return torch.cat([v, ties13, ties16, edges])


def test_quantisers_match_split_tf32_and_torch_bf16_bit_for_bit():
    v = _values()
    hi, lo = tc.split_tf32(v)
    ref = ops_net.split_tf32(v)
    assert torch.equal(hi.view(torch.int32), ref[0].view(torch.int32))
    assert torch.equal(lo.view(torch.int32), ref[1].view(torch.int32))
    assert torch.equal(tc.tf32_rna(v).view(torch.int32), ref[0].view(torch.int32))
    assert torch.equal(tc.bf16_rne(v).view(torch.int32), v.to(torch.bfloat16).float().view(torch.int32))
    # the tie values: RNA rounds away, RNE to even, truncation drops the half step
    t = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11)])
    assert tc.tf32_rna(t).tolist() == [1.0 + 2.0 ** -10, 1.0 + 2 * 2.0 ** -10, -(1.0 + 2.0 ** -10)]
    assert tc.tf32_rne(t).tolist() == [1.0, 1.0 + 2 * 2.0 ** -10, -1.0]
    assert tc.tf32_trunc(t).tolist() == [1.0, 1.0 + 2.0 ** -10, -1.0]
    b = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8])
    assert tc.bf16_rna(b).tolist() == [1.0 + 2.0 ** -7, 1.0 + 2 * 2.0 ** -7]
    assert tc.bf16_rne(b).tolist() == [1.0, 1.0 + 2 * 2.0 ** -7]


def test_patch_geometry_covers_every_pixel_once():
    for Hs, Ws, bxy in [(32, 64, (32, 1)), (32, 48, (16, 2)), (32, 24, (8, 4)), (32, 20, (4, 8)), (32, 6, (2, 16)),
                        (32, 5, (1, 32))]:
        assert tc.wgt_pick_patch(Hs, Ws) == bxy
        n, y, x = tc.patch_pixels(2, Hs, Ws, *bxy)
        lin = (n * Hs + y) * Ws + x
        assert torch.equal(lin.sort().values, torch.arange(2 * Hs * Ws))
    assert tc.wgt_pick_patch(3, 5) is None
    for Hs, Ws, bx in [(1, 128, 128), (2, 64, 64), (4, 32, 32), (8, 16, 16), (16, 8, 8), (32, 4, 4), (64, 2, 2), (128, 3, 1)]:
        assert tc.tg_pick_patch(Hs, Ws) == (bx, 128 // bx)
    ranges, per = tc.cta_patch_ranges(10, 7)
    assert per == 2 and ranges[-2:] == [(10, 10), (10, 10)] and sum(b - a for a, b in ranges) == 10
