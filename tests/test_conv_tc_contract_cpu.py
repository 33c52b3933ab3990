"""The fp64 contract of the 3-tap tensor-core convolution (tests/conv_tc_contract.py) checked without a GPU:
  * the restatement agrees with torch's float64 conv2d / conv_transpose2d for both tap orders, and with explicit shifted
    sums for any three taps, and its epilogue with the formulas of include/lanefit_b200.h; the FP8 restatement agrees with
    conv2d of the separately quantised operands, dequantised per image and output channel, and its e4m3 quantiser
    rounds to nearest even, keeps subnormals and saturates at 448;
  * a kernel-faithful fp32 emulation passes the gate at every precision, its per-CTA partials included;
  * each seeded bug fails the gate: a tap shifted by one pixel, a dropped chunk, a halo row read as zero, RNE instead of
    RNA, a dropped a_lo * w_hi, rounded instead of truncated weights on the ties class, a tile-to-CTA map shifted by one;
    for FP8 also image n quantised and dequantised with image n+1's scale, flushed e4m3 subnormals and round-toward-zero
    on e4m3 midpoints;
  * lf_conv1d_tc_plan reports every planner outcome the coverage table of the GPU tests claims, and that table reaches
    every outcome the planner produces over a wide range of shapes;
  * every argument check of the three entry points (and of the plan query) refuses with LF_ERR_INVALID_ARGUMENT before
    the planner runs, so no device is needed.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import conv_tc_contract as cc

SMALL = [  # N, H, W, C, vertical, dil: slab shapes with several tiles per CTA row when m_ctas is small
    (2, 16, 32, 64, True, 1), (1, 32, 16, 64, False, 2), (2, 16, 16, 128, True, 3), (1, 16, 64, 64, False, 40),
]


def _x(N, H, W, C, seed, cls="randn"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, C, generator=g)
    w = torch.randn(C, 3 * C, generator=g) / (3 * C) ** 0.5
    if cls == "ties":
        x = cc.with_low_bits(x.abs() + 2.0 ** -20, 0x1000, 13)
        w = cc.tf32_trunc(w.abs())
    elif cls == "ties_w":
        x = cc.tf32_trunc(x.abs())
        w = cc.with_low_bits(w.abs() + 2.0 ** -20, 0x1000, 13)
    elif cls == "ties_bf16":
        x = cc.with_low_bits(x.abs() + 2.0 ** -20, 0x8000, 16)
        w = cc.bf16_rne(w.abs())
    return x, w, g


def e4m3_midpoints(shape, generator, device=None):
    """Non-negative values exactly half way between two adjacent e4m3 values (subnormal and normal, below 448)."""
    codes = torch.randint(0, 0x7e, shape, generator=generator, device=device, dtype=torch.int16)   # 0x7e = 448
    lo = codes.to(torch.uint8).view(torch.float8_e4m3fn).float()
    hi = (codes + 1).to(torch.uint8).view(torch.float8_e4m3fn).float()
    return (lo + hi) / 2


def _x_fp8(N, H, W, C, seed, cls="randn"):
    """FP8 operands: activations with per-image scales 10^-3 .. 10^3, or (subnormal) one outlier per image that puts most
    quantised activations among the e4m3 subnormals, or (ties) e4m3 midpoints under x_amax = 448 (inv = 1 exactly);
    -> (x, w, x_amax, generator)"""
    x, w, g = _x(N, H, W, C, seed)
    if cls == "ties":
        x = e4m3_midpoints((N, H, W, C), g)
        return x, w.abs(), torch.full((N,), 448.0), g
    x = x * (10.0 ** torch.linspace(-3, 3, N)).view(-1, 1, 1, 1)[torch.randperm(N, generator=g)]
    if cls == "subnormal":
        big = x.abs().flatten(1).amax(1) * 2.0 ** 14
        x.view(N, -1)[:, 7] = big
    return x, w, x.abs().flatten(1).amax(1), g


def _plan(N, H, W, C, taps, prec=cc.TC_TF32):
    rc, pl = cc.query_plan(prec, 0, N, H, W, C, taps)
    assert rc == 0, rc
    return pl


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _w4(wpack, C, vertical):
    """[C][3C] weight-slot matrix -> the [Co, Ci, kh, kw] conv2d weight (slot t = kernel position t)"""
    w = wpack.view(C, 3, C).permute(0, 2, 1)
    return w.reshape(C, C, 3, 1) if vertical else w.reshape(C, C, 1, 3)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W,C,vertical,dil", SMALL)
@pytest.mark.parametrize("transposed", [False, True])
def test_reference_matches_torch_conv(N, H, W, C, vertical, dil, transposed):
    """TF32-exact operands (quantisation is the identity): the fp64 restatement is conv2d (forward taps) or
    conv_transpose2d (input-gradient taps, weights [Ci][3*Co] = pack_tc_dgrad) in float64."""
    x, w, _ = _x(N, H, W, C, dil)
    x, w = cc.tf32_rna(x), cc.tf32_trunc(w)
    ref, S = cc.conv_fp64(x, w, cc.TC_TF32, cc.tap_list(vertical, dil, transposed))
    pad, dl = ((dil, 0), (dil, 1)) if vertical else ((0, dil), (1, dil))
    w4 = _w4(w, C, vertical).double()
    if transposed:   # out[ci] = sum_co dy[co] * w[co][ci] at the transposed taps: pack_tc_dgrad(w4T) = the slot matrix
        t = F.conv_transpose2d(_nchw(x.double()), w4.transpose(0, 1), padding=pad, dilation=dl)
    else:
        t = F.conv2d(_nchw(x.double()), w4, padding=pad, dilation=dl)
    want = t.permute(0, 2, 3, 1).reshape(-1, C)
    assert torch.allclose(ref, want, rtol=0, atol=1e-12 * float(S.max()))
    assert bool((S >= ref.abs() - 1e-12).all())


def test_reference_any_three_taps_and_x3_terms():
    """arbitrary taps (some wholly outside the image) = explicit shifted sums; the 3xTF32 reference is the full product
    of (hi + lo) (w_hi + w_lo) less lo * lo"""
    N, H, W, C = 2, 8, 16, 64
    x, w, _ = _x(N, H, W, C, 5)
    taps = [(0, -1), (9, 0), (2, 3)]
    ref, _ = cc.conv_fp64(x, cc.pack_weights(w, cc.TC_BF16), cc.TC_BF16, taps)
    xq, wq = cc.bf16_rne(x).double(), cc.bf16_rne(w).double()
    want = torch.zeros(N, H, W, C, dtype=torch.float64)
    for t, (dy, dx) in enumerate(taps):
        for y in range(H):
            for x_ in range(W):
                if 0 <= y + dy < H and 0 <= x_ + dx < W:
                    want[:, y, x_] += xq[:, y + dy, x_ + dx] @ wq[:, t * C:(t + 1) * C].t()
    assert torch.allclose(ref, want.reshape(-1, C), rtol=0, atol=1e-12)
    wp = cc.pack_weights(w, cc.TC_X3)
    r3, _ = cc.conv_fp64(x, wp, cc.TC_X3, taps)
    hi, lo = (t.double() for t in cc.split_tf32(x))
    whi, wlo = wp[0].double(), wp[1].double()
    full = _plain(hi + lo, whi + wlo, taps)
    assert torch.allclose(r3, full - _plain(lo, wlo, taps), rtol=0, atol=1e-12)


@pytest.mark.parametrize("N,H,W,C,vertical,dil", SMALL)
@pytest.mark.parametrize("transposed", [False, True])
def test_fp8_reference_matches_torch_conv_of_quantised_operands(N, H, W, C, vertical, dil, transposed):
    """FP8: the restatement is float64 conv2d / conv_transpose2d of the activations quantised per image and the weights
    quantised per output channel (oracle/fp8_oracle.py), times the fp32 factors (x_amax[n] / 448) * w_scale[co]; an
    all-zero image and an all-zero output channel give exactly 0."""
    from oracle import fp8_oracle as fo
    x, w, x_amax, _ = _x_fp8(N, H, W, C, dil + 3 * transposed)
    x[N // 2] = 0
    x_amax[N // 2] = 0
    w[5] = 0
    wp, sw = cc.pack_weights(w, cc.TC_FP8), cc.fp8_weight_scale(w)
    ref, S = cc.conv_fp64(x, wp, cc.TC_FP8, cc.tap_list(vertical, dil, transposed), scales=(x_amax, sw))
    w4 = _w4(w, C, vertical)
    qw, sw4 = fo.quantize_weight(w4)
    assert torch.equal(sw4, sw) and torch.equal(_w4(cc.weight_terms(wp, cc.TC_FP8)[0].float(), C, vertical), qw)
    qx = fo.quantize_act(_nchw(x), x_amax).double()
    pad, dl = ((dil, 0), (dil, 1)) if vertical else ((0, dil), (1, dil))
    if transposed:
        t = F.conv_transpose2d(qx, qw.double().transpose(0, 1), padding=pad, dilation=dl)
    else:
        t = F.conv2d(qx, qw.double(), padding=pad, dilation=dl)
    dq = (fo.scale(x_amax).view(-1, 1, 1, 1) * sw.view(1, -1, 1, 1)).double()
    want = (t * dq).permute(0, 2, 3, 1).reshape(-1, C)
    assert torch.allclose(ref, want, rtol=0, atol=1e-12 * float(S.max()))
    assert bool((S >= ref.abs() - 1e-12 * float(S.max())).all())
    zero = ref.view(N, H, W, C)
    assert not bool(zero[N // 2].any()) and not bool(zero[..., 5].any())


def test_e4m3_quantiser_is_round_to_nearest_even_satfinite():
    """e4m3_rne (cvt.rn.satfinite.e4m3x2.f32) on every code: itself; half way between two codes, the even one (also
    between the subnormals and across the normal boundary); just off half way, the nearer one; beyond 448, 448.  And the
    two sensitivity roundings differ from it where they should."""
    codes = torch.arange(0, 0x7f, dtype=torch.int16)                     # 0 .. 448 (0x7f is NaN)
    v = codes.to(torch.uint8).view(torch.float8_e4m3fn).float()
    assert v[1] == 2.0 ** -9 and v[8] == 2.0 ** -6 and v[-1] == 448.0
    for s in (1.0, -1.0):
        assert torch.equal(cc.e4m3_rne(s * v), s * v)
        mid = s * (v[:-1] + v[1:]) / 2
        even = torch.where(codes[:-1] % 2 == 0, v[:-1], v[1:])
        assert torch.equal(cc.e4m3_rne(mid), s * even)
        up = torch.nextafter(mid, torch.full_like(mid, s * 1e9))
        assert torch.equal(cc.e4m3_rne(up), s * v[1:])
        assert torch.equal(cc.e4m3_rne(torch.nextafter(mid, torch.zeros_like(mid))), s * v[:-1])
        assert torch.equal(cc.e4m3_rtz(mid), s * v[:-1])
        big = torch.tensor([448.5, 464.0, 480.0, 1e6, float("inf")]) * s
        assert torch.equal(cc.e4m3_rne(big), torch.full_like(big, 448.0 * s))
    sub = v[1:8]
    assert torch.equal(cc.e4m3_ftz(sub), torch.zeros_like(sub)) and torch.equal(cc.e4m3_ftz(v[8:]), v[8:])


def _plain(a, w, taps):
    C = a.shape[-1]
    return sum(cc.shifted(a, *taps[t]).reshape(-1, C) @ w[:, t * C:(t + 1) * C].t() for t in range(3))


EPI = [dict(), dict(bias=1, relu=1), dict(mask=1), dict(mask=1, affine=1), dict(add=1), dict(add=1, add_mask=1),
       dict(mask=1, add=1), dict(bias=1, add=1, relu=2), dict(bias=1, relu=3, mask=1, add=1, add_mask=1)]


def _epi_tensors(spec, N, H, W, C, g):
    kw = {}
    if "bias" in spec:
        kw["bias"] = torch.randn(C, generator=g)
    kw["relu"] = spec.get("relu", 0)
    if "mask" in spec:
        kw["mask_src"] = torch.randn(N, H, W, C, generator=g)
    if "affine" in spec:
        kw["mask_affine"] = (torch.randn(C, generator=g), torch.randn(C, generator=g))
    if "add" in spec:
        kw["add_src"] = torch.randn(N, H, W, C, generator=g)
    if "add_mask" in spec:
        kw["add_mask"] = torch.randn(N, H, W, C, generator=g)
    return kw


@pytest.mark.parametrize("spec", EPI, ids=["+".join(sorted(s)) or "none" for s in EPI])
def test_epilogue_matches_the_header(spec):
    N, H, W, C = 1, 8, 16, 64
    g = torch.Generator().manual_seed(len(spec))
    z = torch.randn(N * H * W, C, generator=g, dtype=torch.float64)
    S = z.abs() * 3
    kw = _epi_tensors(spec, N, H, W, C, g)
    out, Sp, adds = cc.epilogue(z, S, **kw)
    v = z.clone()
    if kw.get("bias") is not None:
        v = v + kw["bias"].double()
    if kw["relu"] & 1:
        v = torch.relu(v)
    if kw.get("mask_src") is not None:
        m = kw["mask_src"].double().reshape(-1, C)
        if kw.get("mask_affine") is not None:
            m = m * kw["mask_affine"][0].double() + kw["mask_affine"][1].double()
        v = v * (m > 0)
    if kw.get("add_src") is not None:
        a = kw["add_src"].double().reshape(-1, C)
        if kw.get("add_mask") is not None:
            a = a * (kw["add_mask"].reshape(-1, C) > 0)
        v = v + a
    if kw["relu"] & 2:
        v = torch.relu(v)
    assert torch.equal(out, v)
    assert adds == int(kw.get("bias") is not None) + int(kw.get("add_src") is not None)
    assert bool((Sp >= S).all())


# ---------------------------------------------------------------------------------------------------------------------
# the emulation passes, the seeded bugs fail
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [cc.TC_TF32, cc.TC_X3, cc.TC_BF16], ids=["tf32", "tf32x3", "bf16"])
@pytest.mark.parametrize("si", range(len(SMALL)))
def test_emulation_passes_and_seeded_bugs_fail(prec, si):
    N, H, W, C, vertical, dil = SMALL[si]
    for transposed in (False, True):
        taps = cc.tap_list(vertical, dil, transposed)
        pl = _plan(N, H, W, C, taps, prec)
        pl["m_ctas"] = 3                        # several tiles per CTA row whatever the host's SM count
        x, w, g = _x(N, H, W, C, 10 * si + transposed)
        wp = cc.pack_weights(w, prec)
        spec = EPI[(si + 2 * transposed) % len(EPI)]
        kw = _epi_tensors(spec, N, H, W, C, g)
        out, colsum, stats = cc.emulate(x, wp, prec, taps, pl, **kw)
        z, S = cc.conv_fp64(x, wp, prec, taps)
        ref, Sp, adds = cc.epilogue(z, S, **kw)
        nsteps = cc.steps(C, prec, adds)
        assert cc.excess(out, ref, Sp, nsteps, prec) <= 1.0

        def fails(r):
            return cc.excess(r, ref, Sp, nsteps, prec) > 1.0
        mut = lambda **m: cc.epilogue(cc.conv_fp64(x, wp, prec, taps, **m)[0], S, **kw)[0]  # noqa: E731
        assert fails(mut(shift_tap=1)), "a tap shifted by one pixel"
        assert fails(mut(drop_chunk=(1, C // cc.KCH - 1))), "a dropped chunk"
        t_neg = 0 if (taps[0][0] if vertical else taps[0][1]) < 0 else 2
        r = mut(halo_zero=(t_neg, pl["TA"], pl["vertical"]))
        if (H if vertical else W) > pl["TA"] and dil < (H if vertical else W):
            assert fails(r), "a halo row read as zero"
        if prec == cc.TC_X3:
            assert fails(mut(drop_lo_hi=True)), "a dropped a_lo * w_hi"

        # partials: the emulated per-CTA sums pass their gate, a map shifted by one does not
        rows, _, _ = cc.tile_map(N, H, W, pl)
        psteps = cc.partial_steps(N, H, W, pl)
        o = out.double()
        second = o * (kw["mask_src"].double().reshape(-1, C) if kw.get("mask_affine") is not None else o)
        for got, vals in ((colsum, o), (stats[:, 0], o), (stats[:, 1], second)):
            pref = cc.partial_fp64(vals, rows, 3)
            pS = cc.partial_fp64(vals.abs(), rows, 3)
            assert cc.excess(got, pref, pS, psteps, prec, c_tc=0.0) <= 1.0
            assert cc.excess(cc.partial_fp64(vals, (rows + 1) % 3, 3), pref, pS, psteps, prec, c_tc=0.0) > 1.0


FP8_EPI = [s for s in EPI if "affine" not in s]          # lf_conv1d_tc_fp8 takes no affine mask (nor partials)


@pytest.mark.parametrize("cls", ["randn", "subnormal", "ties"])
@pytest.mark.parametrize("si", range(len(SMALL)))
def test_fp8_emulation_passes_and_seeded_bugs_fail(si, cls):
    """the FP8 emulation passes the gate and its out_amax is the per-image max; a shifted tap, a dropped chunk, a halo row
    read as zero, the next image's scale, flushed subnormals (subnormal class) and round-toward-zero (ties class) fail"""
    N, H, W, C, vertical, dil = SMALL[si]
    N = max(N, 3)                                        # images with different scales
    for transposed in (False, True):
        taps = cc.tap_list(vertical, dil, transposed)
        pl = _plan(N, H, W, C, taps, cc.TC_FP8)
        x, w, x_amax, g = _x_fp8(N, H, W, C, 10 * si + transposed, cls)
        wp, sw = cc.pack_weights(w, cc.TC_FP8), cc.fp8_weight_scale(w)
        kw = _epi_tensors(FP8_EPI[(si + 2 * transposed) % len(FP8_EPI)], N, H, W, C, g)
        out, _, _ = cc.emulate(x, wp, cc.TC_FP8, taps, pl, scales=(x_amax, sw), **kw)
        z, S = cc.conv_fp64(x, wp, cc.TC_FP8, taps, scales=(x_amax, sw))
        ref, Sp, adds = cc.epilogue(z, S, **kw)
        nsteps = cc.steps(C, cc.TC_FP8, adds)
        assert cc.excess(out, ref, Sp, nsteps, cc.TC_FP8) <= 1.0
        am = cc.image_amax(out, N)
        assert torch.equal(am, out.abs().view(N, -1).amax(1)) and len(set(am.tolist())) == N

        def fails(**m):
            r = cc.epilogue(cc.conv_fp64(x, wp, cc.TC_FP8, taps, scales=(x_amax, sw), **m)[0], S, **kw)[0]
            return cc.excess(r, ref, Sp, nsteps, cc.TC_FP8) > 1.0
        assert fails(shift_tap=1), "a tap shifted by one pixel"
        assert fails(drop_chunk=(1, C // cc.KCH - 1)), "a dropped chunk"
        t_neg = 0 if (taps[0][0] if vertical else taps[0][1]) < 0 else 2
        if (H if vertical else W) > pl["TA"] and dil < (H if vertical else W):
            assert fails(halo_zero=(t_neg, pl["TA"], pl["vertical"])), "a halo row read as zero"
        if cls == "ties":
            assert fails(a_round=cc.e4m3_rtz), "round toward zero"
        else:
            assert fails(next_image_scale=True), "image n with image n+1's scale"
        if cls == "subnormal":
            assert fails(a_round=cc.e4m3_ftz), "flushed e4m3 subnormals"


@pytest.mark.parametrize("prec,cls",[(cc.TC_TF32, "ties"), (cc.TC_TF32, "ties_w"), (cc.TC_BF16, "ties_bf16")])
def test_rounding_mutations_fail_on_ties(prec, cls):
    """on ties the kernel's rounding passes and every other rounding fails: RNE for the TF32 activations' RNA, RNA for the
    bf16 RNE, rounding (either way) for the truncated TF32 weights"""
    N, H, W, C, vertical, dil = SMALL[0]
    taps = cc.tap_list(vertical, dil)
    x, w, _ = _x(N, H, W, C, 3, cls)
    wp = cc.pack_weights(w, prec)
    pl = _plan(N, H, W, C, taps, prec)
    out, _, _ = cc.emulate(x, wp, prec, taps, pl)
    ref, S = cc.conv_fp64(x, wp, prec, taps)
    nsteps = cc.steps(C, prec, 0)
    assert cc.excess(out, ref, S, nsteps, prec) <= 1.0
    if cls == "ties_w":
        others = [dict(w_round=cc.tf32_rna), dict(w_round=cc.tf32_rne)]
    else:
        others = [dict(a_round=cc.tf32_rne if prec == cc.TC_TF32 else cc.bf16_rna)]
    for m in others:
        r, _ = cc.conv_fp64(x, wp, prec, taps, **m)
        assert cc.excess(r, ref, S, nsteps, prec) > 1.0, m


def test_c_tc_below_its_ceiling():
    assert all(cc.C_TC[p] <= cc.C_TC_CEILING[p] for p in cc.C_TC)


# ---------------------------------------------------------------------------------------------------------------------
# the plan query and the coverage table
# ---------------------------------------------------------------------------------------------------------------------
def test_coverage_table_reaches_every_planner_outcome():
    seen = set()
    for (prec, abf, C, H, W, v, d, var), key in cc.COVERAGE:
        rc, pl = cc.with_variant(var, lambda: cc.query_plan(prec, int(abf), 3, H, W, C, cc.tap_list(v, d)))
        assert rc == 0 and cc.plan_key(prec, int(abf), C, pl) == key, (prec, abf, C, H, W, v, d, var, rc, pl)
        seen.add(key)
    universe = cc.universe_keys()
    missing = {k: universe[k] for k in set(universe) - seen}
    assert not missing, "planner outcomes no GPU case launches: %s" % missing
    assert seen <= set(universe)


def test_plan_query_matches_the_public_queries():
    """the slab / per-tap choice, the rows of the partials and 3xTF32's refusals agree with lf_conv1d_tc_slab_ok,
    lf_conv1d_tc_supported and lf_conv1d_tc_x3_rows"""
    from lanedetection_end2end_b200 import _capi
    h = _capi.lib()
    if h.lf_conv1d_tc_supported(2, 32, 64, 64) == 0:
        pytest.skip("the public queries need the driver's tensor-map encoder")
    for N, H, W, C in ((2, 32, 64, 64), (3, 40, 80, 128), (1, 4, 256, 64), (2, 32, 4, 128)):
        for v in (0, 1):
            for d in (1, 2, 8, 16, 40):
                taps = cc.tap_list(v, d)
                rc, pl = cc.query_plan(cc.TC_TF32, 0, N, H, W, C, taps)
                assert rc == 0 and pl["slab"] == h.lf_conv1d_tc_slab_ok(N, H, W, C, v, d)
                assert pl["m_ctas"] == h.lf_conv1d_tc_supported(N, H, W, C)
                rc3, pl3 = cc.query_plan(cc.TC_X3, 0, N, H, W, C, taps)
                assert (pl3["m_ctas"] if rc3 == 0 else 0) == h.lf_conv1d_tc_x3_rows(N, H, W, C, v, d)


def test_plan_query_refuses_bad_arguments():
    from lanedetection_end2end_b200 import _capi
    h = _capi.lib()
    t3 = (ctypes.c_int * 3)(0, 0, 0)
    info = (ctypes.c_int * _capi.TC_PLAN_INFO)()
    ok = (0, 0, 2, 32, 64, 64, t3, t3, info)
    assert h.lf_conv1d_tc_plan(*ok) == 0 or h.lf_conv1d_tc_plan(*ok) == -2
    for i, bad in ((0, -1), (0, 4), (1, 2), (2, 0), (3, 0), (4, -3), (6, None), (7, None), (8, None)):
        a = list(ok)
        a[i] = bad
        assert h.lf_conv1d_tc_plan(*a) == -1, (i, bad)
    assert h.lf_conv1d_tc_plan(0, 1, 2, 32, 64, 64, t3, t3, info) == -2          # bf16 input: BF16 / FP8 only
    assert h.lf_conv1d_tc_plan(2, 1, 2, 32, 64, 48, t3, t3, info) == -2          # C = 48


# ---------------------------------------------------------------------------------------------------------------------
# argument checks of the entry points
# ---------------------------------------------------------------------------------------------------------------------
P_ = 4096   # a non-NULL pointer that is never dereferenced: every call below is refused before the planner


def _args(**kw):
    from lanedetection_end2end_b200 import _capi
    a = _capi.LfConvTcArgs()
    a.inp = a.wpack = a.out = P_
    a.N, a.H, a.W, a.C = 2, 32, 64, 64
    for i in range(3):
        a.dy[i], a.dx[i] = 0, i - 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


REFUSED = [dict(inp=None), dict(wpack=None), dict(out=None), dict(mask_scale=P_), dict(mask_scale=P_, mask_shift=P_),
           dict(mask_scale=P_, mask_shift=P_, mask_src=P_), dict(mask_scale=P_, mask_src=P_, stats_partial=P_),
           dict(in_dtype=2), dict(out_dtype=-1), dict(mask_dtype=7), dict(N=0), dict(H=0), dict(W=0), dict(N=-1, H=-2),
           dict(H=-1, W=-64), dict(N=-3)]


@pytest.mark.parametrize("entry", ["lf_conv1d_tc", "lf_conv1d_tc_x3", "lf_conv1d_tc_bf16"])
def test_entry_points_refuse_bad_arguments(entry):
    from lanedetection_end2end_b200 import _capi
    fn = getattr(_capi.lib(), entry)
    assert fn(None, None) == -1
    for kw in REFUSED:
        assert fn(ctypes.byref(_args(**kw)), None) == -1, (entry, kw)
    # bf16 operands on the fp32 entry points: LF_ERR_UNSUPPORTED (checked before the planner too)
    if entry != "lf_conv1d_tc_bf16":
        for kw in (dict(in_dtype=1), dict(out_dtype=1), dict(mask_dtype=1)):
            assert fn(ctypes.byref(_args(**kw)), None) == -2, (entry, kw)


def test_fp8_entry_point_refuses_bad_arguments():
    """lf_conv1d_tc_fp8 shares tc_run's checks, and takes no gradient-side outputs"""
    from lanedetection_end2end_b200 import _capi
    fn = _capi.lib().lf_conv1d_tc_fp8
    assert fn(None, None) == -1

    def f8(**kw):
        f = _capi.LfConvTcFp8Args()
        f.conv = _args()
        f.x_amax = f.w_scale = f.out_amax = P_
        for k, v in kw.items():
            if hasattr(f, k) and k in ("x_amax", "w_scale", "out_amax"):
                setattr(f, k, v)
            else:
                setattr(f.conv, k, v)
        return f
    for kw in REFUSED + [dict(x_amax=None), dict(w_scale=None), dict(out_amax=None), dict(colsum_partial=P_),
                         dict(stats_partial=P_)]:
        assert fn(ctypes.byref(f8(**kw)), None) == -1, kw
