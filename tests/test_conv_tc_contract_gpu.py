"""lf_conv1d_tc (TF32), lf_conv1d_tc_x3 (3xTF32), lf_conv1d_tc_bf16 and lf_conv1d_tc_fp8 driven directly through their
C entry points, entry by entry against the fp64 restatement of their contract (tests/conv_tc_contract.py).

Every case builds LfConvTcArgs (LfConvTcFp8Args) by hand and launches into sentinel-filled buffers with guard regions on
both sides of `out`, colsum_partial, stats_partial and out_amax (whose body starts at zero).  Each output entry is held
to the per-entry gate |got - ref| <= (c_tc + steps*2^-23) * S'; every partial row must be written and equal, to its own
gate, the fp64 sum of the kernel's stored output over that CTA's tiles (tile map from lf_conv1d_tc_plan); the guards
must stay untouched.  Cases:
  * coverage: one launch per planner outcome (C, precision, bf16 input, resident / streamed weights, slab / per-tap,
    3xTF32 lo buffer plan, single stage), asserted through lf_conv1d_tc_plan;
  * production: every non_bottleneck_1d layer shape of the 256x512 and 320x640 configurations (the C = 16 layers as their
    C = 64 super-pixel view), forward and input-gradient tap order, TF32, 3xTF32, BF16 and BF16 with bf16 input, FP8
    with fp32 and bf16 input (the C = 128 shapes at batch 32);
  * edges: fewer tiles than SMs, 3+ tiles per CTA, dilations at and beyond the extent, the per-tap fallback shapes (and
    3xTF32's LF_ERR_UNSUPPORTED there), non-symmetric taps, both lf_conv1d_tc_set_variant values; for FP8, CTAs that
    run 3+ tiles and move from one image to the next partway through them (derived from the plan's tile map);
  * operands: randn, post-ReLU, heavy-tailed, an all-zero 32-channel chunk, and rounding ties (low bits 0x1000 for TF32,
    0x8000 for bf16) on the activations or on the weights; for FP8 every image at its own scale (six decades apart), an
    all-zero output channel, and three e4m3 classes: one outlier per image so that most operands are e4m3 subnormals,
    e4m3 midpoints under x_amax = 448 (inv = 1 exactly), and an all-zero image in the batch;
  * epilogues: bias, both ReLU bits, mask_src, the affine mask, add_src with and without add_mask, mask_src together with
    add_src, colsum and statistics (also on the per-tap plan), bf16 `out` (== the fp32 result rounded to nearest even,
    partials unchanged) and bf16 `mask_src`; FP8 runs every combination its entry takes (no partials, no affine mask);
  * FP8 out_amax: exactly the per-image max |stored value| (of the bf16 values for a bf16 `out`), with the per-image
    maxima pairwise distinct so that a maximum reduced into the wrong image cannot pass;
  * per case, in fp64: a tap shifted by one pixel, a dropped 32-channel chunk, a halo row read as zero (slab plans), the
    other operand rounding on the ties classes (RNE for the TF32 RNA, RNA for the bf16 RNE, rounded for the truncated TF32
    weights), a dropped a_lo * w_hi (3xTF32) and a tile-to-CTA map shifted by one must each break the gate; for FP8 also
    image n quantised and dequantised with image n+1's scale, flushed e4m3 subnormals (subnormal class) and
    round-toward-zero (midpoint class).
The largest |err| / S, c_tc use and gate headroom per precision, and the device, are printed at the end (pytest -s).
"""
import ctypes

import pytest
import torch

import conv_tc_contract as cc

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -1.2345e30                     # sentinel: a value no launch here produces
GUARD = 2048                          # elements of sentinel before and after every output
# out_amax's guard: atomicMax on the float bits only raises an entry, so its sentinel is the smallest positive float,
# which any stray maximum of a tile overwrites
AMAX_SENT = 2.0 ** -149
CLASSES = ("randn", "relu", "heavy", "zero_chunk")
FP8_CLASSES = CLASSES + ("subnormal", "ties_a", "zero_image")
MEASURED = {}                         # prec -> [max |err|/S, max c_tc use, max gate excess]
EPILOGUES = [
    ("bias", "relu1"), ("bias", "stats"), ("mask", "colsum"), ("mask", "affine", "stats"), ("add",), ("add", "add_mask"),
    ("mask", "add"), ("mask", "add", "add_mask", "colsum"), ("bias", "add", "relu2"),
    ("bias", "relu1", "add", "relu2", "colsum"), ("bias", "mask", "affine", "add", "stats"), (),
]


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED:
        print(torch.cuda.get_device_name())
    for prec, (rel, use, exc) in sorted(MEASURED.items()):
        print("%s: max |err|/S %.3e, max c_tc use %.3e (c_tc %.3e, ceiling %.3e), gate headroom %.1fx"
              % (cc.ENTRIES[prec], rel, use, cc.C_TC[prec], cc.C_TC_CEILING[prec], 1.0 / max(exc, 1e-30)))
    assert all(c <= cc.C_TC_CEILING[p] for p, c in cc.C_TC.items())


def _record(prec, got, ref, S, nsteps):
    m = MEASURED.setdefault(prec, [0.0, -float("inf"), 0.0])
    m[0] = max(m[0], cc.rel_err(got, ref, S))
    m[1] = max(m[1], cc.tc_usage(got, ref, S, nsteps))
    m[2] = max(m[2], cc.excess(got, ref, S, nsteps, prec))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g):
    return torch.randn(shape, generator=g, device=DEV)


def _exact(t, prec):
    """t made exact in the precision's operand form (so that its rounding is the identity)."""
    return cc.bf16_rne(t) if prec == cc.TC_BF16 else cc.tf32_trunc(t)


def _ties(t, prec):
    """non-negative values whose low bits are exactly half a step: a systematic rounding direction shows in every sum"""
    bits, width = (0x8000, 16) if prec == cc.TC_BF16 else (0x1000, 13)
    return cc.with_low_bits(t.abs() + 2.0 ** -20, bits, width)


def _e4m3_midpoints(shape, g):
    """non-negative values exactly half way between two adjacent e4m3 values, subnormal and normal, below 448"""
    codes = torch.randint(0, 0x7e, shape, generator=g, device=DEV, dtype=torch.int16)   # code 0x7e = 448
    lo = codes.to(torch.uint8).view(torch.float8_e4m3fn).float()
    hi = (codes + 1).to(torch.uint8).view(torch.float8_e4m3fn).float()
    return (lo + hi) / 2


def _operands(cls, prec, N, H, W, C, seed):
    g = _gen(seed)
    x = _randn((N, H, W, C), g)
    w = _randn((C, 3 * C), g) / (3 * C) ** 0.5
    if prec == cc.TC_FP8:
        # images scaled over six decades (every image its own activation scale), an all-zero output channel (w_scale 0)
        w[5] = 0
        scale = (10.0 ** torch.linspace(-3, 3, N, device=DEV))[torch.randperm(N, generator=g, device=DEV)]
        x = x * scale.view(-1, 1, 1, 1)
        if cls == "subnormal":      # one outlier per image: most quantised activations are e4m3 subnormals
            x.view(N, -1)[:, 7] = x.abs().flatten(1).amax(1) * 2.0 ** 14
        elif cls == "ties_a":       # run with x_amax = 448 (inv = 1 exactly): every activation is an e4m3 midpoint
            x, w = _e4m3_midpoints((N, H, W, C), g), w.abs()
        elif cls == "zero_image":
            x[N // 2] = 0
    if cls == "relu":
        x = x.clamp_min(0)
    elif cls == "heavy":
        x = x * torch.exp(2 * _randn((N, H, W, C), g))
    elif cls == "zero_chunk":
        x[..., :cc.KCH] = 0
    elif cls == "ties_a" and prec != cc.TC_FP8:
        x, w = _ties(x, prec), _exact(w.abs(), prec)
    elif cls == "ties_w":
        x, w = _exact(x.abs(), prec), _ties(w, prec)
    return x, w, g


class Launch:
    """One lf_conv1d_tc* launch into sentinel-filled, guarded buffers.  FP8 (scales = (x_amax, w_scale)): out_amax is
    zero with AMAX_SENT guards on both sides."""

    def __init__(self, prec, x, wpack, taps, plan, epi, out_bf16=False, mask_bf16=False, tensors=None, scales=None):
        c = _capi()
        N, H, W, C = x.shape
        self.N, self.P, self.C, self.rows = N, N * H * W, C, plan["m_ctas"]
        self.abuf = None
        if prec == cc.TC_FP8:
            self.abuf = torch.full((2 * GUARD + N,), AMAX_SENT, device=DEV)
            self.abuf[GUARD:GUARD + N] = 0
        t = tensors
        odt = torch.bfloat16 if out_bf16 else torch.float32
        self.obuf = torch.full((2 * GUARD + self.P * C,), SENT, dtype=odt, device=DEV)
        self.cbuf = torch.full((2 * GUARD + self.rows * C,), SENT, device=DEV) if "colsum" in epi else None
        self.sbuf = (torch.full((2 * GUARD + self.rows * 2 * C,), SENT, dtype=torch.float64, device=DEV)
                     if "stats" in epi else None)
        a = c.LfConvTcArgs()
        a.inp, a.wpack = x.data_ptr(), wpack.data_ptr()
        a.out = self.obuf[GUARD:].data_ptr()
        a.bias = t["bias"].data_ptr() if "bias" in epi else None
        if "mask" in epi:
            m = t["mask"].to(torch.bfloat16) if mask_bf16 else t["mask"]
            self.mask = m
            a.mask_src = m.data_ptr()
        if "affine" in epi:
            a.mask_scale, a.mask_shift = t["scale"].data_ptr(), t["shift"].data_ptr()
        if "add" in epi:
            a.add_src = t["add"].data_ptr()
            if "add_mask" in epi:
                a.add_mask = t["add_mask"].data_ptr()
        if self.cbuf is not None:
            a.colsum_partial = self.cbuf[GUARD:].data_ptr()
        if self.sbuf is not None:
            a.stats_partial = self.sbuf[GUARD:].data_ptr()
        a.N, a.H, a.W, a.C = N, H, W, C
        for i, (dy, dx) in enumerate(taps):
            a.dy[i], a.dx[i] = dy, dx
        a.relu = (1 if "relu1" in epi else 0) | (2 if "relu2" in epi else 0)
        a.in_dtype = c.dtype_id(x)
        a.out_dtype = c.LF_BF16 if out_bf16 else c.LF_F32
        a.mask_dtype = c.LF_BF16 if ("mask" in epi and mask_bf16) else c.LF_F32
        if prec == cc.TC_FP8:
            f = c.LfConvTcFp8Args()
            f.conv = a
            f.x_amax, f.w_scale = scales[0].data_ptr(), scales[1].data_ptr()
            f.out_amax = self.abuf[GUARD:].data_ptr()
            self.rc = c.lib().lf_conv1d_tc_fp8(ctypes.byref(f), c.stream_ptr())
        else:
            self.rc = getattr(c.lib(), cc.ENTRIES[prec])(ctypes.byref(a), c.stream_ptr())
        torch.cuda.synchronize()

    def amax(self):
        return self.abuf[GUARD:GUARD + self.N]

    def check_guards(self, tag):
        if self.abuf is not None:
            guards = torch.cat([self.abuf[:GUARD], self.abuf[GUARD + self.N:]])
            assert bool((guards == AMAX_SENT).all()), "%s: wrote outside out_amax" % tag
        for name, buf in (("out", self.obuf), ("colsum_partial", self.cbuf), ("stats_partial", self.sbuf)):
            if buf is None:
                continue
            s = torch.tensor(SENT, dtype=buf.dtype)
            assert bool((buf[:GUARD] == s.to(DEV)).all()) and bool((buf[-GUARD:] == s.to(DEV)).all()), \
                "%s: wrote outside %s" % (tag, name)
            body = buf[GUARD:-GUARD]
            assert not bool((body == s.to(DEV)).any()), "%s: an entry of %s was not written" % (tag, name)

    def out(self):
        return self.obuf[GUARD:-GUARD].view(self.P, self.C)

    def colsum(self):
        return self.cbuf[GUARD:-GUARD].view(self.rows, self.C)

    def stats(self):
        return self.sbuf[GUARD:-GUARD].view(self.rows, 2, self.C)


def _epi_for(prec, epi):
    """the epilogue as the precision's entry takes it: FP8 refuses colsum, statistics and the affine mask"""
    return tuple(e for e in epi if e not in ("colsum", "stats", "affine")) if prec == cc.TC_FP8 else epi


def _must_fail(tag, what, got, ref, S, nsteps, prec, c_tc=None):
    x = cc.excess(got, ref, S, nsteps, prec, c_tc)
    assert x > 1.0, "%s: %s stays within the gate (%.3g)" % (tag, what, x)


def run_case(prec, C, N, H, W, taps, epi=(), cls="randn", abf=False, out_bf16=False, mask_bf16=False, variant=2, seed=0,
             key=None, mutations=True):
    """Launch one case and check it entry by entry; returns the plan."""
    c = _capi()
    tag = "%s C%d %dx%dx%d taps%s %s %s%s%s var%d" % (cc.PREC_NAMES[prec], C, N, H, W, taps, cls, "+".join(epi),
                                                    " abf" if abf else "", " obf" if out_bf16 else "", variant)
    in_dtype = c.LF_BF16 if abf else c.LF_F32
    rc, plan = cc.with_variant(variant, lambda: cc.query_plan(prec, in_dtype, N, H, W, C, taps))
    assert rc == 0, "%s: the plan query refuses the case (%d)" % (tag, rc)
    if key is not None:
        assert cc.plan_key(prec, in_dtype, C, plan) == key, (tag, cc.plan_key(prec, in_dtype, C, plan), key)
    x, w, g = _operands(cls, prec, N, H, W, C, seed)
    if abf:
        x = x.to(torch.bfloat16)
    wpack = cc.pack_weights(w, prec)
    scales = None
    if prec == cc.TC_FP8:
        x_amax = torch.full((N,), 448.0, device=DEV) if cls == "ties_a" else x.float().abs().flatten(1).amax(1)
        scales = (x_amax, cc.fp8_weight_scale(w))
    t = {"bias": _randn((C,), g), "mask": _randn((N, H, W, C), g), "add": _randn((N, H, W, C), g),
         "add_mask": _randn((N, H, W, C), g), "scale": _randn((C,), g), "shift": _randn((C,), g)}
    if mask_bf16:
        t["mask"] = t["mask"].to(torch.bfloat16).float()       # the same mask in both forms
    run = lambda ob: cc.with_variant(variant, lambda: Launch(prec, x, wpack, taps, plan, epi, ob, mask_bf16, t, scales))  # noqa: E731
    L = run(False)
    assert L.rc == 0, "%s: the launch returned %d" % (tag, L.rc)
    L.check_guards(tag)
    got = L.out()
    if prec == cc.TC_FP8:                       # out_amax: exactly the per-image max |stored value|
        am = cc.image_amax(got, N)
        assert torch.equal(L.amax(), am), "%s: out_amax %s != the per-image max %s" % (tag, L.amax().tolist(),
                                                                                      am.tolist())
        assert len(set(am.tolist())) == N, "%s: per-image maxima not distinct, a misattributed one could pass" % tag
    if out_bf16:                                # a bf16 `out` is the fp32 result rounded, with the same partials
        Lb = run(True)
        assert Lb.rc == 0
        Lb.check_guards(tag + " bf16 out")
        assert torch.equal(Lb.out(), got.to(torch.bfloat16)), "%s: bf16 out != the fp32 result rounded" % tag
        if prec == cc.TC_FP8:
            assert torch.equal(Lb.amax(), am.to(torch.bfloat16).float()), "%s: bf16 out_amax != the rounded max" % tag
            assert torch.equal(Lb.amax(), cc.image_amax(Lb.out(), N)), "%s: bf16 out_amax != the stored max" % tag
        if L.cbuf is not None:
            assert torch.equal(Lb.colsum(), L.colsum()), "%s: bf16 out changes the column sums" % tag
        if L.sbuf is not None:
            assert torch.equal(Lb.stats(), L.stats()), "%s: bf16 out changes the statistics" % tag

    epi_kw = dict(bias=t["bias"] if "bias" in epi else None,
                  relu=(1 if "relu1" in epi else 0) | (2 if "relu2" in epi else 0),
                  mask_src=t["mask"] if "mask" in epi else None,
                  mask_affine=(t["scale"], t["shift"]) if "affine" in epi else None,
                  add_src=t["add"] if "add" in epi else None,
                  add_mask=t["add_mask"] if "add_mask" in epi else None)
    z, S = cc.conv_fp64(x, wpack, prec, taps, scales=scales)
    ref, Sp, adds = cc.epilogue(z, S, **epi_kw)
    nsteps = cc.steps(C, prec, adds)
    _record(prec, got, ref, Sp, nsteps)
    x_ = cc.excess(got, ref, Sp, nsteps, prec)
    assert x_ <= 1.0, "%s: |err| reaches %.3g x the gate" % (tag, x_)

    rows, _, _ = cc.tile_map(N, H, W, plan, DEV)
    psteps = cc.partial_steps(N, H, W, plan)
    o = got.double()
    checks = []
    if L.cbuf is not None:
        checks.append(("colsum", L.colsum(), o))
    if L.sbuf is not None:
        st = L.stats()
        checks.append(("stats sum", st[:, 0], o))
        checks.append(("stats second", st[:, 1], o * (t["mask"].double().reshape(-1, C) if "affine" in epi else o)))
    for what, part, vals in checks:
        pref = cc.partial_fp64(vals, rows, plan["m_ctas"])
        pS = cc.partial_fp64(vals.abs(), rows, plan["m_ctas"])
        xp = cc.excess(part, pref, pS, psteps, prec, c_tc=0.0)
        assert xp <= 1.0, "%s: %s partial reaches %.3g x its gate" % (tag, what, xp)
        if mutations and plan["m_ctas"] > 1:
            _must_fail(tag, "a tile-to-CTA map shifted by one (%s)" % what,
                       cc.partial_fp64(vals, (rows + 1) % plan["m_ctas"], plan["m_ctas"]), pref, pS, psteps, prec, 0.0)

    if mutations:
        mut = lambda **m: cc.epilogue(cc.conv_fp64(x, wpack, prec, taps, scales=scales, **m)[0], S, **epi_kw)[0]  # noqa: E731
        _must_fail(tag, "a tap shifted by one pixel", mut(shift_tap=1), ref, Sp, nsteps, prec)
        _must_fail(tag, "a dropped chunk", mut(drop_chunk=(1, C // cc.KCH - 1)), ref, Sp, nsteps, prec)
        if plan["slab"]:
            t_neg = 0 if (taps[0][0] if plan["vertical"] else taps[0][1]) < 0 else 2
            r2 = mut(halo_zero=(t_neg, plan["TA"], plan["vertical"]))
            if not torch.equal(r2, ref):
                _must_fail(tag, "a halo row read as zero", r2, ref, Sp, nsteps, prec)
        if prec == cc.TC_X3 and cls == "randn":
            _must_fail(tag, "a dropped a_lo * w_hi", mut(drop_lo_hi=True), ref, Sp, nsteps, prec)
        if prec == cc.TC_FP8:
            if not torch.equal(scales[0], scales[0].roll(-1)):
                _must_fail(tag, "image n with image n+1's scale", mut(next_image_scale=True), ref, Sp, nsteps, prec)
            if cls == "subnormal":
                _must_fail(tag, "flushed e4m3 subnormals", mut(a_round=cc.e4m3_ftz), ref, Sp, nsteps, prec)
            if cls == "ties_a":
                _must_fail(tag, "e4m3 rounding toward zero", mut(a_round=cc.e4m3_rtz), ref, Sp, nsteps, prec)
        elif cls == "ties_a" and prec != cc.TC_X3 and not abf:
            other = cc.tf32_rne if prec == cc.TC_TF32 else cc.bf16_rna
            _must_fail(tag, "the other activation rounding", mut(a_round=other), ref, Sp, nsteps, prec)
        if cls == "ties_w" and prec == cc.TC_TF32:
            for other in (cc.tf32_rna, cc.tf32_rne):
                _must_fail(tag, "rounded instead of truncated weights (%s)" % other.__name__, mut(w_round=other), ref, Sp,
                           nsteps, prec)
    return plan


# =====================================================================================================================
# coverage: every planner outcome
# =====================================================================================================================
def _cov_id(case):
    (p, abf, C, H, W, v, d, var), _ = case
    return "%s%s-C%d-%dx%d-%s%d-var%d" % (cc.PREC_NAMES[p], "-abf" if abf else "", C, H, W, "v" if v else "h", d, var)


@pytest.mark.parametrize("i", range(len(cc.COVERAGE)), ids=[_cov_id(c) for c in cc.COVERAGE])
def test_every_planner_outcome_against_fp64(i):
    (prec, abf, C, H, W, v, d, var), key = cc.COVERAGE[i]
    cls = FP8_CLASSES[i % len(FP8_CLASSES)] if prec == cc.TC_FP8 else (CLASSES + ("ties_a", "ties_w"))[i % 6]
    bf = prec in (cc.TC_BF16, cc.TC_FP8)
    for j, dgrad in enumerate((False, True)):
        epi = _epi_for(prec, EPILOGUES[(2 * i + j) % len(EPILOGUES)])
        run_case(prec, C, 3, H, W, cc.tap_list(v, d, dgrad), epi, cls=cls, abf=abf, variant=var, seed=10 * i + j,
                 out_bf16=bf and j == 1, mask_bf16=bf and "mask" in epi and "affine" not in epi, key=key)


# =====================================================================================================================
# production layer shapes
# =====================================================================================================================
SHAPES = [  # C, H, W, vertical, dil: the 3-tap layers of the 256x512 and 320x640 configurations
    (64, 64, 128, True, 1), (64, 64, 128, False, 1), (64, 128, 64, True, 1), (64, 128, 64, False, 1),
    (64, 80, 160, True, 1), (64, 80, 160, False, 1), (64, 160, 80, True, 1), (64, 160, 80, False, 1),
] + [(128, 32, 64, v, d) for d in (1, 2, 4, 8, 16) for v in (True, False)] + [
    (128, 40, 80, v, d) for d in (1, 2, 4, 8, 16) for v in (True, False)]
MODES = [(cc.TC_TF32, False), (cc.TC_X3, False), (cc.TC_BF16, False), (cc.TC_BF16, True)]


def _shape_id(s):
    C, H, W, v, d = s
    return "C%d-%dx%d-%s%d" % (C, H, W, "v" if v else "h", d)


@pytest.mark.parametrize("mode", MODES, ids=["tf32", "tf32x3", "bf16", "bf16-abf"])
@pytest.mark.parametrize("si", range(len(SHAPES)), ids=[_shape_id(s) for s in SHAPES])
def test_production_layer_shapes_against_fp64(si, mode):
    prec, abf = mode
    C, H, W, v, d = SHAPES[si]
    k = si * 4 + MODES.index(mode)
    for j, dgrad in enumerate((False, True)):
        epi = EPILOGUES[(2 * k + j) % len(EPILOGUES)]
        run_case(prec, C, 2, H, W, cc.tap_list(v, d, dgrad), epi, cls=CLASSES[(k + j) % 4], abf=abf, seed=1000 + 2 * k + j,
                 out_bf16=prec == cc.TC_BF16 and (k + j) % 3 == 0, mask_bf16=prec == cc.TC_BF16 and "affine" not in epi)


@pytest.mark.parametrize("abf", [False, True], ids=["fp8", "fp8-abf"])
@pytest.mark.parametrize("si", range(len(SHAPES)), ids=[_shape_id(s) for s in SHAPES])
def test_fp8_production_layer_shapes_against_fp64(si, abf):
    """FP8 at the layer shapes, the C = 128 ones at batch 32 (8 to 25 tiles per CTA, most CTAs crossing images), the
    C = 64 super-pixel views at batch 8"""
    C, H, W, v, d = SHAPES[si]
    N = 32 if C == 128 else 8
    k = 2 * si + abf
    for j, dgrad in enumerate((False, True)):
        epi = _epi_for(cc.TC_FP8, EPILOGUES[(2 * k + j) % len(EPILOGUES)])
        pl = run_case(cc.TC_FP8, C, N, H, W, cc.tap_list(v, d, dgrad), epi, cls=FP8_CLASSES[(k + j) % len(FP8_CLASSES)],
                      abf=abf, seed=3000 + 2 * k + j, out_bf16=(k + j) % 3 == 0, mask_bf16=(k + j) % 2 == 0)
        assert _crosses_images(N, H, W, pl), pl


# =====================================================================================================================
# edges
# =====================================================================================================================
PRECS = [(cc.TC_TF32, False), (cc.TC_X3, False), (cc.TC_BF16, False), (cc.TC_BF16, True)]
PREC_IDS = ["tf32", "tf32x3", "bf16", "bf16-abf"]


@pytest.mark.parametrize("mode", PRECS, ids=PREC_IDS)
def test_fewer_tiles_than_ctas_and_many_tiles_per_cta(mode):
    prec, abf = mode
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pl = run_case(prec, 64, 1, 16, 128, cc.tap_list(False, 1), ("bias", "colsum"), abf=abf, seed=1)
    assert pl["m_ctas"] == 16 < sms
    for C, N, H, W, v, d in ((128, 16, 32, 64, True, 2), (64, 8, 64, 128, False, 1)):
        pl = run_case(prec, C, N, H, W, cc.tap_list(v, d, True), ("mask", "add", "stats"), cls="heavy", abf=abf, seed=2)
        assert cc.tiles_per_cta(N, H, W, pl) >= 3, pl


@pytest.mark.parametrize("mode", PRECS, ids=PREC_IDS)
def test_dilation_at_and_beyond_the_extent(mode):
    """taps wholly outside the image: only the centre tap contributes"""
    prec, abf = mode
    for C, H, W, v, d in ((128, 32, 64, True, 32), (128, 32, 64, True, 40), (64, 16, 64, False, 64), (64, 32, 32, False, 33)):
        for dgrad in (False, True):
            run_case(prec, C, 2, H, W, cc.tap_list(v, d, dgrad), ("bias", "relu1", "stats"), abf=abf, seed=d + dgrad)


@pytest.mark.parametrize("mode", [m for m in PRECS if m[0] != cc.TC_X3], ids=["tf32", "bf16", "bf16-abf"])
def test_per_tap_fallback_shapes(mode):
    """shapes the slab does not take run one box per tap (TF32, BF16); statistics on that plan included"""
    prec, abf = mode
    for C, N, H, W, v, d in ((64, 3, 4, 256, False, 1), (128, 2, 32, 4, True, 1), (64, 2, 32, 12, True, 1)):
        for j, epi in enumerate((("bias", "stats"), ("mask", "affine", "stats"), ("mask", "add", "colsum"))):
            pl = run_case(prec, C, N, H, W, cc.tap_list(v, d, j == 1), epi, cls=CLASSES[j], abf=abf, seed=j + C)
            assert not pl["slab"]


def test_x3_refuses_the_per_tap_shapes():
    c = _capi()
    for C, N, H, W, v, d in ((64, 3, 4, 256, False, 1), (128, 2, 32, 4, True, 1), (64, 2, 32, 12, True, 1)):
        taps = cc.tap_list(v, d)
        assert cc.query_plan(cc.TC_X3, c.LF_F32, N, H, W, C, taps)[0] == -2
        x = torch.zeros(N, H, W, C, device=DEV)
        wp = torch.zeros(2, C, 3 * C, device=DEV)
        L = Launch(cc.TC_X3, x, wp, taps, {"m_ctas": 1}, ())
        assert L.rc == -2, L.rc
        assert bool((L.obuf == SENT).all()), "a refused launch wrote its output"


NONSYM = [[(0, -1), (0, 0), (2, 3)], [(1, 1), (-3, 0), (0, 5)], [(-8, 0), (0, 0), (0, -40)]]


@pytest.mark.parametrize("mode", [m for m in PRECS if m[0] != cc.TC_X3], ids=["tf32", "bf16", "bf16-abf"])
def test_non_symmetric_taps_on_the_per_tap_plan(mode):
    prec, abf = mode
    for i, taps in enumerate(NONSYM):
        for C in (64, 128):
            pl = run_case(prec, C, 2, 32, 64, taps, EPILOGUES[i + C // 32], cls=CLASSES[i], abf=abf, seed=i + C)
            assert not pl["slab"]


@pytest.mark.parametrize("mode", PRECS, ids=PREC_IDS)
@pytest.mark.parametrize("cls", ["ties_a", "ties_w"])
def test_rounding_ties_on_slab_and_per_tap(mode, cls):
    """ties on the activations pin RNA (TF32 / 3xTF32) and RNE (bf16); ties on the weights pin the truncation of raw fp32
    TF32 weights"""
    prec, abf = mode
    for variant in ((2, 1) if prec != cc.TC_X3 else (2,)):
        for C, H, W, v, d in ((64, 64, 128, False, 1), (128, 40, 80, True, 4)):
            run_case(prec, C, 2, H, W, cc.tap_list(v, d), ("bias",), cls=cls, abf=abf, variant=variant, seed=C + d)


# =====================================================================================================================
# FP8 (lf_conv1d_tc_fp8): per-image scales and maxima where a CTA runs several tiles
# =====================================================================================================================
def _cta_images(N, H, W, plan):
    """[[image of each tile CTA row r runs, in order] for every r]: tile m runs on CTA row m % m_ctas (tile_map)."""
    tiles_img = H * W // cc.TILE
    m = plan["m_ctas"]
    return [[mt // tiles_img for mt in range(r, N * tiles_img, m)] for r in range(m)]


def _crosses_images(N, H, W, plan):
    """some CTA runs consecutive tiles of different images (its scale and its out_amax image change between them)"""
    return any(a != b for seq in _cta_images(N, H, W, plan) for a, b in zip(seq, seq[1:]))


@pytest.mark.parametrize("abf", [False, True], ids=["fp8", "fp8-abf"])
def test_fp8_many_tiles_per_cta_across_image_boundaries(abf):
    """batches whose CTAs run 3+ tiles each and move from one image to the next partway through them; every class"""
    for i, (C, N, H, W, v, d) in enumerate(((64, 7, 64, 128, False, 1), (128, 9, 40, 80, True, 2),
                                            (64, 5, 80, 160, True, 1), (128, 11, 32, 64, False, 4))):
        for j, cls in enumerate(FP8_CLASSES):
            epi = _epi_for(cc.TC_FP8, EPILOGUES[(3 * i + j) % len(EPILOGUES)])
            pl = run_case(cc.TC_FP8, C, N, H, W, cc.tap_list(v, d, j % 2 == 1), epi, cls=cls, abf=abf, seed=50 * i + j,
                          out_bf16=j % 3 == 1, mask_bf16=j % 2 == 0)
            seqs = _cta_images(N, H, W, pl)
            assert max(len(s) for s in seqs) >= 3 and _crosses_images(N, H, W, pl), (C, N, H, W, pl)


@pytest.mark.parametrize("abf", [False, True], ids=["fp8", "fp8-abf"])
def test_fp8_fewer_tiles_than_ctas(abf):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for C, N, H, W, cls in ((64, 1, 16, 128, "subnormal"), (64, 3, 8, 128, "zero_image"), (128, 3, 32, 32, "ties_a")):
        pl = run_case(cc.TC_FP8, C, N, H, W, cc.tap_list(False, 1), ("bias", "relu1"), cls=cls, abf=abf, seed=C + N)
        assert pl["m_ctas"] == N * H * W // cc.TILE < sms // (C // 64), pl


@pytest.mark.parametrize("abf", [False, True], ids=["fp8", "fp8-abf"])
def test_fp8_dilation_at_and_beyond_the_extent(abf):
    """taps wholly outside the image: only the centre tap contributes"""
    for i, (C, H, W, v, d) in enumerate(((128, 32, 64, True, 32), (128, 32, 64, True, 40), (64, 16, 64, False, 64),
                                         (64, 32, 32, False, 33))):
        for dgrad in (False, True):
            run_case(cc.TC_FP8, C, 3, H, W, cc.tap_list(v, d, dgrad), ("bias", "relu1"),
                     cls=FP8_CLASSES[(2 * i + dgrad) % len(FP8_CLASSES)], abf=abf, seed=d + dgrad)


@pytest.mark.parametrize("variant", [2, 1])
@pytest.mark.parametrize("abf", [False, True], ids=["fp8", "fp8-abf"])
def test_fp8_both_variants(variant, abf):
    """the halo slab and the one-box-per-tap kernel, on the e4m3 classes (subnormals, midpoints, an all-zero image)"""
    for i, (C, N, H, W, v, d) in enumerate(((64, 4, 64, 128, False, 1), (128, 5, 40, 80, True, 4))):
        for j, cls in enumerate(("subnormal", "ties_a", "zero_image")):
            pl = run_case(cc.TC_FP8, C, N, H, W, cc.tap_list(v, d, j == 1), ("bias",) if j else (), cls=cls, abf=abf,
                          variant=variant, seed=C + d + j)
            assert bool(pl["slab"]) == (variant == 2)


FP8_EPI_ALL = [tuple(e for e in (b, r1, m, a, am, r2) if e)
               for b in ("", "bias") for r1 in ("", "relu1") for r2 in ("", "relu2") for m in ("", "mask")
               for a, am in (("", ""), ("add", ""), ("add", "add_mask"))]


def test_fp8_every_epilogue_combination():
    """bias, both ReLU bits, mask_src (fp32 and bf16), add_src with and without add_mask, fp32 and bf16 `out`: every
    combination lf_conv1d_tc_fp8 takes; an all-zero image under the epilogues that keep it zero leaves out_amax at 0"""
    for i, epi in enumerate(FP8_EPI_ALL):
        cls = "zero_image" if not ({"bias", "add"} & set(epi)) else FP8_CLASSES[i % len(FP8_CLASSES)]
        run_case(cc.TC_FP8, 64, 3, 16, 64, cc.tap_list(i % 2 == 0, 1 + i % 3, i % 4 >= 2), epi, cls=cls, abf=i % 5 == 0,
                 seed=700 + i, out_bf16=i % 2 == 1, mask_bf16=i % 4 == 1)
