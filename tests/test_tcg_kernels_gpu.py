"""lf_wgrad_tcg, lf_wgrad_reduce and lf_conv_tcg driven directly through their C entry points, entry by entry against
the fp64 restatement of their contracts (tests/tcg_contract.py).

Every case builds the args struct by hand over strided NHWC views, launches, and holds every output entry -- each
CTA's partial, the reduced result, every conv output -- to the per-entry gate |got - ref| <= (c_tc + steps*2^-23) * S,
where ref and S = sum |a_q b_q| come from the quantised operands.  Around that:
  * every one of the 14 lf_wgrad_tcg instances (Nn in {32, 64, 96, 128} x TF32 / 3xTF32 / BF16, bf16 A views at Nn 64 and
    128) at sizes where each CTA runs well over the 8-stage ring;
  * block tables of 1 .. 24 blocks (odd ones included), two views with different offsets and strides, permuted channel
    blocks, taps of 0, +-1 .. +-16 pixels and taps whose boxes lie wholly outside the image;
  * split counts 1, the library's own, one that does not divide the patches, and more CTAs than patches (those
    partials must be exactly 0);
  * operands: randn, post-ReLU, heavy-tailed, an all-zero channel block, and non-negative values on rounding ties;
  * bitwise determinism, exact power-of-two scale equivariance, sentinel guards after the partial and around the
    conv output;
  * per case, in fp64: dropping a patch / k-step, shifting a tap by one pixel, or rounding ties the other way must
    each break the gate -- so the case would see those bugs.
The largest |err| / S and c_tc use per precision are printed at the end (pytest -s).
"""
import ctypes
import random

import pytest
import torch

import tcg_contract as tc

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = -1.2345e30                     # sentinel: a value no kernel here produces
GUARD = 4096                          # floats of sentinel after the partial
CLASSES = ("randn", "relu", "heavy", "zero_block", "ties")
MEASURED = {}                         # (kernel, prec) -> [max |err|/S, max c_tc use]
S2_TAPS = [(1, -1, -1), (1, -1, 0), (0, 0, -1), (0, 0, 0), (1, 0, -1), (1, 0, 0)]   # ops_net.TCG_S2CONV_TAPS


def _capi():
    from lanedetection_end2end_b200 import _capi as c
    return c


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (kern, prec), (rel, use, exc) in sorted(MEASURED.items()):
        print("%s precision %d: max |err|/S %.3e, max c_tc use %.3e (c_tc %.3e), gate headroom %.1fx"
              % (kern, prec, rel, use, tc.C_TC[prec], 1.0 / max(exc, 1e-30)))
    assert all(c <= tc.C_TC_CEILING[p] for p, c in tc.C_TC.items())


def _record(kern, prec, got, ref, S, steps):
    m = MEASURED.setdefault((kern, prec), [0.0, 0.0, 0.0])
    m[0] = max(m[0], tc.rel_err(got, ref, S))
    m[1] = max(m[1], tc.tc_usage(got, ref, S, steps))
    m[2] = max(m[2], tc.gate_excess(got, ref, S, steps, prec))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g):
    return torch.randn(shape, generator=g, device=DEV)


def _operand(shape, cls, prec, g, zero_c0=None):
    """fp32 operand of class cls; zero_c0: first channel of the block that class zero_block clears."""
    if cls == "relu":
        return _randn(shape, g).clamp_min(0)
    if cls == "heavy":
        return _randn(shape, g) * torch.exp(2 * _randn(shape, g))
    if cls == "ties":
        # non-negative, so a systematic rounding direction shows in every sum
        bits, width = (0x8000, 16) if prec == tc.TC_BF16 else (0x1000, 13)
        return tc.with_low_bits(_randn(shape, g).abs() + 2.0 ** -20, bits, width)
    t = _randn(shape, g)
    if cls == "zero_block" and zero_c0 is not None:
        t[..., zero_c0:zero_c0 + 32] = 0
    return t


def _view(t, off, H, W, sn, sy, sx):
    v = _capi().LfTcgView()
    v.ptr, v.H, v.W, v.sn, v.sy, v.sx = t.data_ptr() + t.element_size() * off, H, W, sn, sy, sx
    return v


def _check_excess(what, got, ref, S, steps, prec, must_pass=True):
    x = tc.gate_excess(got, ref, S, steps, prec)
    if must_pass:
        assert x <= 1.0, "%s: |err| reaches %.3g x the gate" % (what, x)
    return x


# =====================================================================================================================
# lf_wgrad_tcg
# =====================================================================================================================
INSTANCES = [(nn, p, False) for p in (0, 1, 2) for nn in (32, 64, 96, 128)] + [(64, 2, True), (128, 2, True)]


class WgradCase:
    """Storage, views and block table of one lf_wgrad_tcg launch family, plus the fp64 pieces of its reference."""

    def __init__(self, inst, N, Hs, Ws, nb, layout, b_wide, seed):
        self.Nn, self.prec, self.abf = inst
        self.N, self.Hs, self.Ws, self.nb, self.layout, self.b_wide, self.seed = N, Hs, Ws, nb, layout, b_wide, seed
        self.bx, self.by = tc.wgt_pick_patch(Hs, Ws)
        self.total = N * (Hs // self.by) * (Ws // self.bx)
        rng = random.Random(seed)
        if layout == "pair":                     # the pair-pixel / row-parity views of the stride-2 layers
            C = 64
            self.Ka, self.a_shape = 2 * C, (N, 2 * Hs, 2 * Ws, C)
            sn, sy, sx = 4 * Hs * Ws * C, 4 * Ws * C, 2 * C
            self.vspec = [(0, Hs, Ws, sn, sy, sx), (2 * Ws * C, Hs, Ws, sn, sy, sx)]
            taps = [S2_TAPS[(i + 3) % 6] for i in range(6)]
        elif layout == "wide":                   # view 1: other offset (row 1, channel 32) and row stride (every other row)
            self.Ka = 64 if nb < 6 else 128
            Kw = self.Ka + 32
            self.a_shape = (N, Hs + 2, Ws, Kw)
            sn = (Hs + 2) * Ws * Kw
            self.vspec = [(0, Hs, Ws, sn, Ws * Kw, Kw), (Ws * Kw + 32, (Hs + 1) // 2, Ws, sn, 2 * Ws * Kw, Kw)]
            taps = None
        else:
            self.Ka = 64
            self.a_shape = (N, Hs, Ws, self.Ka)
            self.vspec = [(0, Hs, Ws, Hs * Ws * self.Ka, Ws * self.Ka, self.Ka)]
            taps = None
        nk = self.Ka // 32
        perm = list(range(nk))
        rng.shuffle(perm)
        pool = [(0, 1), (0, -1), (1, 0), (-1, 0), (0, 2), (-2, 0), (0, 4), (4, 0), (0, -8), (8, 0), (0, 16), (-16, 0),
                (0, -33), (33, 0), (Hs + 3, 0), (0, -(Ws + 2))]
        self.blocks = []
        for i in range(nb):
            if taps is not None:
                m, dy, dx = taps[(i // nk) % 6]
            else:
                m = (i % 2) if len(self.vspec) > 1 else 0
                dy, dx = (0, 0) if i == 0 else ((Hs + 3, 0) if i == 2 else pool[rng.randrange(len(pool))])
            self.blocks.append((m, dy, dx, perm[(i + i // nk) % nk]))
        if b_wide:                               # B: a 32-channel-offset slice of a wider buffer
            Kb = self.Nn + 32
            self.b_shape, self.bspec = (N, Hs, Ws, Kb), (32, Hs, Ws, Hs * Ws * Kb, Ws * Kb, Kb)
        else:
            self.b_shape, self.bspec = (N, Hs, Ws, self.Nn), (0, Hs, Ws, Hs * Ws * self.Nn, Ws * self.Nn, self.Nn)
        self.pix = tc.patch_pixels(N, Hs, Ws, self.bx, self.by, DEV)

    def operands(self, cls):
        g = _gen(self.seed * 7 + CLASSES.index(cls))
        A = _operand(self.a_shape, cls, self.prec, g, zero_c0=self.a_shape[-1] - 32)
        B = _operand(self.b_shape, cls, self.prec, g, zero_c0=self.bspec[0] + self.Nn - 32 if self.Nn >= 64 else None)
        if self.abf:
            A = A.to(torch.bfloat16)
        return A, B

    def gathered(self, A, B, rows=None, shift=None):
        """raw (unquantised, fp64) [pix, nb*32] A columns and [pix, Nn] B rows in patch order; rows: a slice of the
        patch-ordered pixels; shift = (block, ddx): that block's tap moved by ddx pixels."""
        n, y, x = (t[rows] if rows is not None else t for t in self.pix)
        fa = A.reshape(-1).double()
        cols = []
        for i, (m, dy, dx, cb) in enumerate(self.blocks):
            off, H, W, sn, sy, sx = self.vspec[m]
            ddx = shift[1] if shift is not None and shift[0] == i else 0
            cols.append(tc.gather(fa, off, H, W, sn, sy, sx, n, y + dy, x + dx + ddx, 32 * cb, 32))
        off, H, W, sn, sy, sx = self.bspec
        return torch.cat(cols, 1), tc.gather(B.reshape(-1).double(), off, H, W, sn, sy, sx, n, y, x, 0, self.Nn)

    def quantised(self, Ga, Gb, rounding=None):
        qa = Ga if self.abf else tc.quantise(Ga.float(), self.prec, rounding)
        return qa, tc.quantise(Gb.float(), self.prec, rounding)

    def lib_ctas(self):
        min_patches = 8 if self.prec == tc.TC_X3 else 4
        return int(_capi().lib().lf_wgrad_tcg_ctas(self.N, self.Hs, self.Ws, self.Ka, self.Nn, self.nb, min_patches))

    def launch(self, A, B, nctas):
        c = _capi()
        rows = self.nb * 32
        partial = torch.full((nctas * rows * self.Nn + GUARD,), SENT, device=DEV)
        a = c.LfWgradTcgArgs()
        for i, s in enumerate(self.vspec):
            a.a[i] = _view(A, *s)
        a.b = _view(B, *self.bspec)
        a.partial, a.N, a.Hs, a.Ws, a.Ka, a.Nn, a.nblocks, a.nctas = partial.data_ptr(), self.N, self.Hs, self.Ws, self.Ka, \
            self.Nn, self.nb, nctas
        a.precision, a.a_dtype = self.prec, (c.LF_BF16 if self.abf else c.LF_F32)
        for i, (m, dy, dx, cb) in enumerate(self.blocks):
            a.map[i], a.dy[i], a.dx[i], a.cblk[i] = m, dy, dx, cb
        c.call("lf_wgrad_tcg", ctypes.byref(a), c.stream_ptr())
        assert bool((partial[nctas * rows * self.Nn:] == SENT).all()), "lf_wgrad_tcg wrote past its partial"
        return partial[:nctas * rows * self.Nn].view(nctas, rows, self.Nn)

    def reduce(self, partial):
        c = _capi()
        nctas, rows, Nn = partial.shape
        dst = torch.full((rows, Nn), SENT, device=DEV)
        c.call("lf_wgrad_reduce", c.ptr(partial), nctas, 1, rows, Nn, rows, Nn, c.ptr(dst), 0, Nn, 1, c.stream_ptr())
        return dst


def _check_wgrad(case, cls, splits, scale=False, sensitivity=True):
    A, B = case.operands(cls)
    Ga, Gb = case.gathered(A, B)
    Qa, Qb = case.quantised(Ga, Gb)
    ref, S = tc.exact_and_abs(Qa, Qb)
    tag = "Nn=%d prec=%d abf=%d %s N=%d %dx%d nb=%d %s" % (case.Nn, case.prec, case.abf, cls, case.N, case.Hs, case.Ws,
                                                         case.nb, case.layout)
    lib = case.lib_ctas()
    assert lib >= 1
    for nctas in splits:
        nctas = lib if nctas == "lib" else nctas
        part = case.launch(A, B, nctas)
        ranges, per = tc.cta_patch_ranges(case.total, nctas)
        for c_, (p0, p1) in enumerate(ranges):
            if p0 == p1:
                assert bool((part[c_] == 0).all()), "%s nctas=%d: CTA %d has no patches but a non-zero partial" % (tag, nctas, c_)
                continue
            r_, s_ = tc.exact_and_abs(Qa[p0 * 32:p1 * 32], Qb[p0 * 32:p1 * 32])
            _record("wgrad_tcg", case.prec, part[c_], r_, s_, per + 1)
            _check_excess("%s nctas=%d partial %d" % (tag, nctas, c_), part[c_], r_, s_, per + 1, case.prec)
        red = case.reduce(part)
        _check_excess("%s nctas=%d reduced" % (tag, nctas), red, ref, S, per + 1 + nctas, case.prec)
        if nctas == lib:
            assert torch.equal(case.launch(A, B, nctas), part), "%s: two launches differ" % tag
            if scale:
                for k in (20, -20):
                    got = case.launch(A * 2.0 ** k, B, nctas)
                    assert torch.equal(got, part * 2.0 ** k), "%s: 2^%d A does not scale the partials exactly" % (tag, k)
            if sensitivity:
                _wgrad_sensitivity(case, tag, A, B, Qa, Qb, ranges, per)


def _wgrad_sensitivity(case, tag, A, B, Qa, Qb, ranges, per):
    """In fp64, each of these bugs moves some entry of the last CTA's partial past the gate."""
    p0, p1 = [r for r in ranges if r[0] < r[1]][-1]
    rows = slice(p0 * 32, p1 * 32)
    ref, S = tc.exact_and_abs(Qa[rows], Qb[rows])
    steps = per + 1
    # the last 32-pixel patch dropped
    last = slice(p1 * 32 - 32, p1 * 32)
    x = _check_excess("", ref - Qa[last].t() @ Qb[last], ref, S, steps, case.prec, must_pass=False)
    assert x > 1.0, "%s: a dropped patch stays within the gate (%.3g)" % (tag, x)
    # the tap of the block with the largest operands shifted by one pixel
    blk = int(Qa[rows].abs().sum(0).view(case.nb, 32).sum(1).argmax())
    Ga, Gb = case.gathered(A, B, rows=rows, shift=(blk, 1))
    Sa, Sb = case.quantised(Ga, Gb)
    x = _check_excess("", Sa.t() @ Sb, ref, S, steps, case.prec, must_pass=False)
    assert x > 1.0, "%s: a tap shifted by one pixel stays within the gate (%.3g)" % (tag, x)


def _wgrad_rounding_sensitivity(case, tag, cls):
    """Ties rounded the other way (RNE for the TF32 RNA, RNA for the bf16 RNE) break the gate; 3xTF32 carries the rounding
    error in its lo part, so either rounding gives the same hi + lo."""
    A, B = case.operands(cls)
    ranges, per = tc.cta_patch_ranges(case.total, case.lib_ctas())
    p0, p1 = [r for r in ranges if r[0] < r[1]][-1]
    Ga, Gb = case.gathered(A, B, rows=slice(p0 * 32, p1 * 32))
    Qa, Qb = case.quantised(Ga, Gb)
    ref, S = tc.exact_and_abs(Qa, Qb)
    Ra, Rb = case.quantised(Ga, Gb, rounding=tc.tf32_rne if case.prec == tc.TC_TF32 else tc.bf16_rna)
    x = _check_excess("", Ra.t() @ Rb, ref, S, per + 1, case.prec, must_pass=False)
    assert x > 1.0, "%s: the other tie rounding stays within the gate (%.3g)" % (tag, x)


# realistic sizes: N = 32 at 32x64, N = 16 at 64x128 and at the super-pixel 128x64; every table size, layout and B view
_SHAPES = [(32, 32, 64), (16, 64, 128), (16, 128, 64)]
_TABLES = [24, 1, 16, 3, 12, 5, 6]
_LAYOUTS = ["pair", "wide", "dense"]
BIG = []
for _i, _inst in enumerate(INSTANCES):
    _layout = _LAYOUTS[_i % 3]
    _nb = 24 if _layout == "pair" and _i % 2 == 0 else _TABLES[_i % 7]
    if _layout == "dense":
        _nb = min(_nb, 6)
    BIG.append((_inst, _SHAPES[_i % 3], _nb, _layout, _i % 2 == 1, 100 + _i))


def _big_id(c):
    (nn, p, abf), (N, H, W), nb, layout, bw, _ = c
    return "Nn%d-p%d%s-%dx%dx%d-nb%d-%s%s" % (nn, p, "-abf" if abf else "", N, H, W, nb, layout, "-bwide" if bw else "")


@pytest.mark.parametrize("case", BIG, ids=_big_id)
def test_wgrad_tcg_every_instance_against_fp64(case):
    inst, (N, Hs, Ws), nb, layout, b_wide, seed = case
    wc = WgradCase(inst, N, Hs, Ws, nb, layout, b_wide, seed)
    assert wc.total // max(1, wc.lib_ctas()) > 8, "each CTA must turn the 8-stage ring"
    for cls in CLASSES:
        _check_wgrad(wc, cls, [1, "lib", 7] if cls == "randn" else ["lib"], scale=cls in ("randn", "heavy"),
                     sensitivity=cls != "zero_block")
    if inst[1] != tc.TC_X3:
        _wgrad_rounding_sensitivity(wc, _big_id(case), "ties")


# every patch shape wgt_pick_patch can take (bx = 32 .. 1), small enough for more CTAs than patches
SMALL = [(INSTANCES[i], Ws, [1, 3, 5, 6][i % 4], _LAYOUTS[(i + 1) % 3], i % 2 == 0, 200 + i)
         for i, Ws in zip(range(len(INSTANCES)), [64, 48, 24, 20, 6, 5] * 3)]


def _small_id(c):
    (nn, p, abf), Ws, nb, layout, bw, _ = c
    return "Nn%d-p%d%s-Ws%d-nb%d-%s%s" % (nn, p, "-abf" if abf else "", Ws, nb, layout, "-bwide" if bw else "")


@pytest.mark.parametrize("case", SMALL, ids=_small_id)
def test_wgrad_tcg_patch_shapes_and_splits(case):
    inst, Ws, nb, layout, b_wide, seed = case
    wc = WgradCase(inst, 2, 32, Ws, nb, layout if layout != "pair" else "wide", b_wide, seed)
    assert wc.bx == {64: 32, 48: 16, 24: 8, 20: 4, 6: 2, 5: 1}[Ws]
    for cls in CLASSES:
        _check_wgrad(wc, cls, [1, "lib", 7, wc.total + 3] if cls == "randn" else ["lib"], scale=cls == "randn",
                     sensitivity=cls != "zero_block")


def test_wgrad_tcg_accepts_and_rejects_as_declared():
    """lf_wgrad_tcg_ctas: 24 blocks at Nn = 128 are supported (a CTA takes one pair of blocks whatever Nn is); 25 blocks, Nn
    not a multiple of 32 or above 128, Ka not a multiple of 32 and shapes without a 32-pixel patch are not."""
    lib = _capi().lib()
    assert lib.lf_wgrad_tcg_ctas(32, 32, 64, 128, 128, 24, 4) >= 1
    for args in [(32, 32, 64, 128, 128, 25, 4), (32, 32, 64, 128, 48, 4, 4), (32, 32, 64, 128, 160, 4, 4),
                 (32, 32, 64, 80, 64, 4, 4), (1, 3, 5, 64, 64, 2, 4), (32, 32, 64, 64, 64, 2, 0)]:
        assert lib.lf_wgrad_tcg_ctas(*args) == 0, args


# =====================================================================================================================
# lf_wgrad_reduce
# =====================================================================================================================
@pytest.mark.parametrize("nsplit,ntaps,Cp,Cq,CpPad,CqPad", [(1, 1, 32, 32, 32, 32), (7, 3, 61, 29, 64, 32),
                                                            (40, 2, 16, 13, 20, 16), (133, 1, 5, 3, 8, 4)])
def test_wgrad_reduce_strided_destination(nsplit, ntaps, Cp, Cq, CpPad, CqPad):
    c = _capi()
    g = _gen(nsplit + Cp)
    part = _randn((nsplit, ntaps, CpPad, CqPad), g) * torch.exp(2 * _randn((nsplit, ntaps, CpPad, CqPad), g))
    part[:, :, Cp:] = float("nan")                      # padding rows / columns must not be read into the result
    part[:, :, :, Cq:] = float("nan")
    # destination: [Cq][ntaps][Cp] with a gap, i.e. st = Cp + 3, sp = 1, sq = ntaps * (Cp + 3) + 5
    st, sp, sq = Cp + 3, 1, ntaps * (Cp + 3) + 5
    dst = torch.full((Cq * sq + 64,), SENT, device=DEV)
    c.call("lf_wgrad_reduce", c.ptr(part), nsplit, ntaps, Cp, Cq, CpPad, CqPad, c.ptr(dst), st, sp, sq, c.stream_ptr())
    t, p, q = torch.meshgrid(torch.arange(ntaps), torch.arange(Cp), torch.arange(Cq), indexing="ij")
    idx = (t * st + p * sp + q * sq).reshape(-1).to(DEV)
    body = part[:, :, :Cp, :Cq].double()
    ref, S = body.sum(0).reshape(-1), body.abs().sum(0).reshape(-1)
    got = dst[idx]
    assert bool(((got.double() - ref).abs() <= nsplit * tc.ULP * S).all())
    mask = torch.ones_like(dst, dtype=torch.bool)
    mask[idx] = False
    assert bool((dst[mask] == SENT).all()), "lf_wgrad_reduce wrote outside its destination entries"


# =====================================================================================================================
# lf_conv_tcg
# =====================================================================================================================
_CONV_SHAPES = [(64, 128), (32, 64), (16, 32), (8, 16), (16, 8), (32, 4), (64, 2), (128, 3)]   # (Hs, Ws): bx = 128 .. 1


def _conv_cases():
    cases = []
    i = 0
    for prec in (0, 1, 2):
        for Ng in range(16, 129, 16):
            Hs, Ws = _CONV_SHAPES[(i + prec) % 8]
            N = 4 if Hs * Ws >= 4096 else 8               # >= 256 tiles on the first two shapes (persistent loop)
            Kc = (32, 64, 256)[i % 3]
            ntaps = 1 + (i * 4) % 9 if Kc < 256 else 1 + i % 3
            cases.append((prec, Ng, Kc, ntaps, N, Hs, Ws, i % 2 == 0, i % 4 < 2, (1, 0) if i % 3 == 0 else (2, i % 2), 300 + i))
            i += 1
    return cases


CONV = _conv_cases()


def _conv_id(c):
    prec, Ng, Kc, nt, N, Hs, Ws, bias, relu, (om, o0), _ = c
    return "p%d-Ng%d-Kc%d-t%d-%dx%dx%d%s%s-oy%d.%d" % (prec, Ng, Kc, nt, N, Hs, Ws, "-bias" if bias else "",
                                                      "-relu" if relu else "", om, o0)


class ConvCase:
    def __init__(self, prec, Ng, Kc, ntaps, N, Hs, Ws, bias, relu, oy, seed):
        self.prec, self.Ng, self.Kc, self.ntaps, self.N, self.Hs, self.Ws = prec, Ng, Kc, ntaps, N, Hs, Ws
        self.bias, self.relu, (self.oy_mul, self.oy0), self.seed = bias, relu, oy, seed
        rng = random.Random(seed)
        Kw = Kc + 32
        self.a_shape = (N, Hs + 2, Ws, Kw)
        sn = (Hs + 2) * Ws * Kw
        self.vspec = [(0, Hs, Ws, sn, Ws * Kw, Kw), (Ws * Kw + 32, (Hs + 1) // 2, Ws, sn, 2 * Ws * Kw, Kw)]
        pool = [(0, 1), (0, -1), (1, 0), (-1, 0), (1, 1), (-1, -1), (2, 0), (0, -4), (Hs + 2, 0), (0, Ws + 1), (-8, 3)]
        self.taps = [(0, 0, 0)] + [(rng.randrange(2), *pool[rng.randrange(len(pool))]) for _ in range(ntaps - 1)]
        if ntaps >= 3:
            self.taps[2] = (1, -(Hs + 4), 0)              # wholly outside the image
        self.osx = Ng + 16 * (1 + seed % 3)
        self.osy = Ws * self.osx + 4
        self.rows = Hs * self.oy_mul + 1
        self.osn = self.rows * self.osy
        self.pix = tc.patch_pixels(N, Hs, Ws, *tc.tg_pick_patch(Hs, Ws), DEV)

    def operands(self, cls):
        g = _gen(self.seed * 7 + CLASSES.index(cls))
        A = _operand(self.a_shape, cls, self.prec, g, zero_c0=32)
        W = _operand((self.Ng, self.ntaps * self.Kc), "ties" if cls == "ties" else "randn", self.prec, g) * 0.125
        b = _randn((self.Ng,), g) if self.bias else None
        return A, W, b

    def packed(self, W):
        """the weight operand as the kernel takes it, and the fp64 value the tensor core multiplies"""
        if self.prec == tc.TC_X3:
            hi, lo = tc.split_tf32(W)
            return torch.stack([hi, lo]).contiguous(), hi.double() + lo.double()
        if self.prec == tc.TC_BF16:
            wb = W.to(torch.bfloat16).contiguous()
            return wb, wb.double()
        return W.contiguous(), tc.tf32_trunc(W).double()

    def gathered(self, A, drop_last=False, shift=None):
        n, y, x = self.pix
        fa = A.reshape(-1).double()
        cols = []
        for t, (m, dy, dx) in enumerate(self.taps):
            off, H, W, sn, sy, sx = self.vspec[m]
            ddx = shift if t == 0 and shift else 0
            cols.append(tc.gather(fa, off, H, W, sn, sy, sx, n, y + dy, x + dx + ddx, 0, self.Kc))
        G = torch.cat(cols, 1)
        if drop_last:
            G[:, self.Kc - 32:self.Kc] = 0            # the last k-step of tap 0 (in the image)
        return G

    def quantise_a(self, G, rounding=None):
        return tc.quantise(G.float(), self.prec, rounding)

    def launch(self, A, wg, b):
        c = _capi()
        out = torch.full((self.N * self.osn + GUARD,), SENT, device=DEV)
        a = c.LfConvTcgArgs()
        for i, s in enumerate(self.vspec):
            a.a[i] = _view(A, *s)
        a.wg, a.bias, a.out = wg.data_ptr(), (b.data_ptr() if b is not None else None), out.data_ptr()
        a.osn, a.osy, a.osx, a.oy_mul, a.oy0 = self.osn, self.osy, self.osx, self.oy_mul, self.oy0
        a.N, a.Hs, a.Ws, a.Kc, a.Ng, a.ntaps = self.N, self.Hs, self.Ws, self.Kc, self.Ng, self.ntaps
        for t, (m, dy, dx) in enumerate(self.taps):
            a.map[t], a.dy[t], a.dx[t] = m, dy, dx
        a.precision, a.relu = self.prec, int(self.relu)
        c.call("lf_conv_tcg", ctypes.byref(a), c.stream_ptr())
        return out

    def out_index(self):
        n, y, x = self.pix
        base = n * self.osn + (y * self.oy_mul + self.oy0) * self.osy + x * self.osx
        return base.view(-1, 1) + torch.arange(self.Ng, device=DEV).view(1, -1)

    def reference(self, Qa, Wq, b):
        ref = Qa @ Wq.t()
        S = Qa.abs() @ Wq.abs().t()
        if b is not None:
            ref = ref + b.double()
            S = S + b.double().abs()
        if self.relu:
            ref = ref.clamp_min(0)
        return ref, S


@pytest.mark.parametrize("case", CONV, ids=_conv_id)
def test_conv_tcg_against_fp64(case):
    cc = ConvCase(*case)
    tag = _conv_id(case)
    steps = cc.ntaps * (cc.Kc // 32) + 2
    idx = cc.out_index()
    mask = torch.ones(cc.N * cc.osn + GUARD, dtype=torch.bool, device=DEV)
    mask[idx.reshape(-1)] = False
    for cls in CLASSES:
        A, W, b = cc.operands(cls)
        wg, Wq = cc.packed(W)
        G = cc.gathered(A)
        Qa = cc.quantise_a(G)
        ref, S = cc.reference(Qa, Wq, b)
        out = cc.launch(A, wg, b)
        assert bool((out[mask] == SENT).all()), "%s %s: lf_conv_tcg wrote outside its rows / channels" % (tag, cls)
        got = out[idx]
        _record("conv_tcg", cc.prec, got, ref, S, steps)
        _check_excess("%s %s" % (tag, cls), got, ref, S, steps, cc.prec)
        assert torch.equal(cc.launch(A, wg, b), out), "%s %s: two launches differ" % (tag, cls)
        if cls in ("randn", "heavy"):
            for k in (20, -20):
                s = 2.0 ** k
                o2 = cc.launch(A * s, wg, b * s if b is not None else None)
                assert torch.equal(o2[idx], got * s), "%s %s: 2^%d A does not scale the output exactly" % (tag, cls, k)
        if cls == "randn":
            # one k-step (32 channels of tap 0) dropped, or tap 0 shifted by one pixel: past the gate
            for what, Gm in (("a dropped k-step", cc.gathered(A, drop_last=True)), ("a shifted tap", cc.gathered(A, shift=1))):
                r2, _ = cc.reference(cc.quantise_a(Gm), Wq, b)
                x = _check_excess("", r2, ref, S, steps, cc.prec, must_pass=False)
                assert x > 1.0, "%s: %s stays within the gate (%.3g)" % (tag, what, x)
        if cls == "ties" and cc.prec == tc.TC_TF32:
            # activations rounded to nearest even, or weights rounded instead of truncated: past the gate
            r2, _ = cc.reference(cc.quantise_a(G, tc.tf32_rne), Wq, b)
            x = _check_excess("", r2, ref, S, steps, cc.prec, must_pass=False)
            assert x > 1.0, "%s: RNE activations stay within the gate (%.3g)" % (tag, x)
            r3, _ = cc.reference(Qa, tc.tf32_rna(W).double(), b)
            x = _check_excess("", r3, ref, S, steps, cc.prec, must_pass=False)
            assert x > 1.0, "%s: rounded weights stay within the gate (%.3g)" % (tag, x)


# =====================================================================================================================
# the weight gradients of one real training step, layer by layer
# =====================================================================================================================
def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def _wgrad_fp64(kind, args, w_shape):
    """fp64 weight gradient of the layer a wrapped call computes, from the operands f gives: (x, dy) -> dW"""
    F = torch.nn.functional
    if kind == "wgrad3":
        x, dy, _w, vertical, dil = args[:5]
        pad, dl = ((dil, 0), (dil, 1)) if vertical else ((0, dil), (1, dil))
        return lambda f: torch.nn.grad.conv2d_weight(_nchw(f(x)), w_shape, _nchw(f(dy)), 1, pad, dl)
    if kind == "conv":
        x, cin, dcat, cc = args
        return lambda f: torch.nn.grad.conv2d_weight(_nchw(f(x)), w_shape, _nchw(f(dcat[..., :cc])), 2, 1)
    if kind == "convT":
        x, ci, du, co = args

        def convT(f):
            w = torch.zeros(w_shape, dtype=torch.float64, device=DEV, requires_grad=True)
            with torch.enable_grad():        # the wrapped call runs inside the model's backward
                F.conv_transpose2d(_nchw(f(x)), w, stride=2, padding=1, output_padding=1).backward(_nchw(f(du)))
            return w.grad
        return convT
    x, dy, _w = args
    k = w_shape[-1]
    return lambda f: torch.nn.grad.conv2d_weight(_nchw(f(x)), w_shape, _nchw(f(dy)), 1, (k - 1) // 2)


@pytest.mark.parametrize("mode", ["tf32", "tf32x3", "bf16"])
def test_training_step_weight_gradients_against_fp64(mode, monkeypatch):
    """One training step of the 2-lane model with the Classification heads (--clas 1) at batch 8 and 256x512: every weight
    gradient that runs on lf_wgrad_tcg (3-tap convolutions incl. the C = 16 super-pixel layers, Down / Up stride-2
    layers, heads; in bf16 mode the residual blocks' bf16-stored inputs, i.e. the bf16 A views) against the fp64 weight
    gradient of the quantised operands it received, under the per-entry gate (S from the same gradient of |x|, |dy|)."""
    import bench
    from lanedetection_end2end_b200 import ops_heads, ops_net as o
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    import contextlib
    import io

    o.set_conv_mode(mode)
    prec = o.wgrad_precision()
    launches, pending, failures = [], [], []
    real_run = o.run_wgrad_tcg

    def run_wgrad_tcg(av, bv, blocks, N, Hs, Ws, *rest, **kw):
        partial, nctas = real_run(av, bv, blocks, N, Hs, Ws, *rest, **kw)
        launches.append((N * Hs * Ws // 32, nctas, kw.get("a_dtype", 0)))
        return partial, nctas

    def wrap(kind, fn):
        def wrapped(*args, **kw):
            launches.clear()
            res = fn(*args, **kw)
            dw = res[0] if kind == "wgrad3" else res
            if launches:
                # steps: the patches of the busiest CTA, its hand-over, the partials reduced, and up to 8 adds when the
                # super-pixel gradient is folded back onto the C = 16 weights
                steps = max((t + n - 1) // n + 1 + n for t, n, _ in launches) + 8
                ref_of = _wgrad_fp64(kind, args, tuple(dw.shape))
                q = lambda t: tc.quantise(t.float(), prec)
                ref = ref_of(q)
                S = ref_of(lambda t: q(t).abs())
                name = "%s %s %s" % (kind, tuple(dw.shape), "bf16-A" if any(a for _, _, a in launches) else "")
                # compared after the backward: the 3-tap reductions are deferred to the end of the block's backward
                pending.append((name, dw, ref, S, steps))
            return res
        return wrapped

    monkeypatch.setattr(o, "run_wgrad_tcg", run_wgrad_tcg)
    monkeypatch.setattr(o, "wgrad3", wrap("wgrad3", o.wgrad3))
    monkeypatch.setattr(o, "wgrad_tcg_conv", wrap("conv", o.wgrad_tcg_conv))
    monkeypatch.setattr(o, "wgrad_tcg_convT", wrap("convT", o.wgrad_tcg_convT))
    monkeypatch.setattr(ops_heads, "conv_wgrad", wrap("head", ops_heads.conv_wgrad))

    cfg = dict(name="2lane_clas_b8", nclasses=2, order=2, mask=0.3, resize=256, batch=8, clas=True)
    args = bench.build_args(cfg)
    torch.manual_seed(0)
    model = Net(args)
    with contextlib.redirect_stdout(io.StringIO()):
        define_init_weights(model, "kaiming")
    model = model.cuda().train()
    crit = backprojection_loss(args)
    x, xgt, valid = (t.cuda() for t in bench.host_batch(cfg, 1234, pinned=False))
    bce = torch.nn.BCEWithLogitsLoss()
    gt_cls = torch.ones(8, 4, device=DEV)
    gt_hor = torch.zeros(8, 256, device=DEV)
    gt_hor[:, 80] = 1.0
    out = model(x, torch.zeros(8, 4), True)
    loss = sum(crit(out[l], xgt[:, l], valid[:, l])[0] for l in range(2)) / 2
    loss = loss + (bce(out[6], gt_cls) + bce(out[7], gt_hor)).double()
    loss.backward()
    torch.cuda.synchronize()
    for name, dw, ref, S, steps in pending:
        _record("training step", prec, dw.reshape(-1), ref.reshape(-1), S.reshape(-1), steps)
        x = tc.gate_excess(dw, ref, S, steps, prec)
        if x > 1.0:
            failures.append("%s: %.3g x the gate" % (name, x))
    checked = [p[0] for p in pending]
    kinds = {c.split()[0] for c in checked}
    assert kinds == {"wgrad3", "conv", "convT", "head"}, checked
    if mode == "bf16":
        assert any("bf16-A" in c for c in checked), checked
    assert not failures, failures
