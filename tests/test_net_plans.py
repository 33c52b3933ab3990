"""CPU check of the host-side geometry (net_plans.py + the weight packers in ops_net.py):
a torch emulation of the generic conv / wgrad kernels' contract (LfConvArgs / LfWgradArgs in
include/lanefit_b200.h) fed with the SAME plans and packed weights the CUDA launches get, compared
against torch's own convolutions and autograd."""
import pytest
import torch
import torch.nn.functional as F

from lanedetection_end2end_b200 import net_plans as plans
from lanedetection_end2end_b200 import ops_net as ops
from tcg_contract import emulate_conv_tcg as _emulate_conv_tcg
from tcg_contract import emulate_wgrad_reduce as _emulate_wgrad_reduce
from tcg_contract import emulate_wgrad_tcg as _emulate_wgrad_tcg

torch.manual_seed(0)
DT = torch.float64


def emulate_conv(phases, x, wmat, cin, Hout, Wout, cout):
    """x [N,Hin,Win,Cx] NHWC, wmat [T,cin,CoPad] -> out [N,Hout,Wout,cout]."""
    N, Hin, Win, _ = x.shape
    out = torch.zeros(N, Hout, Wout, cout, dtype=x.dtype)
    for ph in phases:
        for j in range(ph["Hs"]):
            for i in range(ph["Ws"]):
                acc = torch.zeros(N, cout, dtype=x.dtype)
                for dy, dx, slot in ph["taps"]:
                    iy, ix = j * ph["isy"] + dy, i * ph["isx"] + dx
                    if 0 <= iy < Hin and 0 <= ix < Win:
                        acc += x[:, iy, ix, :cin] @ wmat[slot, :, :cout]
                out[:, j * ph["osy"] + ph["oy0"], i * ph["osx"] + ph["ox0"]] = acc
    return out


def emulate_wgrad(plan, P, cp, Q, cq, q_coff):
    """-> dW [T, cp, cq]."""
    N, Hp, Wp, _ = P.shape
    _, Hq, Wq, _ = Q.shape
    T = len(plan["ptaps"])
    dW = torch.zeros(T, cp, cq, dtype=P.dtype)
    for t in range(T):
        for j in range(plan["Hs"]):
            for i in range(plan["Ws"]):
                py, px = j * plan["psy"] + plan["ptaps"][t][0], i * plan["psx"] + plan["ptaps"][t][1]
                qy, qx = j * plan["qsy"] + plan["qtaps"][t][0], i * plan["qsx"] + plan["qtaps"][t][1]
                if 0 <= py < Hp and 0 <= px < Wp and 0 <= qy < Hq and 0 <= qx < Wq:
                    dW[t] += P[:, py, px, :cp].t() @ Q[:, qy, qx, q_coff:q_coff + cq]
    return dW


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("kh,kw,dil", [(3, 1, 1), (1, 3, 1), (3, 1, 2), (1, 3, 4), (3, 1, 8)])
def test_factorised_conv_fwd_dgrad_wgrad(kh, kw, dil):
    N, C, H, W = 2, 8, 9, 11
    ph, pw = (dil, 0) if kh == 3 else (0, dil)
    dh, dw_ = (dil, 1) if kh == 3 else (1, dil)
    x = torch.randn(N, C, H, W, dtype=DT, requires_grad=True)
    w = torch.randn(C, C, kh, kw, dtype=DT, requires_grad=True)
    y = F.conv2d(x, w, None, 1, (ph, pw), (dh, dw_))
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, w), gy)
    phases, (Ho, Wo) = plans.conv_fwd_plan(H, W, kh, kw, 1, ph, pw, dh, dw_)
    got = emulate_conv(phases, nhwc(x.detach()), ops.pack_conv_fwd(w.detach()), C, Ho, Wo, C)
    torch.testing.assert_close(nchw(got), y.detach())
    pd, _ = plans.conv_dgrad_plan_s1(H, W, kh, kw, ph, pw, dh, dw_)
    got = emulate_conv(pd, nhwc(gy), ops.pack_conv_dgrad(w.detach()), C, H, W, C)
    torch.testing.assert_close(nchw(got), gx)
    wp = plans.conv_wgrad_plan(H, W, kh, kw, 1, ph, pw, dh, dw_)
    dW = emulate_wgrad(wp, nhwc(x.detach()), C, nhwc(gy), C, 0)          # [T, ci, co]
    torch.testing.assert_close(dW.permute(2, 1, 0).reshape(C, C, kh, kw), gw)


@pytest.mark.parametrize("cin,cout", [(3, 16), (8, 24)])
def test_downsampler_conv(cin, cout):
    N, H, W = 2, 10, 12
    cc = cout - cin
    x = torch.randn(N, cin, H, W, dtype=DT, requires_grad=True)
    w = torch.randn(cc, cin, 3, 3, dtype=DT, requires_grad=True)
    y = F.conv2d(x, w, None, 2, 1)
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, w), gy)
    cin_g = plans.pad_to(cin, 4)
    xp = F.pad(nhwc(x.detach()), (0, cin_g - cin))
    phases, (Ho, Wo) = plans.conv_fwd_plan(H, W, 3, 3, 2, 1, 1, 1, 1)
    got = emulate_conv(phases, xp, ops.pack_conv_fwd(w.detach(), cin_g), cin_g, Ho, Wo, cc)
    torch.testing.assert_close(nchw(got), y.detach())
    # input gradient = transposed-conv gather over the output gradient (4 phases)
    pd, _ = plans.transposed_gather_plan(Ho, Wo, H, W, 3, 1)
    wd = ops.pack_conv_dgrad(w.detach())
    got = emulate_conv(pd, nhwc(gy), wd, cc, H, W, cin)
    torch.testing.assert_close(nchw(got), gx)
    wp = plans.conv_wgrad_plan(H, W, 3, 3, 2, 1, 1, 1, 1)
    dW = emulate_wgrad(wp, xp, cin_g, nhwc(gy), cc, 0)[:, :cin]
    torch.testing.assert_close(dW.permute(2, 1, 0).reshape(cc, cin, 3, 3), gw)


def test_upsampler_convT():
    N, ci, co, H, W = 2, 8, 4, 5, 6
    x = torch.randn(N, ci, H, W, dtype=DT, requires_grad=True)
    w = torch.randn(ci, co, 3, 3, dtype=DT, requires_grad=True)
    y = F.conv_transpose2d(x, w, None, 2, 1, 1)
    assert y.shape[2:] == (2 * H, 2 * W)
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, w), gy)
    phases, (Ho, Wo) = plans.transposed_gather_plan(H, W, 2 * H, 2 * W, 3, 1)
    got = emulate_conv(phases, nhwc(x.detach()), ops.pack_convT_fwd(w.detach()), ci, Ho, Wo, co)
    torch.testing.assert_close(nchw(got), y.detach())
    pd, _ = plans.convT_dgrad_plan(2 * H, 2 * W, H, W, 3, 1)
    got = emulate_conv(pd, nhwc(gy), ops.pack_convT_dgrad(w.detach()), co, H, W, ci)
    torch.testing.assert_close(nchw(got), gx)
    wp = plans.convT_wgrad_plan(H, W, 3, 1)
    dW = emulate_wgrad(wp, nhwc(x.detach()), ci, nhwc(gy), co, 0)          # [T, ci, co]
    torch.testing.assert_close(dW.permute(1, 2, 0).reshape(ci, co, 3, 3), gw)


def test_wgrad_destination_strides_match_weight_layouts():
    # (st, sp, sq) used by ops_net for Conv2d [Co,Ci,kh,kw] and ConvTranspose2d [Ci,Co,kh,kw]
    Co, Ci, kh, kw = 5, 3, 3, 1
    w = torch.arange(Co * Ci * kh * kw).reshape(Co, Ci, kh, kw)
    st, sp, sq = 1, kh * kw, Ci * kh * kw
    for t in range(kh * kw):
        for ci in range(Ci):
            for co in range(Co):
                assert w.reshape(-1)[t * st + ci * sp + co * sq] == w[co, ci, t // kw, t % kw]
    wT = torch.arange(Ci * Co * 9).reshape(Ci, Co, 3, 3)
    st, sp, sq = 1, Co * 9, 9
    for t in range(9):
        for ci in range(Ci):
            for co in range(Co):
                assert wT.reshape(-1)[t * st + ci * sp + co * sq] == wT[ci, co, t // 3, t % 3]


@pytest.mark.parametrize("vertical,dil", [(True, 1), (False, 1), (True, 4), (False, 16)])
def test_tc_kernel_contract_fwd_and_dgrad(vertical, dil):
    """Contract of lf_conv1d_tc (LfConvTcArgs): out = sum_t in[y+dy_t, x+dx_t] @ wpack[:, t*C:(t+1)*C]^T with the
    taps / packings ops_net.conv3 builds, vs torch conv2d and its input gradient."""
    N, C, H, W = 2, 8, 9, 20
    kh, kw = (3, 1) if vertical else (1, 3)
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    x = torch.randn(N, C, H, W, dtype=DT, requires_grad=True)
    w = torch.randn(C, C, kh, kw, dtype=DT)
    y = F.conv2d(x, w, None, 1, pad, dl)
    gy = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, x, gy)

    def emulate(inp, wpack, sgn):
        out = torch.zeros(N, H, W, C, dtype=DT)
        for t in range(3):
            dy, dx = ((sgn * (t - 1) * dil, 0) if vertical else (0, sgn * (t - 1) * dil))
            for yy in range(H):
                for xx in range(W):
                    iy, ix = yy + dy, xx + dx
                    if 0 <= iy < H and 0 <= ix < W:
                        out[:, yy, xx] += inp[:, iy, ix] @ wpack[:, t * C:(t + 1) * C].t()
        return out

    torch.testing.assert_close(nchw(emulate(nhwc(x.detach()), ops.pack_tc_fwd(w), 1)), y.detach())
    torch.testing.assert_close(nchw(emulate(nhwc(gy), ops.pack_tc_dgrad(w), -1)), gx)


@pytest.mark.parametrize("vertical", [True, False])
@pytest.mark.parametrize("transposed", [False, True])
def test_super_pixel_packing_of_16_channel_convs(vertical, transposed):
    """ops_net.pack_tc_super: a 3-tap 16->16 conv on [N,H,W,16] == the lf_conv1d_tc contract on the
    [N,H,W/4,64] view with the packed 64x(3*64) operand; and unpack_wgrad_super inverts the weight-gradient."""
    N, C, H, W = 2, 16, 6, 16
    kh, kw = (3, 1) if vertical else (1, 3)
    pad = (1, 0) if vertical else (0, 1)
    x = torch.randn(N, C, H, W, dtype=DT, requires_grad=True)
    w = torch.randn(C, C, kh, kw, dtype=DT, requires_grad=True)
    y = F.conv2d(x, w, None, 1, pad)
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, w), gy)
    inp, ref = (nhwc(gy), gx) if transposed else (nhwc(x.detach()), y.detach())
    xs = inp.reshape(N, H, W // 4, 64)
    wp = ops.pack_tc_super(w.detach(), vertical, transposed)
    sgn = -1 if transposed else 1
    out = torch.zeros(N, H, W // 4, 64, dtype=DT)
    for t in range(3):
        dy, dx = ((sgn * (t - 1), 0) if vertical else (0, sgn * (t - 1)))
        for yy in range(H):
            for xx in range(W // 4):
                iy, ix = yy + dy, xx + dx
                if 0 <= iy < H and 0 <= ix < W // 4:
                    out[:, yy, xx] += xs[:, iy, ix] @ wp[:, t * 64:(t + 1) * 64].t()
    torch.testing.assert_close(nchw(out.reshape(N, H, W, C)), ref)
    if not transposed:
        # weight gradient of the super conv (Conv2d layout [co_s][ci_s][T]) -> original
        xsup = xs.permute(0, 3, 1, 2).contiguous().requires_grad_(False)
        wsup = torch.zeros(64, 64, kh, kw, dtype=DT, requires_grad=True)
        ysup = F.conv2d(xsup, wsup, None, 1, pad)
        (gws,) = torch.autograd.grad(ysup, wsup, nhwc(gy).reshape(N, H, W // 4, 64).permute(0, 3, 1, 2))
        got = ops.unpack_wgrad_super(gws.reshape(64, 64, 3), vertical).reshape(C, C, kh, kw)
        torch.testing.assert_close(got, gw)


def test_weight_pack_gather_tables_reproduce_every_packer():
    """ops_net.WeightPackCache packs all operands with one gather kernel; its index tables are derived by running
    each packer on element numbers.  Check table-gather == packer on random weights for every packer / layer shape."""
    from lanedetection_end2end_b200 import ops_net as o
    g = torch.Generator().manual_seed(5)
    cases = [
        (o.pack_tc_fwd, (64, 64, 3, 1)), (o.pack_tc_fwd, (128, 128, 1, 3)), (o.pack_tc_dgrad, (64, 64, 1, 3)),
        (o.pack_tc_dgrad, (128, 128, 3, 1)),
        (o.pack_conv_fwd, (16, 16, 3, 1)), (o.pack_conv_dgrad, (16, 16, 1, 3)), (o.pack_conv_fwd, (48, 16, 3, 3)),
        (lambda t: o.pack_conv_fwd(t, 4), (13, 3, 3, 3)), (o.pack_conv_dgrad, (64, 64, 3, 3)),
        (o.pack_convT_fwd, (128, 64, 3, 3)), (o.pack_convT_dgrad, (64, 16, 3, 3)),
    ]
    for vertical in (True, False):
        for transposed in (True, False):
            cases.append((lambda t, v=vertical, tr=transposed: o.pack_tc_super(t, v, tr),
                          (16, 16, 3, 1) if vertical else (16, 16, 1, 3)))
    for fn, shape in cases:
        w = torch.randn(*shape, generator=g)
        idx = o.pack_gather_table(fn, shape)
        ref = fn(w)
        assert idx.shape == ref.shape
        src = torch.cat([w.reshape(-1), w.new_zeros(1)])
        got = src[idx.to(torch.int64).clamp(min=-1)]          # -1 wraps to the appended zero
        assert torch.equal(got, ref), (fn, shape)


def test_tcg_pair_pixel_forms_match_torch_convs(monkeypatch):
    """The four layer forms served by lf_conv_tcg (Down forward / input gradient, Up forward / input gradient) are
    re-expressed as unit-stride gathers over pair-pixel / row-parity views.  Run the host code on CPU with the kernel
    replaced by a literal restatement of its contract and compare with torch's own stride-2 convolutions."""
    import torch.nn.functional as F
    from lanedetection_end2end_b200 import ops_net as o, _capi
    live = []
    monkeypatch.setattr(o, "_stream", lambda: None)
    monkeypatch.setattr(_capi, "call", lambda name, ref, *rest, **kw: _emulate_conv_tcg(ref._obj, live))
    g = torch.Generator().manual_seed(7)
    # ---- Conv2d 3x3 stride 2 (DownsamplerBlock: 16 -> 48 into a 64-channel concat buffer) and its input gradient
    for (C, O, tot, H, W) in [(16, 48, 64, 16, 32), (64, 64, 128, 8, 32)]:
        N = 2
        x = torch.randn(N, H, W, C, generator=g)
        w = torch.randn(O, C, 3, 3, generator=g) * 0.1
        b = torch.randn(O, generator=g)
        cat = torch.full((N, H // 2, W // 2, tot), 7.0)
        wg = o.pack_tcg_s2conv(w)
        bp = torch.cat([b, torch.zeros(wg.shape[0] - O)])
        live[:] = [x, wg, bp, cat]
        o.run_tcg_s2conv(x, wg, O, cat, bias=bp)
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1).permute(0, 2, 3, 1)
        assert torch.allclose(cat[..., :O].double(), ref, atol=1e-5), (C, O)
        assert bool((cat[..., wg.shape[0]:] == 7.0).all())             # channels beyond pad16(O) untouched
        # input gradient of that conv = transposed conv of the output gradient with the same weight
        dcat = torch.randn(N, H // 2, W // 2, tot, generator=g)
        kc = ((O + 31) // 32) * 32
        wgs = (o.pack_tcg_s2convT(w, 0, kc), o.pack_tcg_s2convT(w, 1, kc))
        dx = torch.full((N, H, W, C), 3.0)
        live[:] = [dcat, wgs[0], wgs[1], dx]
        o.run_tcg_s2convT(dcat, O, wgs, C, dx)
        ref = F.conv_transpose2d(dcat[..., :O].permute(0, 3, 1, 2).double(), w.double(), stride=2, padding=1,
                                 output_padding=1).permute(0, 2, 3, 1)
        assert torch.allclose(dx.double(), ref, atol=1e-5), (C, O)
    # ---- ConvTranspose2d 3x3 stride 2 (UpsamplerBlock) and its input gradient
    for (I, O, H, W) in [(128, 64, 8, 16), (64, 16, 8, 32)]:
        N = 2
        x = torch.randn(N, H, W, I, generator=g)
        w = torch.randn(I, O, 3, 3, generator=g) * 0.1
        b = torch.randn(O, generator=g)
        wgs = (o.pack_tcg_s2convT(w, 0, I), o.pack_tcg_s2convT(w, 1, I))
        u = torch.zeros(N, 2 * H, 2 * W, O)
        b2 = b.repeat(2)
        live[:] = [x, wgs[0], wgs[1], b2, u]
        o.run_tcg_s2convT(x, I, wgs, O, u, bias2=b2)
        ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=2, padding=1,
                                 output_padding=1).permute(0, 2, 3, 1)
        assert torch.allclose(u.double(), ref, atol=1e-5), (I, O)
        du = torch.randn(N, 2 * H, 2 * W, O, generator=g)
        wg = o.pack_tcg_s2conv(w)                                      # [I][6*2*O]: out = I, in = O
        dx = torch.zeros(N, H, W, I)
        live[:] = [du, wg, dx]
        o.run_tcg_s2conv(du, wg, I, dx)
        xin = x.permute(0, 3, 1, 2).double().requires_grad_(True)
        F.conv_transpose2d(xin, w.double(), stride=2, padding=1, output_padding=1).backward(du.permute(0, 3, 1, 2).double())
        assert torch.allclose(dx.double(), xin.grad.permute(0, 2, 3, 1), atol=1e-5), (I, O)


def test_tcg_weight_gradients_through_one_launcher_match_torch(monkeypatch):
    """wgrad_tcg_conv / wgrad_tcg_convT (pair-pixel taps, block lists, split launches, partial reduction, final gather)
    against autograd's weight gradients of the stride-2 Conv2d / ConvTranspose2d, with the kernel replaced by a literal
    restatement of its contract."""
    import ctypes
    import torch.nn.functional as F
    from lanedetection_end2end_b200 import ops_net as o, _capi
    live = []

    class FakeLib:
        @staticmethod
        def lf_wgrad_tcg_ctas(N, Hs, Ws, Ka, Nn, nblocks, min_patches):
            assert min_patches == 4
            return 3 if ((nblocks + 3) // 4) * Nn <= 512 else 0

    def fake_call(name, *args, **kw):
        if name == "lf_wgrad_tcg":
            _emulate_wgrad_tcg(args[0]._obj, live)
        elif name == "lf_wgrad_reduce":
            _emulate_wgrad_reduce(args, live)
        else:
            raise AssertionError(name)

    real_empty = torch.empty

    def tracking_empty(*a_, **kw):
        t = real_empty(*a_, **kw)
        live.append(t)
        return t

    monkeypatch.setattr(o, "_stream", lambda: None)
    monkeypatch.setattr(o, "_lib", lambda: FakeLib)
    monkeypatch.setattr(o, "ptr", lambda t: t.data_ptr() if t is not None else None)
    monkeypatch.setattr(_capi, "call", fake_call)
    monkeypatch.setattr(o, "CONV_MODE", "tf32")
    monkeypatch.setattr(torch, "empty", tracking_empty)
    g = torch.Generator().manual_seed(11)
    for (C, O, tot, H, W) in [(16, 48, 64, 16, 32), (64, 64, 128, 8, 16)]:
        N = 2
        x = torch.randn(N, H, W, C, generator=g)
        dcat = torch.randn(N, H // 2, W // 2, tot, generator=g)
        live[:] = [x, dcat]
        assert o.wgrad_tcg_ok(x, C, dcat, ((O + 31) // 32) * 32)
        dw = o.wgrad_tcg_conv(x, C, dcat, O)
        w = torch.zeros(O, C, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv2d(x.permute(0, 3, 1, 2).double(), w, stride=2, padding=1).backward(dcat[..., :O].permute(0, 3, 1, 2).double())
        assert torch.allclose(dw.double(), w.grad, atol=1e-4, rtol=1e-5), (C, O)
    for (I, O, H, W) in [(128, 64, 4, 8), (64, 16, 8, 16)]:
        N = 2
        x = torch.randn(N, H, W, I, generator=g)
        du = torch.randn(N, 2 * H, 2 * W, O, generator=g)
        live[:] = [x, du]
        assert o.wgrad_tcg_ok(du, O, x, I)
        dw = o.wgrad_tcg_convT(x, I, du, O)
        w = torch.zeros(I, O, 3, 3, dtype=torch.float64, requires_grad=True)
        F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w, stride=2, padding=1, output_padding=1).backward(
            du.permute(0, 3, 1, 2).double())
        assert torch.allclose(dw.double(), w.grad, atol=1e-4, rtol=1e-5), (I, O)


def test_heads_dense_conv_and_wgrad_tcg_forms_match_torch(monkeypatch):
    """ops_heads: the Classification heads' 1x1 / 3x3 stride-1 convolutions, their input gradients and weight gradients are
    expressed as run-time-tap launches of lf_conv_tcg / lf_wgrad_tcg (tap lists, packed operands, split launches, the final
    view / permute).  Run that host code on the CPU with the two kernels replaced by literal restatements of their contracts
    and compare with torch's own convolutions and autograd."""
    import torch.nn.functional as F
    from lanedetection_end2end_b200 import ops_net as o, ops_heads as hd, _capi
    live = []

    class FakeLib:
        @staticmethod
        def lf_conv_tcg_supported(N, H, W, Kc, Ng):
            return 1

        @staticmethod
        def lf_wgrad_tcg_ctas(N, Hs, Ws, Ka, Nn, nblocks, min_patches):
            assert min_patches == 4
            return 3 if ((nblocks + 3) // 4) * Nn <= 512 else 0

    def fake_call(name, *args, **kw):
        if name == "lf_conv_tcg":
            _emulate_conv_tcg(args[0]._obj, live)
        elif name == "lf_wgrad_tcg":
            _emulate_wgrad_tcg(args[0]._obj, live)
        elif name == "lf_wgrad_reduce":
            _emulate_wgrad_reduce(args, live)
        else:
            raise AssertionError(name)

    real_empty = torch.empty

    def tracking_empty(*a_, **kw):
        t = real_empty(*a_, **kw)
        live.append(t)
        return t

    monkeypatch.setattr(o, "_stream", lambda: None)
    monkeypatch.setattr(o, "_lib", lambda: FakeLib)
    monkeypatch.setattr(_capi, "lib", lambda: FakeLib)
    monkeypatch.setattr(o, "ptr", lambda t: t.data_ptr() if t is not None else None)
    monkeypatch.setattr(_capi, "call", fake_call)
    monkeypatch.setattr(o, "CONV_MODE", "tf32")            # single operands (the hi/lo split is a pure re-encoding of the same matrix)
    monkeypatch.setattr(torch, "empty", tracking_empty)
    g = torch.Generator().manual_seed(3)
    for (Ci, Co, k, H, W) in [(128, 128, 1, 4, 32), (128, 64, 3, 8, 16), (64, 64, 3, 4, 32)]:
        N = 2
        x = torch.randn(N, H, W, Ci, generator=g)
        w = torch.randn(Co, Ci, k, k, generator=g) * 0.1
        b = torch.randn(Co, generator=g)
        live[:] = [x, b]
        monkeypatch.setattr(o, "packed", lambda w_, kind, fn, split=False: _keep(live, fn(w_)))
        y = hd.conv_fwd(x, w, b)
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=(k - 1) // 2).permute(0, 2, 3, 1)
        assert torch.allclose(y.double(), ref, atol=1e-5), ("fwd", Ci, Co, k)
        dy = torch.randn(N, H, W, Co, generator=g)
        live.append(dy)
        dx = hd.conv_dgrad(dy, w)
        xin = x.permute(0, 3, 1, 2).double().requires_grad_(True)
        wd = w.double().requires_grad_(True)
        F.conv2d(xin, wd, padding=(k - 1) // 2).backward(dy.permute(0, 3, 1, 2).double())
        assert torch.allclose(dx.double(), xin.grad.permute(0, 2, 3, 1), atol=1e-5), ("dgrad", Ci, Co, k)
        dw = hd.conv_wgrad(x, dy, w)
        assert dw.shape == w.shape and torch.allclose(dw.double(), wd.grad, atol=1e-4, rtol=1e-5), ("wgrad", Ci, Co, k)


def _keep(live, t):
    """Register a freshly packed operand so that the emulators can resolve its pointer."""
    live.append(t)
    return t


def test_wgrad3_matches_torch(monkeypatch):
    """ops_net.wgrad3 on its tensor-core route (the 3-tap block table, the super-pixel view of C = 16 and its unpacking,
    the reduction into the [Co,Ci,3] weight layout, a bf16 A view) against fp64 autograd, with lf_wgrad_tcg replaced by a
    literal restatement of its contract; per mode also the launch's precision, its trace label and the split policy (at
    least 8 patches per CTA for the 3xTF32 weight gradients, 4 otherwise)."""
    import torch.nn.functional as F
    from lanedetection_end2end_b200 import ops_net as o, _capi
    live, launches = [], []

    class FakeLib:
        @staticmethod
        def lf_wgrad_tcg_ctas(N, Hs, Ws, Ka, Nn, nblocks, min_patches):
            launches.append(("ctas", min_patches))
            return 3 if ((nblocks + 3) // 4) * Nn <= 512 else 0

        @staticmethod
        def lf_conv1d_tc_supported(N, H, W, C):
            return 1

        @staticmethod
        def lf_conv1d_tc_x3_rows(N, H, W, C, vertical, dil):
            return 1

    def fake_call(name, *args, **kw):
        if name == "lf_wgrad_tcg":
            launches.append((kw["label"], args[0]._obj.precision))
            _emulate_wgrad_tcg(args[0]._obj, live)
        elif name == "lf_wgrad_reduce":
            _emulate_wgrad_reduce(args, live)
        else:
            raise AssertionError(name)

    def tracking(fn):
        def alloc(*a_, **kw):
            t = fn(*a_, **kw)
            live.append(t)
            return t
        return alloc

    monkeypatch.setattr(o, "_stream", lambda: None)
    monkeypatch.setattr(o, "_lib", lambda: FakeLib)
    monkeypatch.setattr(o, "ptr", lambda t: t.data_ptr() if t is not None else None)
    monkeypatch.setattr(_capi, "call", fake_call)
    monkeypatch.setattr(torch, "empty", tracking(torch.empty))
    monkeypatch.setattr(torch, "empty_like", tracking(torch.empty_like))
    g = torch.Generator().manual_seed(5)
    # (mode, single-pass weight gradients, layer input dtype) -> (precision, trace label, fewest patches per CTA)
    modes = {("tf32", False, torch.float32): (0, "lf_wgrad3_tc", 4),
             ("tf32x3", False, torch.float32): (1, "lf_wgrad3_tc_x3", 8),
             ("tf32x3", True, torch.float32): (0, "lf_wgrad3_tc", 4),
             ("bf16", False, torch.float32): (2, "lf_wgrad3_tc_bf16", 4),
             ("bf16", False, torch.bfloat16): (2, "lf_wgrad3_tc_bf16a", 4)}
    for (mode, single, dtype), (prec, label, min_patches) in modes.items():
        monkeypatch.setattr(o, "CONV_MODE", mode)
        monkeypatch.setattr(o, "WGRAD_SINGLE_PASS", single)
        for (C, vertical, dil) in [(64, True, 1), (64, False, 2), (128, True, 2), (128, False, 1), (16, True, 1), (16, False, 1)]:
            N, H, W = 2, 8, 16
            x = torch.randn(N, H, W, C, generator=g).to(dtype)
            dy = torch.randn(N, H, W, C, generator=g)
            kh, kw = (3, 1) if vertical else (1, 3)
            w = torch.zeros(C, C, kh, kw)
            live[:] = [x, dy]
            launches.clear()
            dw, db = o.wgrad3(x, dy, w, vertical, dil, bias_grad="skip")
            assert db is None and launches[-1] == (label, prec), (mode, C, launches)
            assert {m for kind, m in launches if kind == "ctas"} == {min_patches}, (mode, C, launches)
            wd = torch.zeros(C, C, kh, kw, dtype=torch.float64, requires_grad=True)
            pad, dl = ((dil, 0), (dil, 1)) if vertical else ((0, dil), (1, dil))
            F.conv2d(x.double().permute(0, 3, 1, 2), wd, None, 1, pad, dl).backward(dy.double().permute(0, 3, 1, 2))
            assert dw.shape == w.shape and torch.allclose(dw.double(), wd.grad, atol=1e-4, rtol=1e-5), (mode, dtype, C,
                                                                                                           vertical, dil)
