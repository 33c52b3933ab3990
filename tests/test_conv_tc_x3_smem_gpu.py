"""3xTF32 3-tap convolution (csrc/conv_tc.cu, lf_conv1d_tc_x3) at every layer shape of configs 2/3 (256x512) and 4
(320x640), both tap orders, every epilogue, against fp64.

The kernel takes A from shared memory: each slab is split once into hi (in place) and lo (a separate buffer), and the
lo buffer sits where shared memory allows -- two buffers after the TMA ring, one, or one over the staging tile (reaching
back before it for the 320x640 slabs of 48 and 80 KB).  The shape list covers each of those plans; the batch gives
every persistent CTA several tiles, so the buffers are reused across tiles."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

N = 6
SHAPES = [  # C, H, W, vertical, dil: lo buffer plan (weights resident for C = 64, streamed for C = 128)
    (64, 64, 128, True, 1), (64, 64, 128, False, 1),          # two lo buffers, three stages
    (64, 128, 64, True, 1), (64, 128, 64, False, 1),          # C = 16 decoder layers as 4-pixel super-pixels
    (64, 80, 160, True, 1), (64, 80, 160, False, 1),
    (64, 160, 80, True, 1), (64, 160, 80, False, 1),
] + [(128, 32, 64, v, d) for d in (1, 2, 4, 8, 16) for v in (True, False)] + [  # 32x64 v8 / h16: one; v16: staging
    (128, 40, 80, v, d) for d in (1, 2, 4, 8, 16) for v in (True, False)]      # 40x80 v8, h8, v16, h16: staging (+ before)

EPILOGUES = ["bias_relu", "colsum", "bn_stats", "mask", "affine_mask", "add", "add_mask"]


def _id(s):
    C, H, W, v, d = s
    return "C%d_%dx%d_%s_d%d" % (C, H, W, "v" if v else "h", d)


@pytest.mark.parametrize("dgrad", [False, True], ids=["fwd", "dgrad"])
@pytest.mark.parametrize("C,H,W,vertical,dil", SHAPES, ids=[_id(s) for s in SHAPES])
def test_x3_every_config_shape_and_epilogue_vs_fp64(C, H, W, vertical, dil, dgrad):
    from lanedetection_end2end_b200 import ops_net as o
    g = torch.Generator().manual_seed(C * 100 + H + 7 * dil + int(vertical) + 2 * int(dgrad))
    x = torch.randn(N, H, W, C, generator=g).cuda()
    kh, kw = (3, 1) if vertical else (1, 3)
    w = (torch.randn(C, C, kh, kw, generator=g) / (3 * C) ** 0.5).cuda()
    b = torch.randn(C, generator=g).cuda()
    mask, add, addm, xbn = (torch.randn(N, H, W, C, generator=g).cuda() for _ in range(4))
    scale, shift = torch.randn(C, generator=g).cuda(), torch.randn(C, generator=g).cuda()

    o.set_conv_mode("tf32x3")
    try:
        rows = o.tc_rows(x, vertical, dil)
        assert rows > 0, "lf_conv1d_tc_x3_rows is 0: the layer would fall back to the FFMA kernels"
        sgn = -1 if dgrad else 1
        taps = [((sgn * (k - 1) * dil, 0) if vertical else (0, sgn * (k - 1) * dil)) for k in range(3)]
        wp = o.tc_operand(o.pack_tc_dgrad(w) if dgrad else o.pack_tc_fwd(w))

        def run(**epi):
            return o.run_conv_tc(taps, x, wp, torch.empty_like(x), **epi)

        cs = torch.empty(C, device="cuda")
        sp_stats = torch.zeros(rows * 2 * C, dtype=torch.float64, device="cuda")
        sp_aff = torch.zeros(rows * 2 * C, dtype=torch.float64, device="cuda")
        got = {
            "bias_relu": run(bias=b, relu=True),
            "colsum": run(colsum=cs),
            "bn_stats": run(bias=b, stats_partial=sp_stats),
            "mask": run(mask_src=mask),
            "affine_mask": run(mask_src=xbn, mask_affine=(scale, shift), stats_partial=sp_aff),
            "add": run(add_src=add),
            "add_mask": run(add_src=add, add_mask=addm),
        }
        torch.cuda.synchronize()
    finally:
        o.set_conv_mode("fp32")

    # fp64 reference of the bare convolution (forward) or of its input gradient (transposed taps)
    xd, wd = x.double().permute(0, 3, 1, 2), w.double()
    pad = (dil, 0) if vertical else (0, dil)
    dl = (dil, 1) if vertical else (1, dil)
    z = (F.conv_transpose2d(xd, wd, padding=pad, dilation=dl) if dgrad else F.conv2d(xd, wd, None, 1, pad, dl))
    z = z.permute(0, 2, 3, 1)
    bd = b.double()
    # x * scale is exact in fp64, so this sign is the sign of the kernel's fp32 fma(x, scale, shift)
    aff = xbn.double() * scale.double() + shift.double()
    want = {
        "bias_relu": torch.relu(z + bd),
        "colsum": z,
        "bn_stats": z + bd,
        "mask": z * (mask > 0),
        "affine_mask": z * (aff > 0),
        "add": z + add.double(),
        "add_mask": z + add.double() * (addm > 0),
    }
    assert set(got) == set(EPILOGUES)
    for name in EPILOGUES:
        ref = want[name]
        err = float((got[name].double() - ref).abs().max()) / float(ref.abs().max())
        assert err <= 3e-6, (name, err)

    # fused sums against fp64 sums of the kernel's own output (the fp32 partial sums round like an fp32 reduction)
    def close(a, r, what):
        assert float((a - r).abs().max()) <= 1e-4 * float(r.abs().max()), what
    close(cs.double(), got["colsum"].double().sum(dim=(0, 1, 2)), "colsum")
    st = sp_stats.view(rows, 2, C).sum(0)
    y = got["bn_stats"].double()
    close(st[0], y.sum(dim=(0, 1, 2)), "bn_stats sum")
    close(st[1], (y * y).sum(dim=(0, 1, 2)), "bn_stats sum of squares")
    st = sp_aff.view(rows, 2, C).sum(0)
    y = got["affine_mask"].double()
    close(st[0], y.sum(dim=(0, 1, 2)), "affine_mask sum")
    close(st[1], (y * xbn.double()).sum(dim=(0, 1, 2)), "affine_mask sum of out * x")
