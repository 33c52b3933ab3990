"""The *_lanes least-squares entry points against the plain ones: fitting lanes [0, K) of [B, 4, H, W] maps gives, bit for
bit, what the plain entry point gives on a contiguous copy of o[:, :K] -- beta, zinv, masked, rowsums, status and d_o --
while the backward leaves d_o exactly +0.0 on lanes [K, 4); masked is compact, [B, K, H, W].  With K = 4 the new
entry points are the old ones."""
import numpy as np
import pytest
import torch

from lanedetection_end2end_b200 import _capi
from lanedetection_end2end_b200.Networks.LSQ_layer import ProjectiveGridGenerator, trapezium_keep
from lanedetection_end2end_b200.Networks.utils import get_homography
from lanedetection_end2end_b200 import ops_lsq
from oracle import inputs

pytestmark = pytest.mark.gpu

B, LMAP = 2, 4
VARIANTS = ["shared", "shared_keep", "rowsums", "rowsums_keep", "per_image", "per_image_keep", "general", "general_keep"]
_INT = {torch.float64: torch.int64, torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int32: torch.int32}


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(_INT[a.dtype]),
                                                                   b.contiguous().view(_INT[b.dtype]))


def tables(variant):
    """(H, W, mask_rows, xtab, ytab, yrow, keep) on the device: the fixed warp at 256 x 512 (row-separable), per-image
    tables moved per image, or a general (non-separable) 64 x 96 grid."""
    if variant.startswith("general"):
        H, W, mr = 64, 96, 10
        r = torch.arange(H, dtype=torch.float32)[:, None]
        c = torch.arange(W, dtype=torch.float32)[None, :]
        xtab = (2.0 * c + 0.1 * r).reshape(-1).cuda()
        ytab = (255.0 - 3.0 * r - 0.01 * c).reshape(-1).cuda()
        keep = (torch.rand(H, W, generator=torch.Generator().manual_seed(3)) > 0.2).to(torch.uint8).cuda()
        return H, W, mr, xtab, ytab, None, keep
    H, W, mr = 256, 512, 77
    M, _ = get_homography(256)
    grid = ProjectiveGridGenerator((B, LMAP, H, W), torch.from_numpy(M).unsqueeze(0).float(), False)
    t = ops_lsq.GridTables(grid, H, W, 255.0)
    assert t.rowsep
    keep = trapezium_keep(256, mr).cuda()
    if variant.startswith("per_image"):
        xtab = torch.stack([t.xtab.view(H, W) + 0.5 * b for b in range(B)]).contiguous()
        yrow = torch.stack([t.yrow + 0.25 * b for b in range(B)]).contiguous()
        return H, W, mr, xtab, None, yrow, keep
    return H, W, mr, t.xtab, t.ytab, t.yrow, keep


def forward(variant, o, K, lanes, order, tabs):
    """One forward launch: the *_lanes entry point on o (K of its lanes) or the plain one on o itself (K = its lanes)."""
    H, W, mr, xtab, ytab, yrow, keep = tabs
    if variant.startswith("general"):
        yrow = None
    Lm, n, p = o.shape[1], order + 1, _capi.ptr
    dev = o.device
    beta = torch.full((B, K, n), float("nan"), dtype=torch.float64, device=dev)
    zinv = torch.full((B, K, n, n), float("nan"), dtype=torch.float64, device=dev)
    masked = torch.full((B, K, H, W), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    rowsums = torch.full((B, K, H, 3), float("nan"), device=dev) if variant in ("rowsums", "rowsums_keep", "per_image") \
        else None
    ws = torch.zeros(_capi.lib().lf_lsq_workspace_bytes(B, K, H, W, order), dtype=torch.uint8, device=dev)
    use_keep = variant.endswith("_keep")
    ls, sfx = ((K, Lm), "_lanes") if lanes else ((K,), "")
    head = (p(o), _capi.dtype_id(o), p(xtab))
    tail = (H, W, order, mr, _capi.ACT_IDS["square"], 0.0, _capi.SOLVER_INVERSE, p(beta), p(zinv), p(masked), p(status))
    wsa = (p(ws), ws.numel(), _capi.stream_ptr())
    if variant.startswith("per_image"):
        _capi.call("lf_lsq_fwd_per_image" + sfx, *head, p(yrow), p(keep) if use_keep else None, B, *ls, *tail, p(rowsums),
                   *wsa)
    elif variant.startswith("rowsums"):
        kp = (p(keep),) if use_keep else ()
        _capi.call("lf_lsq_fwd_rowsums" + ("_keep" if use_keep else "") + sfx, *head, p(yrow), *kp, B, *ls, *tail,
                   p(rowsums), *wsa)
    else:
        kp = (p(keep),) if use_keep else ()
        _capi.call("lf_lsq_fwd" + ("_keep" if use_keep else "") + sfx, *head, p(ytab), p(yrow), *kp, B, *ls, *tail, *wsa)
    torch.cuda.synchronize()
    return dict(beta=beta, zinv=zinv, masked=masked, status=status, rowsums=rowsums)


def backward(variant, o, K, lanes, order, tabs, beta, zinv, gbeta):
    H, W, mr, xtab, ytab, yrow, keep = tabs
    if variant.startswith("general"):
        yrow = None
    p = _capi.ptr
    d_o = torch.full_like(o, float("nan"))
    use_keep = variant.endswith("_keep")
    ls, sfx = ((K, o.shape[1]), "_lanes") if lanes else ((K,), "")
    tail = (H, W, order, mr, _capi.ACT_IDS["square"], p(beta), p(zinv), p(gbeta), p(d_o), _capi.stream_ptr())
    if variant.startswith("per_image"):
        _capi.call("lf_lsq_bwd_per_image" + sfx, p(o), _capi.dtype_id(o), p(xtab), p(yrow),
                   p(keep) if use_keep else None, B, *ls, *tail)
    else:
        kp = (p(keep),) if use_keep else ()
        _capi.call("lf_lsq_bwd" + ("_keep" if use_keep else "") + sfx, p(o), _capi.dtype_id(o), p(xtab), p(ytab),
                   p(yrow), *kp, B, *ls, *tail)
    torch.cuda.synchronize()
    return d_o


@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_prefix_fit_is_the_plain_fit_of_the_copy(variant, dtype, order, K):
    tabs = tables(variant)
    H, W = tabs[0], tabs[1]
    o = torch.from_numpy(inputs.make_lane_maps(B, LMAP, H, W, seed=100 * order + K)).cuda()
    if dtype == "bf16":
        o = o.bfloat16()
    copy = o[:, :K].contiguous()
    got = forward(variant, o, K, True, order, tabs)
    want = forward(variant, copy, K, False, order, tabs)
    assert int(want["status"].item()) == 0
    for k in ("beta", "zinv", "status"):
        assert same_bits(got[k], want[k]), k
    assert same_bits(got["masked"], want["masked"]), "masked"
    if want["rowsums"] is not None:
        assert same_bits(got["rowsums"], want["rowsums"]), "rowsums"
    g = torch.Generator(device="cuda").manual_seed(K)
    gbeta = torch.randn(B, K, order + 1, dtype=torch.float64, device="cuda", generator=g)
    d_got = backward(variant, o, K, True, order, tabs, want["beta"], want["zinv"], gbeta)
    d_want = backward(variant, copy, K, False, order, tabs, want["beta"], want["zinv"], gbeta)
    assert same_bits(d_got[:, :K], d_want), "d_o"
    assert not torch.isnan(d_want).any()
    zero = d_got[:, K:].contiguous().view(_INT[d_got.dtype])
    assert (zero == 0).all(), "d_o past K must be +0.0"


def test_a_singular_unfitted_lane_does_not_reach_status():
    """Lane 2 all zeros makes its system singular: the 2-lane prefix fit never sees it, the full fit reports it."""
    tabs = tables("shared")
    o = torch.from_numpy(inputs.make_lane_maps(B, LMAP, 256, 512, seed=7)).cuda()
    o[:, 2] = 0
    assert int(forward("shared", o, 2, True, 3, tabs)["status"].item()) == 0
    assert int(forward("shared", o, 4, False, 3, tabs)["status"].item()) & _capi.STATUS_SINGULAR


def test_ops_lsq_routes_lanes():
    """ops_lsq.lsq(..., lanes=K): beta and masked of the copy's fit, the gradient of the copy's fit on lanes [0, K) and
    zero past them."""
    H, W = 256, 512
    M, _ = get_homography(256)
    grid = ProjectiveGridGenerator((B, LMAP, H, W), torch.from_numpy(M).unsqueeze(0).float(), False)
    o = torch.from_numpy(inputs.make_lane_maps(B, LMAP, H, W, seed=9)).cuda().requires_grad_()
    c = o.detach()[:, :2].contiguous().requires_grad_()
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    b1, m1 = ops_lsq.lsq(o, grid, 2, mask_rows=52, act="square", want_masked=True, status_out=st, lanes=2)
    b2, m2 = ops_lsq.lsq(c, grid, 2, mask_rows=52, act="square", want_masked=True, status_out=st)
    assert tuple(b1.shape) == (B, 2, 3) and tuple(m1.shape) == (B, 2, H, W)
    assert same_bits(b1, b2) and torch.equal(m1, m2)
    w = torch.randn(B, 2, 3, dtype=torch.float64, device="cuda")
    (b1 * w).sum().backward()
    (b2 * w).sum().backward()
    assert same_bits(o.grad[:, :2].contiguous(), c.grad) and (o.grad[:, 2:] == 0).all()
    with pytest.raises(ValueError, match="lanes"):
        ops_lsq.lsq(o, grid, 2, lanes=5)
    np.testing.assert_array_equal(st.cpu().numpy(), [0])
