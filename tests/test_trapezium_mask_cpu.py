"""--trapezium_mask without a GPU: the flag's default, the unchanged state_dict, the keep map against the reference
constructor's own masks (tests/golden/trapezium_*.npz), and the *_keep entry points' refusals and header prototypes."""
import json
import os
import re
from math import ceil

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle.make_trapezium_golden import CASES, case_dict


def _args(*extra, L=4):
    from lanedetection_end2end_b200.Networks.utils import define_args
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--nclasses", str(L),
                                     "--batch_size", "2"] + list(extra))


def test_flag_defaults_to_off_in_both_parsers():
    from lanedetection_end2end_b200.bev.Networks.utils import define_args as bev_args
    assert _args().trapezium_mask is False
    assert _args("--trapezium_mask", "True").trapezium_mask is True
    assert bev_args().parse_args(["--image_dir", "x", "--gt_dir", "y"]).trapezium_mask is False


@pytest.mark.parametrize("variant", ["bp", "bev"])
def test_state_dict_is_the_same_with_the_flag(variant):
    if variant == "bp":
        from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    else:
        from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    torch.manual_seed(0)
    off = Net(_args())
    torch.manual_seed(0)
    on = Net(_args("--trapezium_mask", "True"))
    assert off.keep is None
    assert [(k, v.shape) for k, v in off.state_dict().items()] == [(k, v.shape) for k, v in on.state_dict().items()]
    assert not any("keep" in k for k in on.state_dict())
    assert on.keep.dtype == torch.uint8 and tuple(on.keep.shape) == (256, 512)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_keep_map_equals_the_reference_constructors_masks(case):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net as BevNet
    c = case_dict(case)
    g = np.load(os.path.join(GOLDEN, c["name"] + ".npz"))
    assert json.loads(str(g["meta"]))["name"] == c["name"]
    net_cls = Net if c["variant"] == "Backprojection_Loss" else BevNet
    args = _args("--trapezium_mask", "True", "--resize", str(c["resize"]), "--mask_percentage", str(c["mask_pct"]),
                  "--order", str(c["order"]), L=c["L"])
    m = net_cls(args)
    keep = m.keep.numpy()
    np.testing.assert_array_equal(keep, g["keep"])
    H = c["resize"]
    assert not keep[:ceil(H * c["mask_pct"])].any()
    # linspace(1, 13, 14).long() truncates to [1, 1, 2, .., 13]: column 0 is kept, 1..13 are not; the last 14 are not
    assert keep[-1, 0] == 1 and not keep[:, 1:14].any() and not keep[:, -14:].any() and keep[-1, 14] == 1


def test_entry_points_refuse_bad_arguments_without_a_launch():
    from lanedetection_end2end_b200 import _capi
    h = _capi.lib()
    fake = 1 << 20                          # never dereferenced: every call below is refused before a launch
    k = fake
    # keep NULL
    assert h.lf_lsq_fwd_keep(fake, 0, fake, fake, fake, None, 1, 1, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake, fake,
                             1 << 20, None) == -1
    assert h.lf_lsq_fwd_rowsums_keep(fake, 0, fake, fake, None, 1, 1, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake, fake,
                                     fake, 1 << 20, None) == -1
    assert h.lf_lsq_bwd_keep(fake, 0, fake, fake, fake, None, 1, 1, 8, 8, 2, 0, 1, fake, fake, fake, fake, None) == -1
    # keep misaligned on the row-separable kernel
    assert h.lf_lsq_fwd_keep(fake, 0, fake, None, fake, k + 4, 1, 1, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake, fake,
                             1 << 20, None) == -1
    assert h.lf_lsq_bwd_keep(fake, 0, fake, None, fake, k + 4, 1, 1, 8, 8, 2, 0, 1, fake, fake, fake, fake, None) == -1
    # the plain entry points' checks hold for the keep variants: order, mask_rows, solver, dtype, workspace
    assert h.lf_lsq_fwd_keep(fake, 0, fake, fake, fake, k, 1, 1, 8, 8, 5, 0, 1, 0.0, 0, fake, fake, None, fake, fake,
                             1 << 20, None) == -1
    assert h.lf_lsq_fwd_keep(fake, 0, fake, fake, fake, k, 1, 1, 8, 8, 2, 9, 1, 0.0, 0, fake, fake, None, fake, fake,
                             1 << 20, None) == -1
    assert h.lf_lsq_fwd_keep(fake, 0, fake, fake, fake, k, 1, 1, 8, 8, 2, 0, 1, 0.0, 7, fake, fake, None, fake, fake,
                             1 << 20, None) == -1
    assert h.lf_lsq_bwd_keep(fake, 2, fake, fake, fake, k, 1, 1, 8, 8, 2, 0, 1, fake, fake, fake, fake, None) == -1
    assert h.lf_lsq_fwd_keep(fake, 0, fake, fake, fake, k, 1, 1, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake, fake,
                             16, None) == _capi.lib().lf_lsq_fwd(fake, 0, fake, fake, fake, 1, 1, 8, 8, 2, 0, 1, 0.0, 0,
                                                                  fake, fake, None, fake, fake, 16, None)


def test_op_level_keep_refusals():
    from lanedetection_end2end_b200 import ops_lsq
    assert ops_lsq.keep_map(None, 4, 8, "cpu") is None
    with pytest.raises(ValueError, match="shape"):
        ops_lsq.keep_map(torch.ones(4, 9, dtype=torch.bool), 4, 8, "cpu")
    with pytest.raises(ValueError, match="uint8"):
        ops_lsq.keep_map(torch.ones(4, 8), 4, 8, "cpu")
    k = ops_lsq.keep_map(torch.eye(4, 8, dtype=torch.bool), 4, 8, "cpu")
    assert k.dtype == torch.uint8 and torch.equal(k, torch.eye(4, 8, dtype=torch.uint8))


def test_header_prototypes_match_the_bindings():
    from lanedetection_end2end_b200 import _capi
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    for name, plain in (("lf_lsq_fwd_keep", "lf_lsq_fwd"), ("lf_lsq_fwd_rowsums_keep", "lf_lsq_fwd_rowsums"),
                        ("lf_lsq_bwd_keep", "lf_lsq_bwd")):
        decl = re.search(r"\bint %s\((.*?)\);" % name, hdr, re.S).group(1)
        params = [p.strip() for p in decl.split(",")]
        assert len(_capi.PROTOTYPES[name][1]) == len(params), name
        # the plain entry point's parameters with `const uint8_t* keep` inserted after the tables
        base = [p.strip() for p in re.search(r"\bint %s\((.*?)\);" % plain, hdr, re.S).group(1).split(",")]
        i = params.index("const uint8_t* keep")
        assert params[:i] + params[i + 1:] == base, name
        assert _capi.PROTOTYPES[name][1][:i] + _capi.PROTOTYPES[name][1][i + 1:] == _capi.PROTOTYPES[plain][1], name
