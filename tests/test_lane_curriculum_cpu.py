"""--lane_curriculum without a GPU: the flag and its refusals, the epoch -> fitted-lanes schedule, Net._split after a
prefix fit, expand_lanes on CPU-built state dicts, and the *_lanes entry points' exports, prototypes and refusals."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from conftest import ROOT

LANES_ENTRIES = [("lf_lsq_fwd_lanes", "lf_lsq_fwd"), ("lf_lsq_fwd_keep_lanes", "lf_lsq_fwd_keep"),
                 ("lf_lsq_fwd_rowsums_lanes", "lf_lsq_fwd_rowsums"),
                 ("lf_lsq_fwd_rowsums_keep_lanes", "lf_lsq_fwd_rowsums_keep"), ("lf_lsq_bwd_lanes", "lf_lsq_bwd"),
                 ("lf_lsq_bwd_keep_lanes", "lf_lsq_bwd_keep"), ("lf_lsq_fwd_per_image_lanes", "lf_lsq_fwd_per_image"),
                 ("lf_lsq_bwd_per_image_lanes", "lf_lsq_bwd_per_image")]


def _args(*extra, L=4):
    from lanedetection_end2end_b200.Networks.utils import define_args
    return define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--no_cuda", "--nclasses", str(L),
                                     "--batch_size", "2"] + list(extra))


def test_flag_defaults_to_off_in_both_parsers():
    from lanedetection_end2end_b200.bev.Networks.utils import define_args as bev_args
    assert _args().lane_curriculum == 0
    assert _args("--lane_curriculum", "3").lane_curriculum == 3
    assert bev_args().parse_args(["--image_dir", "x", "--gt_dir", "y"]).lane_curriculum == 0


@pytest.mark.parametrize("check", ["bp", "bev"])
def test_flag_refusals(check):
    from lanedetection_end2end_b200 import engine

    def run(args):
        if check == "bp":
            engine.check_bp_args(args, SimpleNamespace(), None)
        else:
            engine.check_bev_args(args)
    run(_args("--lane_curriculum", "5"))
    run(_args("--lane_curriculum", "0", L=2))
    with pytest.raises(ValueError, match="--nclasses 4"):
        run(_args("--lane_curriculum", "1", L=2))
    with pytest.raises(ValueError, match=">= 0"):
        run(_args("--lane_curriculum", "-1"))


def test_epoch_schedule():
    from lanedetection_end2end_b200.engine import curriculum_lanes
    assert [curriculum_lanes(_args("--lane_curriculum", "3"), e) for e in range(6)] == [2, 2, 2, None, None, None]
    assert [curriculum_lanes(_args(), e) for e in range(3)] == [None] * 3
    assert curriculum_lanes(SimpleNamespace(nclasses=4), 0) is None          # an args without the flag: off


@pytest.mark.parametrize("variant", ["bp", "bev"])
def test_split_after_a_prefix_fit(variant):
    if variant == "bp":
        from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    else:
        from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    m = Net(_args())
    assert m.fit_lanes is None
    beta = torch.arange(2 * 3 * 3, dtype=torch.float64).view(2, 3, 3)
    for K in (1, 2, 3):
        parts = m.ls_layer._split(beta[:, :K])
        assert [p is None for p in parts] == [k >= K for k in range(4)]
        for k in range(K):
            assert torch.equal(parts[k].double().squeeze(-1), beta[:, k])
    assert all(p is not None for p in m.ls_layer._split(torch.zeros(2, 4, 3)))


def test_check_lanes():
    from lanedetection_end2end_b200.ops_lsq import check_lanes
    assert check_lanes(None, 4) is None and check_lanes(2, 4) == 2 and check_lanes(4, 4) == 4
    for bad in (0, 5, -1, 2.0, True):
        with pytest.raises(ValueError, match="lanes"):
            check_lanes(bad, 4)


def _net(L, *extra, seed=0):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    torch.manual_seed(seed)
    m = Net(_args(*extra, L=L))
    define_init_weights(m, "normal")
    return m


def test_expand_lanes_fills_the_egolane_channels():
    from lanedetection_end2end_b200.Networks.utils import expand_lanes
    m2, m4 = _net(2), _net(4, seed=1)
    before = {k: v.clone() for k, v in m4.state_dict().items()}
    sd2 = m2.state_dict()
    assert expand_lanes(sd2, m4) == []
    heads = [k for k in before if k.endswith("output_conv.weight") or k.endswith("output_conv.bias")]
    assert "net.decoder.output_conv.weight" in heads
    for k, v in m4.state_dict().items():
        if k in heads:
            d = [i for i in range(v.dim()) if v.shape[i] != sd2[k].shape[i]][0]
            assert v.shape[d] == 4 and sd2[k].shape[d] == 2
            assert torch.equal(v.narrow(d, 0, 2), sd2[k])
            assert torch.equal(v.narrow(d, 2, 2), before[k].narrow(d, 2, 2))      # the outer lanes keep their init
        else:
            assert torch.equal(v, sd2[k]), k


def test_expand_lanes_reports_what_it_did_not_fill():
    from lanedetection_end2end_b200.Networks.utils import expand_lanes
    m2, m4 = _net(2), _net(4, "--clas", "True", seed=1)
    before = {k: v.clone() for k, v in m4.state_dict().items()}
    missing = expand_lanes(m2.state_dict(), m4)
    assert missing and all(k.startswith(("line_classification.", "horizon_estimation.")) for k in missing)
    assert set(missing) == set(before) - set(m2.state_dict())
    for k in missing:
        assert torch.equal(m4.state_dict()[k], before[k])


def test_expand_lanes_refuses_other_shape_changes():
    from lanedetection_end2end_b200.Networks.utils import expand_lanes
    m4 = _net(4)
    sd = dict(m4.state_dict())
    k = next(k for k, v in sd.items() if "output_conv" not in k and v.dim() == 4)
    sd[k] = torch.zeros(tuple(s + 1 for s in sd[k].shape))
    with pytest.raises(ValueError, match=re.escape(k)):
        expand_lanes(sd, m4)
    sd = dict(m4.state_dict())
    sd["net.decoder.output_conv.weight"] = torch.zeros(16, 5, 2, 2)      # more lanes than the model: refused
    with pytest.raises(ValueError, match="output_conv"):
        expand_lanes(sd, m4)


def _decl(hdr, name):
    return [p.strip() for p in re.search(r"\bint %s\((.*?)\);" % name, hdr, re.S).group(1).split(",")]


@pytest.mark.parametrize("name,plain", LANES_ENTRIES, ids=[e[0] for e in LANES_ENTRIES])
def test_lanes_entry_points_are_exported_with_lmap_after_l(name, plain):
    from lanedetection_end2end_b200 import _capi
    assert hasattr(_capi.lib(), name)
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    params, base = _decl(hdr, name), _decl(hdr, plain)
    i = params.index("int Lmap")
    assert params[i - 1] == "int L" and params[:i] + params[i + 1:] == base
    proto, base_proto = _capi.PROTOTYPES[name], _capi.PROTOTYPES[plain]
    assert proto[0] == base_proto[0] and proto[1][:i] + proto[1][i + 1:] == base_proto[1]
    assert proto[1][i] is _capi._i


def test_lanes_entry_points_refuse_bad_lane_counts_without_a_launch():
    from lanedetection_end2end_b200 import _capi
    h = _capi.lib()
    fake = 1 << 20                          # never dereferenced: every call below is refused before a launch
    for L, Lmap in ((3, 2), (0, 4), (2, 65536)):
        assert h.lf_lsq_fwd_lanes(fake, 0, fake, None, fake, 1, L, Lmap, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake,
                                  fake, 1 << 20, None) == -1
        assert h.lf_lsq_fwd_rowsums_lanes(fake, 0, fake, fake, 1, L, Lmap, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None, fake,
                                          fake, fake, 1 << 20, None) == -1
        assert h.lf_lsq_bwd_lanes(fake, 0, fake, None, fake, 1, L, Lmap, 8, 8, 2, 0, 1, fake, fake, fake, fake,
                                  None) == -1
        assert h.lf_lsq_fwd_per_image_lanes(fake, 0, fake, fake, None, 1, L, Lmap, 8, 8, 2, 0, 1, 0.0, 0, fake, fake,
                                            None, fake, None, fake, 1 << 20, None) == -1
        assert h.lf_lsq_bwd_per_image_lanes(fake, 0, fake, fake, None, 1, L, Lmap, 8, 8, 2, 0, 1, fake, fake, fake,
                                            fake, None) == -1
    # keep NULL is refused by the keep forms, as by the plain ones
    assert h.lf_lsq_fwd_keep_lanes(fake, 0, fake, None, fake, None, 1, 2, 4, 8, 8, 2, 0, 1, 0.0, 0, fake, fake, None,
                                   fake, fake, 1 << 20, None) == -1
    assert h.lf_lsq_bwd_keep_lanes(fake, 0, fake, None, fake, None, 1, 2, 4, 8, 8, 2, 0, 1, fake, fake, fake, fake,
                                   None) == -1
