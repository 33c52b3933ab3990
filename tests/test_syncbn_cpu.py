"""SyncBatchNorm without a GPU: the C ABI of the collapse / finalize-from-totals entry points against the header and the
library's exports, and torch.nn.SyncBatchNorm.convert_sync_batchnorm on the library's Net (with and without the --clas
heads): unchanged state_dict, and the running statistics the graphed step bumps after a replay."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT

NEW_ENTRIES = ("lf_bn_collapse", "lf_bn_finalize_tot", "lf_bn_bwd_finalize_tot", "lf_bn_bwd_finalize_sx_tot")


def _header():
    text = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", text, flags=re.S)


def _ctype_of(decl_arg):
    a = decl_arg.strip()
    if "*" in a:
        return ctypes.c_void_p
    if a.startswith("long long"):
        return ctypes.c_longlong
    if a.startswith("float"):
        return ctypes.c_float
    if a.startswith("int"):
        return ctypes.c_int
    if a.startswith("lf_stream_t"):
        return ctypes.c_void_p
    raise AssertionError(a)


def test_prototypes_match_declarations_and_exports():
    from lanedetection_end2end_b200 import _capi
    hdr = _header()
    h = _capi.lib()
    for name in NEW_ENTRIES:
        decl = re.search(r"\bint\s+%s\s*\((.*?)\);" % name, hdr, re.S)
        assert decl, name
        want = [_ctype_of(a) for a in decl.group(1).split(",")]
        res, args = _capi.PROTOTYPES[name]
        assert res is ctypes.c_int, name
        assert args == want, (name, args, want)
        assert hasattr(h, name), name


def _net(clas):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    argv = ["--image_dir", "x", "--gt_dir", "y", "--nclasses", "2", "--order", "2", "--batch_size", "2", "--no_cuda",
            "--loss_policy", "backproject"]
    if clas:
        argv += ["--clas", "1"]
    return Net(define_args().parse_args(argv))


@pytest.mark.parametrize("clas", [False, True])
def test_convert_sync_batchnorm_keeps_the_checkpoint_layout(clas):
    from lanedetection_end2end_b200.engine import batchnorm_running_stats
    torch.manual_seed(0)
    model = _net(clas)
    before = {k: (tuple(v.shape), v.dtype) for k, v in model.state_dict().items()}
    plain = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert len(plain) == (47 if clas else 39)
    stats = batchnorm_running_stats(model)
    assert len(stats) == 2 * len(plain)
    model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert not any(isinstance(m, torch.nn.BatchNorm2d) for m in model.modules())
    conv = [m for m in model.modules() if isinstance(m, torch.nn.SyncBatchNorm)]
    assert len(conv) == len(plain)
    assert {k: (tuple(v.shape), v.dtype) for k, v in model.state_dict().items()} == before
    # the graphed step bumps the converted containers' running statistics (the same tensors) after a replay
    after = batchnorm_running_stats(model)
    assert [t.data_ptr() for t in after] == [t.data_ptr() for t in stats]
    assert {id(t) for t in after} == {id(b) for m in conv for b in (m.running_mean, m.running_var)}
    # the ERFNet blocks keep their eps; the heads keep torch's default
    assert {m.eps for m in conv} == ({1e-3, 1e-5} if clas else {1e-3})


def test_bn_sync_selects_converted_containers_in_training_mode_only():
    from lanedetection_end2end_b200 import ops_net
    plain = torch.nn.BatchNorm2d(8)
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(torch.nn.Sequential(torch.nn.BatchNorm2d(8)))[0]
    assert ops_net.bn_sync(plain, True) is None
    assert ops_net.bn_sync(sync, False) is None
    s = ops_net.bn_sync(sync, True)
    assert isinstance(s, ops_net.BNSync) and s.group is None
