"""The proxy segmentation decoder (--seg_proxy) without a GPU: the branch's state_dict keys and shapes against the
reference module's (golden), the refusals, the unchanged model without the flag, SyncBatchNorm conversion of the branch,
lf_seg_confusion's prototype, argument refusals and register report, and a numpy restatement of its counts against
torch.argmax + bincount."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from lanedetection_end2end_b200 import _capi
from lanedetection_end2end_b200.Networks.utils import define_args

INVALID = -1
CASES = ("seg_proxy_l2_d2", "seg_proxy_l4_d3_clas")


def _args(*extra):
    return define_args().parse_args(["--image_dir", ".", "--gt_dir", ".", "--no_cuda", "--loss_policy", "backproject",
                                     "--batch_size", "2"] + list(extra))


def _case_args(name, *extra):
    meta = json.loads(str(np.load(os.path.join(GOLDEN, name + ".npz"))["meta"]))
    return meta, _args("--nclasses", str(meta["L"]), "--order", str(meta["order"]), "--clas", str(int(meta["clas"])),
                       "--mask_percentage", str(meta["mask_pct"]), *extra)


def confusion_restated(logits, target):
    """The counts lf_seg_confusion adds: the winner starts at class 0 and moves to class c only where logit c is greater
    (the first maximum wins; a NaN in class c >= 1 never wins, a NaN in class 0 is never beaten); pixels whose target
    lies outside [0, C) are skipped.  logits [B, C, H, W] float32, target [B, H, W] int64 -> [C * C] int64."""
    C = logits.shape[1]
    best, arg = logits[:, 0].copy(), np.zeros(logits[:, 0].shape, np.int64)
    for c in range(1, C):
        win = logits[:, c] > best
        best = np.where(win, logits[:, c], best)
        arg = np.where(win, c, arg)
    ok = (target >= 0) & (target < C)
    return np.bincount((target[ok] * C + arg[ok]).ravel(), minlength=C * C).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_branch_keys_and_shapes_match_reference_module(name):
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    _, args = _case_args(name, "--seg_proxy", "1")
    ref = [(k, s) for k, s in json.loads(str(np.load(os.path.join(GOLDEN, name + ".npz"))["state_dict_keys"]))]
    ours = [(k, list(v.shape)) for k, v in Net(args).state_dict().items()]
    assert ours == ref
    branch = [k for k, _ in ours if k.startswith("net.decoder.layers1.")]
    assert "net.decoder.layers1.6.weight" in branch and "net.decoder.layers1.6.bias" in branch
    assert {k.split(".")[3] for k in branch} == {str(i) for i in range(7)}


def test_branch_head_has_background_class():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    for L in (2, 4):
        m = Net(_args("--nclasses", str(L), "--seg_proxy", "1"))
        assert tuple(m.net.decoder.layers1[6].weight.shape) == (16, L + 1, 2, 2)
        assert m.seg_proxy and m.net.decoder.do_segmentation


def test_refusals():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net as BevNet
    with pytest.raises(ValueError, match="end_to_end"):
        Net(_args("--seg_proxy", "1", "--end_to_end", "0", "--nclasses", "4"))
    with pytest.raises(ValueError, match="pretrained"):
        Net(_args("--seg_proxy", "1", "--pretrained", "1"))
    with pytest.raises(ValueError, match="bird's-eye-view"):
        BevNet(_args("--seg_proxy", "1", "--loss_policy", "area"))


@pytest.mark.parametrize("L,clas", [(2, 0), (4, 1)])
def test_flag_off_leaves_model_unchanged(L, clas):
    from lanedetection_end2end_b200.Networks import ERFNet
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    m = Net(_args("--nclasses", str(L), "--clas", str(clas)))
    assert m.seg_proxy is False and not hasattr(m.net.decoder, "layers1")
    assert not any(".layers1." in k for k in m.state_dict())
    # the same parameters and keys as the reference's ERFNet (whole-path golden's record) and a keyword-free build
    g = np.load(os.path.join(GOLDEN, "net_l%d_d%d.npz" % (L, 2 if L == 2 else 3)))
    ref = [k for k, _, _ in json.loads(str(g["state_dict_keys"]))]
    assert [k for k in m.state_dict() if not k.startswith(("line_classification.", "horizon_estimation."))] == ref
    torch.manual_seed(0)
    a = ERFNet.Net(in_channels=3, out_channels=L)
    torch.manual_seed(0)
    b = ERFNet.Net(in_channels=3, out_channels=L, do_segmentation=False)
    assert [(k, v.shape) for k, v in a.state_dict().items()] == [(k, v.shape) for k, v in b.state_dict().items()]
    for (ka, pa), (kb, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert ka == kb and torch.equal(pa, pb)


def test_checkpoint_without_branch_loads_non_strict():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    plain = Net(_args())
    proxy = Net(_args("--seg_proxy", "1"))
    define_init_weights(proxy, "kaiming")
    before = {k: v.clone() for k, v in proxy.state_dict().items() if ".layers1." in k}
    missing, unexpected = proxy.load_state_dict(plain.state_dict(), strict=False)
    assert not unexpected and missing and all(".layers1." in k for k in missing)
    # BatchNorm fills an absent num_batches_tracked itself (0), without listing it
    assert set(missing) == {k for k in before if not k.endswith("num_batches_tracked")}
    for k, v in proxy.state_dict().items():
        if k in before:
            assert torch.equal(v, before[k]), k          # the branch keeps its initialisation
        else:
            assert torch.equal(v, plain.state_dict()[k]), k


def test_syncbatchnorm_conversion_covers_branch():
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(Net(_args("--seg_proxy", "1")))
    bns = [(n, type(mod)) for n, mod in m.named_modules() if ".layers1." in n and "bn" in n.rsplit(".", 1)[-1]]
    assert len(bns) == 2 + 4 * 2                         # two upsamplers' bn, four residual blocks' bn1 / bn2
    assert all(t is torch.nn.SyncBatchNorm for _, t in bns), bns


def test_parser_flags():
    a = _args()
    assert a.seg_proxy is False and a.weight_seg_proxy == 1.0
    a = _args("--seg_proxy", "--weight_seg_proxy", "0.25")
    assert a.seg_proxy is True and a.weight_seg_proxy == 0.25


# ---------------------------------------------------------------------------------------------------------------------
# lf_seg_confusion
# ---------------------------------------------------------------------------------------------------------------------
def test_confusion_prototype_matches_declaration_and_export():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "lanefit_b200.h")).read(), flags=re.S)
    decl = re.search(r"\bint\s+lf_seg_confusion\s*\((.*?)\);", hdr, re.S)
    assert decl
    assert len(_capi.PROTOTYPES["lf_seg_confusion"][1]) == len(decl.group(1).split(","))
    assert hasattr(_capi.lib(), "lf_seg_confusion")


no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="host addresses as device pointers: CPU-only machines")


@no_device
@pytest.mark.parametrize("bad", [dict(C=1), dict(C=0), dict(C=9), dict(C=-3), dict(B=0), dict(B=-1), dict(H=0), dict(W=0),
                                 dict(H=-2), dict(logits=None), dict(target=None), dict(counts=None)])
def test_confusion_refuses_bad_arguments(bad):
    mem = np.zeros(1 << 10, np.float64)
    a = dict(logits=mem.ctypes.data, target=mem.ctypes.data + 1024, B=2, C=3, H=4, W=4, counts=mem.ctypes.data + 4096)
    a.update(bad)
    rc = _capi.lib().lf_seg_confusion(a["logits"], a["target"], a["B"], a["C"], a["H"], a["W"], None, a["counts"], None)
    assert rc == INVALID
    assert not mem.any()


def test_restatement_equals_torch_argmax_bincount():
    rng = np.random.default_rng(0)
    for C in (2, 3, 5, 8):
        x = rng.standard_normal((3, C, 7, 11)).astype(np.float32)          # continuous draws: no ties
        t = rng.integers(-2, C + 2, size=(3, 7, 11))
        got = confusion_restated(x, t)
        pred = torch.from_numpy(x).argmax(1)
        tt = torch.from_numpy(t)
        ok = (tt >= 0) & (tt < C)
        want = torch.bincount((tt[ok] * C + pred[ok]), minlength=C * C).numpy()
        np.testing.assert_array_equal(got, want)
        assert got.sum() == int(ok.sum())


def test_restatement_ties_and_nan():
    x = np.array([[1, 1, 0], [0, 2, 2], [np.nan, 5, 6], [3, np.nan, 1], [0, 1, np.nan], [np.nan, np.nan, np.nan]],
                 np.float32).T.reshape(1, 3, 1, 6)
    t = np.zeros((1, 1, 6), np.int64)
    got = confusion_restated(x, t).reshape(3, 3)[0]
    # first maximum wins (0, 1); a NaN at class 0 is never beaten (0, 0); a NaN elsewhere never wins (0, 1)
    assert got.tolist() == [4, 2, 0]


def test_confusion_kernel_does_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "seg.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            found[name] = (int(m.group(1)), int(m.group(2)))
    k = [n for n in found if "seg_confusion_kernel" in n]
    assert len(k) == 1, sorted(found)
    assert found[k[0]] == (0, 0), found
