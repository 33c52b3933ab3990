"""The bird's-eye-view GPU loader (bev/Dataloader/Load_Data_new.py over csrc/loader.cu and the device decoders) against the
reference's own BEV get_loader (tests/golden/loader_bev.npz, oracle/make_loader_bev_golden.py): every element of every batch
bit-identical, for every case, both epochs, train and validation, with the cache on and off; the unlabelled-map error at
the end of every epoch that serves the map; one sample by index; an eager BEV training step fed by the device batch."""
import hashlib
import io
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import make_loader_bev_golden as mbg
from lanedetection_end2end_b200 import _capi
from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L

pytestmark = pytest.mark.gpu
DECODE = ("lf_jpeg_decode", "lf_png_decode", "lf_loader_stage", "lf_loader_label_rows")


@pytest.fixture(scope="module")
def fixture(tmp_path_factory):
    z = np.load(os.path.join(GOLDEN, "loader_bev.npz"))
    return z, mbg.from_fixture(z, str(tmp_path_factory.mktemp("bev")))


def sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.cpu().numpy()).tobytes()).hexdigest()


def _loaders(paths, case, **kw):
    resize, flip_on, seed = mbg.CASES[case]
    torch.manual_seed(seed)
    return L.get_loader(mbg.NUM_TRAIN, paths["json_file"], paths["image_dir"], paths["gt_dir"], flip_on, mbg.BATCH, True, 0, True,
                        resize, line_file=paths["line_file"], **kw)


def _check_batch(b, z, key, k, split):
    val = split == "valid"
    assert len(b) == (7 if val else 6)
    image, gt, params, idx, line, horizon = b[:6]
    for t in (image, gt, params, line, horizon):
        assert t.is_cuda
    assert idx.device.type == "cpu" and idx.dtype == torch.int64
    assert (image.dtype, gt.dtype, params.dtype, line.dtype, horizon.dtype) == (
        torch.float32, torch.int64, torch.float32, torch.int64, torch.float32)
    assert torch.equal(idx, torch.from_numpy(z[key + "idx"][k]))
    if val:
        assert b[6].device.type == "cpu" and torch.equal(b[6], torch.from_numpy(z[key + "index"][k]))
    assert sha(image) == z[key + "image_sha"][k], (key, k)
    assert sha(gt) == z[key + "gt_sha"][k], (key, k)
    assert params.cpu().numpy().tobytes() == z[key + "params"][k].tobytes(), (key, k)
    for name, t in (("line_lst", line), ("horizon", horizon)):
        assert torch.equal(t.cpu(), torch.from_numpy(z[key + name][k])), (key, k, name)


@pytest.mark.parametrize("cache", ["cached", "uncached"])
@pytest.mark.parametrize("case", sorted(mbg.CASES))
def test_batches_bit_identical_to_reference(fixture, case, cache):
    """Two epochs of train and validation.  Every yielded batch is overwritten after it is checked, which must not change
    later epochs.  Cached: the second epoch launches no decode, staging or label-row search."""
    z, paths = fixture
    kw = {} if cache == "cached" else {"cache_bytes": 0}
    train, valid, _ = _loaders(paths, case, **kw)
    assert train.dataset._store.cached == (cache == "cached")
    for e in range(mbg.EPOCHS):
        _capi.TRACE = [] if e == 1 else None
        try:
            for split, loader in (("train", train), ("valid", valid)):
                key = "%s/e%d/%s/" % (case, e, split)
                n = 0
                for k, b in enumerate(loader):
                    _check_batch(b, z, key, k, split)
                    for t in b:
                        t.fill_(7)
                    n += 1
                assert n == z[key + "idx"].shape[0]
            trace = [t[0] for t in _capi.TRACE or []]
        finally:
            _capi.TRACE = None
        if e == 1:
            assert trace.count("lf_loader_assemble_bev") == len(train) + len(valid)
            decodes = [t for t in trace if t in DECODE]
            assert (not decodes) if cache == "cached" else len(decodes) == 4 * (len(train) + len(valid)), decodes


def _small_dir(tmp, cache_bytes=None, n=8):
    """n unpadded names over two frames of the fixture; map 3 (names 3 and 7) has classes 3 / 4 only."""
    from PIL import Image
    from oracle.make_png_golden import pil_png
    z = np.load(os.path.join(GOLDEN, "loader_bev.npz"))
    for d in ("img", "gt", "Labels"):
        os.makedirs(os.path.join(tmp, d))
    fr = [z["jpeg/0"].tobytes(), z["jpeg/1"].tobytes()]
    m = np.zeros((720, 1280), np.uint8)
    m[300:340, 200:260] = 3
    m[500:560, 900:980] = 4
    unlabelled = pil_png(m)
    assert Image.open(io.BytesIO(unlabelled)).size == (1280, 720)
    rows = [json.loads(line) for line in z["params_jsonl"].tobytes().decode().splitlines()]
    lines = [json.loads(line) for line in z["lines_jsonl"].tobytes().decode().splitlines()]
    for k in range(1, n + 1):
        open(os.path.join(tmp, "img", "%d.jpg" % k), "wb").write(fr[k % 2])
        open(os.path.join(tmp, "gt", "%d.png" % k), "wb").write(unlabelled if k % 4 == 3 else z["png/%d" % (k % 2)].tobytes())
    for name, src in (("params.json", rows), ("lines.json", lines)):
        with open(os.path.join(tmp, "Labels", name), "w") as f:
            for k in range(n):
                f.write(json.dumps(src[k % len(src)]) + "\n")
    torch.manual_seed(0)
    return L.get_loader(n, os.path.join(tmp, "Labels", "params.json"), os.path.join(tmp, "img"), os.path.join(tmp, "gt"), True, 2,
                        True, 0, True, 256, 0.25, expected_count=None, line_file=os.path.join(tmp, "Labels", "lines.json"),
                        cache_bytes=cache_bytes)


@pytest.mark.parametrize("cache", ["cached", "uncached"])
def test_unlabelled_map_raises_at_epoch_end_and_again_next_epoch(tmp_path, cache):
    train, valid, valid_idx = _small_dir(str(tmp_path), cache_bytes=None if cache == "cached" else 0)
    ds = train.dataset
    assert ds._store.cached == (cache == "cached")
    served_bad = lambda rows: [r for r in rows if (r + 1) % 4 == 3]
    for epoch in range(2):
        it = iter(train)
        got, rows = 0, []
        with pytest.raises(ValueError, match=r"gt/[37]\.png: no labelled pixel"):
            while True:
                b = next(it)
                rows += b[3].tolist()
                got += 1
        assert got == len(train) and served_bad(rows), epoch       # every batch was yielded; the error comes at the end
    if cache == "cached":                                           # the unlabelled maps stay cached: decoding them was clean
        assert (ds._store.state[[ds.rows.index(r) for r in rows]] == 2).all()
    assert not served_bad([ds.rows[i] for i in valid_idx])
    for _ in valid:                                                 # an epoch without the unlabelled maps ends cleanly
        pass


def test_getitem_returns_one_sample(fixture):
    """ds[i] is element i of a batch: the validation sample (no flip) of the fixture's first validation batch."""
    z, paths = fixture
    case = "r256_flip"
    train, valid, _ = _loaders(paths, case)
    ds = valid.dataset
    key = case + "/e0/valid/"
    list(train.plans())                                             # the torch RNG as the fixture's first training epoch left it
    b = next(iter(valid))
    _check_batch(b, z, key, 0, "valid")
    row = int(z[key + "idx"][0][0])
    s = ds[ds.rows.index(row)]
    assert len(s) == 7 and s[3] == row and s[6] == int(z[key + "index"][0][0])
    for k in (0, 1, 2, 4, 5):
        assert s[k].is_cuda and torch.equal(s[k], b[k][0]), k


def test_bev_step_fed_by_device_batch_equals_cpu_batch(fixture):
    """One eager BEV step (bev Net + Area_Loss, the reference main.py's end-to-end loss) fed by the device batch equals the
    step fed by the reference's CPU batch (the same bits, checked against the fixture, moved to the device as main.py does)."""
    from lanedetection_end2end_b200.bev.Loss_crit import Area_Loss
    from lanedetection_end2end_b200.bev.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    z, paths = fixture
    case = "r256_flip"
    train, _, _ = _loaders(paths, case)
    b = next(iter(train))
    _check_batch(b, z, case + "/e0/train/", 0, "train")
    cpu = [t.cpu() for t in b]
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--batch_size", str(mbg.BATCH), "--nclasses", "2",
                                     "--order", "2"])
    torch.manual_seed(0)
    model = Net(args).cuda().train()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0
    crit = Area_Loss(args.order, "none")

    def step(image, params):
        model.zero_grad()
        out = model(image, True)
        loss = crit(out[0], params[:, 0, :]) + crit(out[1], params[:, 1, :])
        loss.backward()
        return loss.detach().clone(), [p.grad.detach().clone() for p in model.parameters() if p.grad is not None]

    l_dev, g_dev = step(b[0], b[2])
    l_cpu, g_cpu = step(cpu[0].cuda(non_blocking=True).float(), cpu[2].cuda(non_blocking=True))
    assert torch.isfinite(l_dev) and len(g_dev) == len(g_cpu) > 0
    torch.testing.assert_close(l_dev, l_cpu, rtol=1e-6, atol=0)
    for a, c in zip(g_dev, g_cpu):
        torch.testing.assert_close(a, c, rtol=1e-5, atol=1e-7)
