"""The GPU loader (Dataloader/Load_Data_new.py over csrc/loader.cu and the device decoders) against the reference's own
get_loader / get_testloader (tests/golden/loader_tusimple.npz, oracle/make_loader_golden.py): every element of every batch
bit-identical, for every case, both epochs, train, validation and test; epoch 2 served from the device cache; the
preprocessors' output on the same files and flips; decoder errors; inference.test_model fed by the test loader."""
import hashlib
import io
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import make_loader_golden as mlg
from lanedetection_end2end_b200 import _capi
from lanedetection_end2end_b200.Dataloader import Load_Data_new as L

pytestmark = pytest.mark.gpu
DECODE = ("lf_jpeg_decode", "lf_png_decode", "lf_loader_stage")


@pytest.fixture(scope="module")
def fixture(tmp_path_factory):
    z = np.load(os.path.join(GOLDEN, "loader_tusimple.npz"))
    return z, mlg.from_fixture(z, str(tmp_path_factory.mktemp("tusimple")))


def sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.cpu().numpy()).tobytes()).hexdigest()


def _loaders(paths, resize, nclasses, seed, **kw):
    torch.manual_seed(seed)
    return L.get_loader(mlg.NUM_TRAIN, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"], True, mlg.BATCH,
                        mlg.BATCH, True, 0, True, resize, nclasses, line_file=paths["line_file"], **kw)


def _check_batch(b, z, key, k, split):
    val = split == "valid"
    assert len(b) == (8 if val else 7)
    image, gt, lanes, idx, line, horizon = b[:6]
    valid = b[-1]
    for t in (image, gt, lanes, line, horizon, valid):
        assert t.is_cuda
    assert idx.device.type == "cpu" and idx.dtype == torch.int64
    assert (image.dtype, gt.dtype, lanes.dtype, line.dtype, horizon.dtype, valid.dtype) == (
        torch.float32, torch.int64, torch.float64, torch.float32, torch.float32, torch.float64)
    assert torch.equal(idx, torch.from_numpy(z[key + "idx"][k]))
    if val:
        assert b[6].device.type == "cpu" and torch.equal(b[6], torch.from_numpy(z[key + "index"][k]))
    assert sha(image) == z[key + "image_sha"][k], (key, k)
    assert sha(gt) == z[key + "gt_sha"][k], (key, k)
    for name, t in (("lanes", lanes), ("line_lst", line), ("horizon", horizon), ("valid_points", valid)):
        assert torch.equal(t.cpu(), torch.from_numpy(z[key + name][k])), (key, k, name)


@pytest.mark.parametrize("cache", ["cached", "uncached"])
@pytest.mark.parametrize("case", sorted(mlg.CASES))
def test_batches_bit_identical_to_reference(fixture, case, cache):
    """Two epochs of train and validation and the test loader twice.  Every yielded batch is overwritten after it is checked,
    which must not change later epochs.  Cached: the second epoch launches no decode or staging."""
    z, paths = fixture
    resize, nclasses, seed = mlg.CASES[case]
    kw = {} if cache == "cached" else {"cache_bytes": 0}
    train, valid, _ = _loaders(paths, resize, nclasses, seed, **kw)
    assert train.dataset._store.cached == (cache == "cached")
    for e in range(mlg.EPOCHS):
        _capi.TRACE = [] if e == 1 else None
        try:
            for split, loader in (("train", train), ("valid", valid)):
                key = "%s/e%d/%s/" % (case, e, split)
                n = 0
                for k, b in enumerate(loader):
                    _check_batch(b, z, key, k, split)
                    for t in b:
                        t.fill_(7)                  # the batch is the caller's: later epochs do not see this
                    n += 1
                assert n == z[key + "idx"].shape[0]
            trace = [t[0] for t in _capi.TRACE or []]
        finally:
            _capi.TRACE = None
        if e == 1:
            assert trace.count("lf_loader_assemble") == len(train) + len(valid)
            decodes = [t for t in trace if t in DECODE]
            assert (not decodes) if cache == "cached" else len(decodes) == 3 * (len(train) + len(valid)), decodes
    for rep in range(2):
        test = L.get_testloader(paths["test_dir"], mlg.BATCH, 0, resize=resize, **kw) if rep == 0 else test
        got = [b for b in test]
        assert [tuple(b.shape) for b in got] == [tuple(s) for s in z[case + "/test/shape"]]
        assert all(b.is_cuda and b.dtype == torch.float32 for b in got)
        assert [sha(b) for b in got] == z[case + "/test/image_sha"].tolist(), rep


def test_loader_equals_preprocessors_on_the_same_files_and_flips(fixture):
    """The staged-then-assembled batch equals JpegDecoder / PngDecoder -> FramePreprocessor / LabelPreprocessor on the same
    files with the same flips (the flip draws of the fixture)."""
    from lanedetection_end2end_b200 import jpeg, png
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor, LabelPreprocessor
    z, paths = fixture
    case = "r256_c2"
    resize, nclasses, seed = mlg.CASES[case]
    train, _, _ = _loaders(paths, resize, nclasses, seed)
    fpre, lpre = FramePreprocessor(resize), LabelPreprocessor(resize, nclasses)
    draws = z[case + "/e0/train/draws"]
    nflip = 0
    for k, b in enumerate(train):
        rows = b[3].tolist()
        flips = torch.tensor([bool(u > 0.5) for u in draws[4 * k:4 * k + 4]])
        nflip += int(flips.sum())
        frames = jpeg.JpegDecoder()([open(os.path.join(paths["image_dir"], "%d.jpg" % (r + 1)), "rb").read() for r in rows])
        maps = png.PngDecoder()([open(os.path.join(paths["gt_dir"], "%d.png" % (r + 1)), "rb").read() for r in rows])
        assert torch.equal(b[0], fpre(frames, flip=flips))
        assert torch.equal(b[1], lpre(maps, flip=flips))
    assert 0 < nflip < 4 * len(train)


def _small_dir(tmp, n=8, progressive=False, corrupt=False):
    """n unpadded names over two frames / two maps of the fixture, with label files of n rows."""
    from PIL import Image
    z = np.load(os.path.join(GOLDEN, "loader_tusimple.npz"))
    for d in ("img", "gt", "Labels"):
        os.makedirs(os.path.join(tmp, d))
    fr = [z["jpeg/0"].tobytes(), z["jpeg/1"].tobytes()]
    if progressive:
        bio = io.BytesIO()
        Image.open(io.BytesIO(fr[1])).save(bio, "JPEG", progressive=True)
        fr[1] = bio.getvalue()
    mp = [z["png/0"].tobytes(), z["png/1"].tobytes()]
    if corrupt:                                        # flip bits in the middle of the first map's IDAT payload
        b = bytearray(mp[0])
        i = b.index(b"IDAT") + 4
        n_idat = int.from_bytes(b[i - 8:i - 4], "big")
        for j in range(i + n_idat // 2, i + n_idat // 2 + 64):
            b[j] ^= 0x5A
        mp[0] = bytes(b)
    rows = [json.loads(line) for line in z["lanes_jsonl"].tobytes().decode().splitlines()]
    lines = [json.loads(line) for line in z["lines_jsonl"].tobytes().decode().splitlines()]
    for k in range(1, n + 1):
        open(os.path.join(tmp, "img", "%d.jpg" % k), "wb").write(fr[k % 2])
        open(os.path.join(tmp, "gt", "%d.png" % k), "wb").write(mp[k % 2])
    for name, src in (("lanes.json", rows), ("lines.json", lines)):
        with open(os.path.join(tmp, "Labels", name), "w") as f:
            for k in range(n):
                f.write(json.dumps(src[k % len(src)]) + "\n")
    lf = os.path.join(tmp, "Labels", "lanes.json")
    torch.manual_seed(0)
    return L.get_loader(n, lf, lf, os.path.join(tmp, "img"), os.path.join(tmp, "gt"), True, 2, 1, True, 0, True, 256, 4,
                        expected_count=None, line_file=os.path.join(tmp, "Labels", "lines.json"))


def test_corrupt_png_raises_at_epoch_end_and_again_next_epoch(tmp_path):
    train, _, _ = _small_dir(str(tmp_path), corrupt=True)
    assert train.dataset._store.cached
    for epoch in range(2):
        it = iter(train)
        got = 0
        with pytest.raises(ValueError, match="corrupt PNG"):
            while True:
                next(it)
                got += 1
        assert got == len(train), epoch                 # every batch was yielded; the error comes at the end
        assert not (train.dataset._store.state == 2).any()


def test_unsupported_jpeg_raises_naming_the_file(tmp_path):
    train, _, _ = _small_dir(str(tmp_path), progressive=True)
    with pytest.raises(ValueError, match=r"img/\d*[13579]\.jpg: unsupported JPEG: progressive"):
        for _ in train:
            pass


def test_test_model_fed_by_the_test_loader(fixture, tmp_path, capsys):
    """inference.test_model over get_testloader's device batches gives the accuracy and prediction file it gives over CPU
    tensors of the same frames."""
    from lanedetection_end2end_b200 import inference
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_args
    z, paths = fixture
    args = define_args().parse_args(["--image_dir", "x", "--gt_dir", "y", "--nclasses", "4", "--order", "3", "--batch_size",
                                     str(mlg.BATCH), "--clas", "1", "--end_to_end", "True"])
    torch.manual_seed(0)
    model = Net(args).cuda().eval()
    args.test_dir, args.save_path = paths["test_dir"], str(tmp_path)
    out = tmp_path / "test_set_predictions.json"
    cpu = [b.cpu() for b in L.get_testloader(paths["test_dir"], mlg.BATCH, 0)]
    assert sum(b.shape[0] for b in cpu) == mlg.NTEST
    acc_cpu = inference.test_model(cpu, model, None, None, None, None, args)
    want = out.read_text()
    acc_dev = inference.test_model(L.get_testloader(paths["test_dir"], mlg.BATCH, 2), model, None, None, None, None, args)
    assert acc_dev == acc_cpu and out.read_text() == want
    assert "===> Average ACC on TESTSET is" in capsys.readouterr().out
