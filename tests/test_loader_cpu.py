"""The GPU loader (Dataloader/Load_Data_new.py, csrc/loader.cu) without a GPU, against tests/golden/loader_tusimple.npz (the
reference's own get_loader / get_testloader on a synthetic 3626-file directory, oracle/make_loader_golden.py):
  * the batch plans (order, label rows, validation index, flip draws) over two epochs of train and validation;
  * the host label tables, gathered by those plans, equal the reference's lanes / valid_points / horizon / line_lst;
  * load_valid_set_file_all writes the reference's bytes;
  * the reference main.py's loader import resolves to this package;
  * the C prototypes match the header, and both loader kernels compile for sm_90a without spilling."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import make_loader_golden as mlg


@pytest.fixture(scope="module")
def fixture(tmp_path_factory):
    z = np.load(os.path.join(GOLDEN, "loader_tusimple.npz"))
    paths = mlg.from_fixture(z, str(tmp_path_factory.mktemp("tusimple")))
    return z, paths


def _loaders(L, paths, resize, nclasses, seed):
    torch.manual_seed(seed)
    return L.get_loader(mlg.NUM_TRAIN, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"], True, mlg.BATCH,
                        mlg.BATCH, True, 0, True, resize, nclasses, line_file=paths["line_file"])


@pytest.mark.parametrize("case", sorted(mlg.CASES))
def test_plans_and_label_tables_match_reference(fixture, case):
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    z, paths = fixture
    resize, nclasses, seed = mlg.CASES[case]
    train, valid, valid_idx = _loaders(L, paths, resize, nclasses, seed)
    assert valid_idx == z["valid_idx/" + case].tolist()
    ds = train.dataset
    assert valid.dataset is ds and len(ds) == mlg.COUNT            # the reference's __len__ raises; this one works
    t = ds.tables
    hz = L.horizon_vectors(t["horizon"], resize)
    nflip = 0
    for e in range(mlg.EPOCHS):
        for split, loader in (("train", train), ("valid", valid)):
            key = "%s/e%d/%s/" % (case, e, split)
            plans = list(loader.plans())
            assert len(plans) == len(loader) == z[key + "idx"].shape[0]
            np.testing.assert_array_equal(np.array([p.rows for p in plans]), z[key + "idx"])
            np.testing.assert_array_equal(np.concatenate([p.draws for p in plans]), z[key + "draws"])
            if split == "valid":
                np.testing.assert_array_equal(np.array([p.index for p in plans]), z[key + "index"])
                assert not any(f for p in plans for f in p.flips)
            else:
                assert all(p.index is None for p in plans)
            for k, p in enumerate(plans):
                f = np.array(p.flips, np.int64)
                nflip += int(f.sum())
                pos = np.array(p.positions)
                np.testing.assert_array_equal(t["lanes"][f, pos], z[key + "lanes"][k])
                np.testing.assert_array_equal(t["valid"][pos], z[key + "valid_points"][k])
                np.testing.assert_array_equal(hz[pos], z[key + "horizon"][k])
                np.testing.assert_array_equal(t["line"][f, pos], z[key + "line_lst"][k])
    assert nflip > 0


def test_label_row_quirks():
    """The reference's label quirks, one by one, on hand-made rows."""
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    h48 = list(range(240, 720, 10))
    lanes = [[-2] * 10 + [500 + j for j in range(38)], [0] + [-2] * 47, [-2] * 48, [-2] * 48]
    (l0, l1), v, nh, (c0, c1) = L.label_row(lanes, h48, [-1, -1, 1, 0, -1, 1, 1, 0, -1, -1], 256)
    assert l0.shape == (4, 56) and (l0[:, :8] == -2).all()                 # 48 samples: left-padded with -2
    assert l0[0, 18] == 500 / 2.5                                           # /2.5 whatever the resize
    assert l0[1, 8] == 0 and v[1, 8] == 0                                   # x = 0: not a valid point ...
    # ... but it counts for the horizon, through the misaligned zip: lane 1's x = 0 is at padded index 8, paired with
    # h_samples[8] = 320 -> 320 / 2.5 - 32 = 96
    assert nh == 96
    assert l1[0, 8] == 511 and (l1[0, 9:] == -2).all()                      # flipped: (2R - 1) - x, lanes [1, 0, 3, 2]
    assert l1[1, 18] == 511 - 500 / 2.5
    assert (l1[1, :8] == -2).all()                                          # -2 entries restored after the flip
    np.testing.assert_array_equal(c0, [1, 0, 1, 1])                         # lines[3:7] + 1, clamped to [0, 1]
    np.testing.assert_array_equal(c1, np.clip(np.array(L.mirror_list([-1, -1, 1, 0, -1, 1, 1, 0, -1, -1])[3:7]) + 1, 0, 1))
    (n0, _), _, nh0, _ = L.label_row([[-2] * 56] * 4, list(range(160, 720, 10)), [0] * 10, 320)
    assert nh0 == 320 and (n0 == -2).all()                                  # no lane point: horizon = resize


def test_load_valid_set_file_all_matches_reference(fixture, tmp_path, monkeypatch):
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    z, paths = fixture
    monkeypatch.chdir(os.path.dirname(os.path.dirname(paths["lanes_file"])))
    target = str(tmp_path / "valid_set.json")
    L.load_valid_set_file_all(z["valid_idx/r256_c4"].tolist(), target, paths["image_dir"])
    assert open(target, "rb").read() == z["valid_set_all"].tobytes()


def test_reference_main_loader_import_resolves_to_the_package():
    """BP/main.py:20-21 `from Dataloader.Load_Data_new import get_loader, get_testloader, load_valid_set_file_all` with
    this package directory first on sys.path."""
    code = ("import sys; sys.path.insert(0, %r);"
            "from Dataloader.Load_Data_new import get_loader, get_testloader, load_valid_set_file_all;"
            "import Dataloader.Load_Data_new as m; print(m.__file__)")
    pkg = os.path.join(ROOT, "lanedetection_end2end_b200")
    out = subprocess.run([sys.executable, "-c", code % pkg], capture_output=True, text=True, cwd="/tmp")
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == os.path.join(pkg, "Dataloader", "Load_Data_new.py")
    from lanedetection_end2end_b200.Dataloader import Load_Data_new as L
    for name in ("get_loader", "get_testloader", "LaneDataset", "LaneTestSet", "load_valid_set_file_all", "load_valid_set_file",
                 "load_0313_valid_set_file", "SequentialIndicesSampler", "mirror_list", "homogenous_transformation",
                 "get_homography"):
        assert hasattr(L, name), name


def test_loader_prototypes_match_header():
    from lanedetection_end2end_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_loader_stage", "lf_loader_assemble"):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        nargs = len(decl.split(","))
        assert len(_capi.PROTOTYPES[name][1]) == nargs, name
        assert hasattr(_capi.lib(), name)
    assert re.search(r"#define LF_LOADER_LANES (\d+)", hdr).group(1) == str(_capi.LOADER_LANES)
    assert re.search(r"#define LF_LOADER_POINTS (\d+)", hdr).group(1) == str(_capi.LOADER_POINTS)


def test_loader_kernels_do_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    found = {}
    for src in ("loader.cu", "input_pipe.cu"):
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, src), "-o", str(tmp_path / "k.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        name = spills = None
        for line in r.stderr.splitlines():
            m = re.search(r"Compiling entry function '(\w+)'", line)
            if m:
                name, spills = m.group(1), None
                continue
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                spills = (int(m.group(1)), int(m.group(2)))
                continue
            m = re.search(r"Used (\d+) registers", line)
            if m and name:
                found[re.search(r"lf\d+(\w+?_kernel)", name).group(1)] = (spills, int(m.group(1)))
                name = None
    for k in ("loader_stage_kernel", "loader_assemble_kernel", "frame_preprocess_kernel", "label_preprocess_kernel"):
        assert k in found, (k, sorted(found))
        assert found[k][0] == (0, 0) and found[k][1] <= 255, (k, found[k])
