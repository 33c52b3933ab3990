"""The bird's-eye-view GPU loader (bev/Dataloader/Load_Data_new.py) without a GPU, against tests/golden/loader_bev.npz (the
reference's own BEV get_loader on a synthetic 2535-file directory, oracle/make_loader_bev_golden.py):
  * the batch plans (order, label rows, validation index, flip draws) over two epochs of train and validation;
  * the host params / line tables, gathered by those plans, equal the reference's batches;
  * write_lsq_results, load_valid_set_file_all and get_homography give the reference's bytes and values;
  * label rows past the end of the label files raise IndexError when the dataset is built;
  * the reference BEV main.py's loader import resolves to this package;
  * the C prototypes match the header, and the new kernels compile for sm_90a without spilling."""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import make_loader_bev_golden as mbg


@pytest.fixture(scope="module")
def fixture(tmp_path_factory):
    z = np.load(os.path.join(GOLDEN, "loader_bev.npz"))
    return z, mbg.from_fixture(z, str(tmp_path_factory.mktemp("bev")))


def _loaders(L, paths, resize, flip_on, seed):
    torch.manual_seed(seed)
    return L.get_loader(mbg.NUM_TRAIN, paths["json_file"], paths["image_dir"], paths["gt_dir"], flip_on, mbg.BATCH, True, 0, True,
                        resize, line_file=paths["line_file"])


@pytest.mark.parametrize("case", sorted(mbg.CASES))
def test_plans_and_label_tables_match_reference(fixture, case):
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    z, paths = fixture
    resize, flip_on, seed = mbg.CASES[case]
    train, valid, valid_idx = _loaders(L, paths, resize, flip_on, seed)
    assert valid_idx == z["valid_idx/" + case].tolist()
    assert len(valid_idx) % mbg.BATCH == 0
    ds = train.dataset
    assert valid.dataset is ds and len(ds) == mbg.COUNT            # the reference's __len__ raises; this one works
    t = ds.tables
    nflip = 0
    for e in range(mbg.EPOCHS):
        for split, loader in (("train", train), ("valid", valid)):
            key = "%s/e%d/%s/" % (case, e, split)
            plans = list(loader.plans())
            assert len(plans) == len(loader) == z[key + "idx"].shape[0]
            assert all(len(p.positions) == mbg.BATCH for p in plans)
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
                got = t["params"][f, pos]
                assert got.tobytes() == z[key + "params"][k].tobytes(), (key, k)     # bits: -0.0 included
                np.testing.assert_array_equal(t["line"][f, pos], z[key + "line_lst"][k])
    assert (nflip > 0) == flip_on


def test_label_row_tables_by_hand():
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    pp = [[0.5, -0.25, 0.125], [0, 0, 0], [1e-3, 2e-2, 0.3], [0, 0, 0]]
    lines = [-1, -1, 1, 0, -1, 1, 1, 0, -1, -1]
    t = L.label_tables([{"poly_params": pp}, {"poly_params": [[0, 0, 0]] * 4}], [{"lines": lines}] * 2, [0, 1])
    np.testing.assert_array_equal(t["params"][0, 0], np.array(pp, np.float32))
    want = -np.array([pp[1], pp[0], pp[3], pp[2]])
    want[:, -1] += 1
    assert t["params"][1, 0].tobytes() == want.astype(np.float32).tobytes()
    assert np.signbit(t["params"][1, 0, 0, 0])                   # float rows: the negated zeros stay -0.0
    assert not np.signbit(t["params"][1, 1]).any()               # integer-only rows negate in int64: +0
    np.testing.assert_array_equal(t["params"][1, 1, :, 2], 1)
    assert t["line"].dtype == np.int64
    np.testing.assert_array_equal(t["line"][0, 0], [1, 0, 2, 2])                 # lines[3:7] + 1, not clamped
    np.testing.assert_array_equal(t["line"][1, 0], np.array(L.mirror_list(lines)[3:7]) + 1)
    with pytest.raises(IndexError, match="label row 2 is past the end of the params file"):
        L.label_tables([{"poly_params": pp}] * 2, [{"lines": lines}] * 3, [0, 2])
    with pytest.raises(IndexError, match="past the end of the line file"):
        L.label_tables([{"poly_params": pp}] * 3, [{"lines": lines}] * 2, [2])


def test_dataset_rejects_label_rows_past_the_files(tmp_path):
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    for d in ("img", "gt"):
        os.makedirs(tmp_path / d)
    for n in (1, 2, 5):
        (tmp_path / "img" / ("%d.jpg" % n)).write_bytes(b"")
        (tmp_path / "gt" / ("%d.png" % n)).write_bytes(b"")
    row = json.dumps({"poly_params": [[0, 0, 0]] * 4}) + "\n"
    (tmp_path / "p.json").write_text(row * 4)
    (tmp_path / "l.json").write_text((json.dumps({"lines": [0] * 10}) + "\n") * 5)
    with pytest.raises(IndexError, match="label row 4 is past the end of the params file"):
        L.get_loader(3, str(tmp_path / "p.json"), str(tmp_path / "img"), str(tmp_path / "gt"), False, 1, True, 0, True, 256,
                     expected_count=None, line_file=str(tmp_path / "l.json"))


def test_write_lsq_results_matches_reference(fixture, tmp_path):
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    z, _ = fixture
    src = tmp_path / "src.json"
    src.write_bytes(z["lsq_src"].tobytes())
    for k, (ncl, ready, hor, resize, no_ortho, test_phase) in enumerate(mbg.LSQ_ARGS):
        dst = tmp_path / ("dst%d.json" % k)
        L.write_lsq_results(str(src), str(dst), ncl, ready, hor, resize, no_ortho=no_ortho, test_phase=test_phase)
        assert dst.read_bytes() == z["lsq/%d" % k].tobytes(), mbg.LSQ_ARGS[k]
    with pytest.raises(NotImplementedError):
        L.write_lsq_results(str(src), str(tmp_path / "x.json"), 4, False, False, 256, False, draw_image=True)


def test_load_valid_set_file_all_and_homography_match_reference(fixture, tmp_path, monkeypatch):
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    z, paths = fixture
    monkeypatch.chdir(paths["root"])
    target = str(tmp_path / "valid_set.json")
    L.load_valid_set_file_all(z["valid_idx/r256_flip"].tolist(), target, paths["image_dir"])
    assert open(target, "rb").read() == z["valid_set_all"].tobytes()
    for resize in (256, 320):
        np.testing.assert_array_equal(L.get_homography(resize), z["homography/%d" % resize])


def test_reference_bev_main_loader_import_resolves_to_the_package():
    """BEV/main.py:20-21 `from Dataloader.Load_Data_new import get_loader, get_homography, load_valid_set_file_all,
    write_lsq_results` with the bev directory first on sys.path."""
    code = ("import sys; sys.path.insert(0, %r);"
            "from Dataloader.Load_Data_new import get_loader, get_homography, load_valid_set_file_all, write_lsq_results;"
            "import Dataloader.Load_Data_new as m; print(m.__file__)")
    bev = os.path.join(ROOT, "lanedetection_end2end_b200", "bev")
    out = subprocess.run([sys.executable, "-c", code % bev], capture_output=True, text=True, cwd="/tmp")
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == os.path.join(bev, "Dataloader", "Load_Data_new.py")
    from lanedetection_end2end_b200.bev.Dataloader import Load_Data_new as L
    for name in ("get_loader", "LaneDataset", "get_homography", "load_valid_set_file_all", "write_lsq_results", "mirror_list",
                 "homogenous_transformation"):
        assert hasattr(L, name), name


def test_bev_loader_prototypes_match_header():
    from lanedetection_end2end_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "lanefit_b200.h")).read()
    for name in ("lf_loader_label_rows", "lf_loader_assemble_bev"):
        decl = re.search(r"int %s\((.*?)\);" % name, hdr, re.S).group(1)
        assert len(_capi.PROTOTYPES[name][1]) == len(decl.split(",")), name
        assert hasattr(_capi.lib(), name)
    assert re.search(r"#define LF_LOADER_BEV_COEFFS (\d+)", hdr).group(1) == str(_capi.LOADER_BEV_COEFFS)


def test_bev_loader_kernels_do_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "loader.cu"), "-o", str(tmp_path / "k.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    found, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = re.search(r"lf\d+(\w+?_kernel)", m.group(1)).group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            found[name] = (int(m.group(1)), int(m.group(2)))
    for k in ("loader_label_rows_kernel", "loader_assemble_bev_kernel", "loader_assemble_kernel"):
        assert found.get(k) == (0, 0), (k, found)
