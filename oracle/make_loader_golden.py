"""Golden fixture of the TuSimple loader: `python -m oracle.make_loader_golden` -> tests/golden/loader_tusimple.npz.
TEST INFRASTRUCTURE; needs the reference checkout (oracle/reference_import.py), Pillow, torchvision and OpenCV.

It runs the reference's own get_loader and get_testloader (BP/Dataloader/Load_Data_new.py, imported unmodified with the
numpy-2 RankWarning shim and the matplotlib stub) with num_workers=0 and a seeded torch RNG on a synthetic directory of
3626 unpadded file names ("1.jpg" .. "3626.jpg", so the string sort differs from the numeric one).  The names are links to a
handful of distinct synthetic 1280x720 JPEG frames (4:2:0, 4:2:2, 4:4:4, grayscale) and PNG label maps (Pillow L, 4-bit
palette).  Label files: NREAL rows of the reference's lanes_ordered.json / label_new.json (48- and 56-sample rows, row 0
among them) and hand-built edge rows (a point at x = 0, no lanes, -1 line entries), tiled to 3626 rows (row r = base row
r % len(base)).

Contents (everything a test needs to rebuild the directory; the reference is not needed to read it):
  jpeg/<k>, png/<k>          the distinct files; frame_of / map_of [3626]: file of name n + 1
  lanes_jsonl, lines_jsonl, all_jsonl   the base rows (lanes_ordered.json, label_new.json, label_data_all.json)
  test_jsonl                 test_label.json (10 rows), test_frame_of [10]
  valid_set_all              bytes of load_valid_set_file_all(valid_idx of case 0) ; valid_idx/<case>
  <case>/e<epoch>/<split>/{idx,index,lanes,valid_points,horizon,line_lst,image_sha,gt_sha,draws}  per batch, stacked
  <case>/test/image_sha      per test batch
Cases: "r256_c4", "r256_c2", "r320_c4" (resize / nclasses), flip on, num_train 40, batch 4, 2 epochs of train + valid."""
import hashlib
import io
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "loader_tusimple.npz")
COUNT = 3626
NUM_TRAIN, BATCH, EPOCHS = 40, 4, 2
CASES = {"r256_c4": (256, 4, 1), "r256_c2": (256, 2, 2), "r320_c4": (320, 4, 3)}     # resize, nclasses, torch seed
NREAL = 8
NTEST = 10


def install_loader():
    """Copy the reference's Dataloader/Load_Data_new.py verbatim into oracle/_ref/ (git-ignored), so tools/bench_loader.py
    can time the reference's own loader where the checkout is absent.  Called by __graft_entry__.build(); no-op (False) when
    the checkout is absent or unreadable."""
    from oracle import reference_import as ri
    src = os.path.join(ri.SOURCE_ROOT, "Backprojection_Loss", "Dataloader", "Load_Data_new.py")
    if not os.access(src, os.R_OK):
        return False
    dst = os.path.join(ri.INSTALLED_ROOT, "Backprojection_Loss", "Dataloader", "Load_Data_new.py")
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    shutil.copyfile(src, dst)
    return True


def frames():
    """Distinct synthetic JPEG frames: smooth road-like gradients with bright lane stripes and some texture."""
    from PIL import Image
    out = []
    yy, xx = np.mgrid[0:720, 0:1280].astype(np.float64)
    for k, (mode, sub) in enumerate((("RGB", 2), ("RGB", 1), ("RGB", 0), ("L", None))):
        rng = np.random.default_rng(100 + k)
        img = np.stack([60 + 80 * yy / 720 + 20 * np.sin(xx / (37 + 9 * k)), 70 + 60 * xx / 1280, 90 + 40 * np.cos(yy / 53)], -1)
        for j in range(4):
            cx = 640 + (xx - 640) * 0 + (200 + 250 * j - 640) * (yy - 250) / 470
            img[(np.abs(xx - cx) < 3 + 6 * (yy - 250) / 470) & (yy > 260 + 10 * k)] = 235
        img += rng.normal(0, 6, img.shape)
        a = np.clip(img, 0, 255).astype(np.uint8)
        im = Image.fromarray(a) if mode == "RGB" else Image.fromarray(a[..., 1])
        bio = io.BytesIO()
        if sub is None:
            im.save(bio, "JPEG", quality=80)
        else:
            im.save(bio, "JPEG", quality=80, subsampling=sub)
        out.append(bio.getvalue())
    return out


def maps():
    from oracle.make_png_golden import lane_map, pil_png
    a, b, c = lane_map(720, 1280, 71), lane_map(720, 1280, 72), lane_map(720, 1280, 73)
    return [pil_png(a, compress_level=6), pil_png(b, "P", 16), pil_png(c, compress_level=1)]


def base_rows():
    """(lanes_ordered rows, label_new rows, label_data_all rows): NREAL real rows, then the edge rows."""
    from oracle import reference_import as ri
    lab = os.path.join(ri.REFERENCE_ROOT, "Backprojection_Loss", "Labels")
    rd = lambda n: [json.loads(line) for line in open(os.path.join(lab, n))]
    lanes, lines, alls = rd("lanes_ordered.json"), rd("label_new.json"), rd("label_data_all.json")
    s56 = [i for i, r in enumerate(lanes) if len(r["h_samples"]) == 56]
    pick = [0, 1, 2, 1500] + s56[:2] + s56[200:202]                # row 0 and three other 48-sample rows, four 56-sample rows
    assert len(pick) == NREAL
    L = [lanes[i] for i in pick]
    C = [lines[i] for i in pick]
    A = [alls[i] for i in pick]
    hs56 = lanes[s56[0]]["h_samples"]
    x0 = json.loads(json.dumps(lanes[s56[0]]))                      # a point at x = 0 (valid, and one in the first 8)
    x0["lanes"][1][20] = 0
    x0["lanes"][2][3] = 0
    none = {"lanes": [[-2] * 56 for _ in range(4)], "h_samples": hs56}   # no lanes: horizon = resize
    neg = json.loads(json.dumps(lanes[s56[1]]))
    L += [x0, none, neg]
    C += [{"lines": [0, 1, 1, 0, 1, 0, 1, 1, 0, 0]}, {"lines": [-1] * 10}, {"lines": [-1, 0, 1, -1, -1, 1, 0, -1, 1, -1]}]
    A += [alls[s56[0]], alls[s56[3]], alls[s56[1]]]
    return L, C, A


def build_dir(d, fr, mp, lanes, lines, alls, test_rows, frame_of, map_of, test_frame_of):
    """The synthetic TuSimple directory under `d`: img/, gt/, Labels/, test/ (links to d/files/)."""
    os.makedirs(os.path.join(d, "files"))
    for k, b in enumerate(fr):
        open(os.path.join(d, "files", "f%d.jpg" % k), "wb").write(b)
    for k, b in enumerate(mp):
        open(os.path.join(d, "files", "m%d.png" % k), "wb").write(b)
    for sub in ("img", "gt", "Labels", "test/clips"):
        os.makedirs(os.path.join(d, sub))
    for n in range(1, COUNT + 1):
        os.symlink(os.path.join(d, "files", "f%d.jpg" % frame_of[n - 1]), os.path.join(d, "img", "%d.jpg" % n))
        os.symlink(os.path.join(d, "files", "m%d.png" % map_of[n - 1]), os.path.join(d, "gt", "%d.png" % n))
    T = len(lanes)
    for name, rows in (("lanes_ordered.json", lanes), ("label_new.json", lines), ("label_data_all.json", alls)):
        with open(os.path.join(d, "Labels", name), "w") as f:
            for r in range(COUNT):
                f.write(json.dumps(rows[r % T]) + "\n")
    open(os.path.join(d, "Labels", "params.json"), "w").write("{}\n")
    with open(os.path.join(d, "test", "test_label.json"), "w") as f:
        for k, row in enumerate(test_rows):
            os.symlink(os.path.join(d, "files", "f%d.jpg" % test_frame_of[k]), os.path.join(d, "test", row["raw_file"]))
            f.write(json.dumps(row) + "\n")


def from_fixture(z, d):
    """Rebuild the directory of a fixture `z` (np.load of the npz) under `d`; returns the paths the loaders take."""
    fr = [z["jpeg/%d" % k].tobytes() for k in range(int(z["n_jpeg"]))]
    mp = [z["png/%d" % k].tobytes() for k in range(int(z["n_png"]))]
    rows = lambda key: [json.loads(line) for line in z[key].tobytes().decode().splitlines()]
    build_dir(d, fr, mp, rows("lanes_jsonl"), rows("lines_jsonl"), rows("all_jsonl"), rows("test_jsonl"), z["frame_of"],
              z["map_of"], z["test_frame_of"])
    return {"image_dir": os.path.join(d, "img"), "gt_dir": os.path.join(d, "gt"), "json_file": os.path.join(d, "Labels", "params.json"),
            "lanes_file": os.path.join(d, "Labels", "lanes_ordered.json"), "line_file": os.path.join(d, "Labels", "label_new.json"),
            "test_dir": os.path.join(d, "test")}


def digest(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().cpu().numpy()).tobytes()).hexdigest()


def load_reference():
    import importlib.util
    from oracle import reference_import as ri
    ri._stub_matplotlib()
    if not hasattr(np, "RankWarning"):
        np.RankWarning = np.exceptions.RankWarning
    path = os.path.join(ri.REFERENCE_ROOT, "Backprojection_Loss", "Dataloader", "Load_Data_new.py")
    spec = importlib.util.spec_from_file_location("_ref_load_data_new", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def run_reference(mod, paths, resize, nclasses, seed):
    """The reference's batches: {(epoch, split): [batch tuples]}, the flip draws per (epoch, split), valid_idx, test batches."""
    import torch
    torch.manual_seed(seed)
    train, valid, valid_idx = mod.get_loader(NUM_TRAIN, paths["json_file"], paths["lanes_file"], paths["image_dir"], paths["gt_dir"],
                                             True, BATCH, BATCH, True, 0, True, resize, nclasses)
    out, draws = {}, {}
    real_uniform = np.random.uniform
    for e in range(EPOCHS):
        for split, loader in (("train", train), ("valid", valid)):
            rec = []

            def uniform(*a, **k):
                v = real_uniform(*a, **k)
                rec.append(v)
                return v
            np.random.uniform = uniform
            try:
                out[(e, split)] = [b for b in loader]
            finally:
                np.random.uniform = real_uniform
            draws[(e, split)] = np.array(rec, np.float64)
    test = [b for b in mod.get_testloader(paths["test_dir"], BATCH, 0, resize=resize)]
    return out, draws, valid_idx, test


def main():
    lanes, lines, alls = base_rows()
    fr, mp = frames(), maps()
    frame_of = np.array([n % len(fr) for n in range(1, COUNT + 1)], np.int32)
    map_of = np.array([(n // 3) % len(mp) for n in range(1, COUNT + 1)], np.int32)
    test_rows = [{"raw_file": "clips/%d.jpg" % k, "lanes": lanes[4 + k % 4]["lanes"], "h_samples": lanes[4 + k % 4]["h_samples"]}
                 for k in range(NTEST)]
    test_frame_of = np.array([(3 * k + 1) % len(fr) for k in range(NTEST)], np.int32)
    jl = lambda rows: np.frombuffer("".join(json.dumps(r) + "\n" for r in rows).encode(), np.uint8)
    z = {"n_jpeg": len(fr), "n_png": len(mp), "frame_of": frame_of, "map_of": map_of, "lanes_jsonl": jl(lanes),
         "lines_jsonl": jl(lines), "all_jsonl": jl(alls), "test_jsonl": jl(test_rows), "test_frame_of": test_frame_of,
         "cases": np.array(sorted(CASES))}
    for k, b in enumerate(fr):
        z["jpeg/%d" % k] = np.frombuffer(b, np.uint8)
    for k, b in enumerate(mp):
        z["png/%d" % k] = np.frombuffer(b, np.uint8)
    mod = load_reference()
    cwd = os.getcwd()
    d = tempfile.mkdtemp()
    try:
        paths = from_fixture(z, d)
        os.chdir(d)                                   # the reference reads Labels/label_new.json, Labels/label_data_all.json
        used_rows = set()
        for case, (resize, nclasses, seed) in sorted(CASES.items()):
            batches, draws, valid_idx, test = run_reference(mod, paths, resize, nclasses, seed)
            z["valid_idx/" + case] = np.array(valid_idx, np.int64)
            for (e, split), bl in batches.items():
                key = "%s/e%d/%s/" % (case, e, split)
                val = split == "valid"
                z[key + "idx"] = np.stack([b[3].numpy() for b in bl])
                used_rows.update(z[key + "idx"].ravel().tolist())
                if val:
                    z[key + "index"] = np.stack([b[6].numpy() for b in bl])
                z[key + "lanes"] = np.stack([b[2].numpy() for b in bl])
                z[key + "line_lst"] = np.stack([b[4].numpy() for b in bl])
                z[key + "horizon"] = np.stack([b[5].numpy() for b in bl])
                z[key + "valid_points"] = np.stack([b[-1].numpy() for b in bl])
                z[key + "image_sha"] = np.array([digest(b[0]) for b in bl])
                z[key + "gt_sha"] = np.array([digest(b[1]) for b in bl])
                z[key + "draws"] = draws[(e, split)]
                assert all(b[0].dtype.is_floating_point and b[1].dtype == __import__("torch").int64 for b in bl)
            z[case + "/test/image_sha"] = np.array([digest(b) for b in test])
            z[case + "/test/shape"] = np.array([tuple(b.shape) for b in test])
            if case == "r256_c4":
                mod.load_valid_set_file_all(valid_idx, os.path.join(d, "valid_set.json"), paths["image_dir"])
                z["valid_set_all"] = np.frombuffer(open(os.path.join(d, "valid_set.json"), "rb").read(), np.uint8)
        T = len(lanes)
        missing = set(range(T)) - {r % T for r in used_rows}
        assert not missing, ("base rows not reached by any batch", missing)
    finally:
        os.chdir(cwd)
        shutil.rmtree(d)
    np.savez_compressed(GOLDEN, **z)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
