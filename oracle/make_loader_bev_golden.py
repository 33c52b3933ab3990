"""Golden fixture of the bird's-eye-view loader: `python -m oracle.make_loader_bev_golden` -> tests/golden/loader_bev.npz.
TEST INFRASTRUCTURE; needs the reference checkout (oracle/reference_import.py), Pillow, torchvision and OpenCV.

It runs the reference's own BEV get_loader (Birds_Eye_View_Loss/Dataloader/Load_Data_new.py, imported unmodified with the
numpy-2 RankWarning shim) with num_workers=0 and a seeded torch RNG on a synthetic directory of 2535 unpadded file names
drawn from 1..3625 (so the string sort, the numeric sort and the positions all differ).  The names are links to the JPEG
frames of oracle/make_loader_golden.py and to three BEV label maps (Pillow L and a 4-bit palette): lanes 1..4, classes 3 / 4
above the first lane row (they must not set the horizon), values >= 5 (one map's first labelled row is one), and 1 / 2 on
both halves.  Label files: NREAL rows of the reference's Curve_parameters.json / label_new.json (a row with an all-zero lane
among them) and hand-built rows (integer-only params, -1 line entries), tiled to 3625 rows (row r = base row r % len(base)).

The reference's flip path cannot run: it calls F.hflip on the numpy label map, which torchvision rejects.  The flip-off case
runs the reference as it is; the flip-on cases run it with F.hflip shimmed to np.flip(a, 1) for arrays (PIL images still
go through F.hflip), which is what the code after that call specifies.  The shim lives here only.

Contents (everything a test needs to rebuild the directory; the reference is not needed to read it):
  jpeg/<k>, png/<k>          the distinct files; names [2535]: the file numbers; frame_of / map_of [2535]: their files
  params_jsonl, lines_jsonl  the base rows (Curve_parameters.json, label_new.json)
  valid_set_all              bytes of load_valid_set_file_all(valid_idx of r256_flip)
  homography/<resize>        get_homography(resize)
  lsq_src, lsq/<k>           a write_lsq_results input and the bytes of the reference's output for LSQ_ARGS[k]
  valid_idx/<case>
  <case>/e<epoch>/<split>/{idx,index,params,line_lst,horizon,image_sha,gt_sha,draws}  per batch, stacked
Cases: "r256_noflip", "r256_flip", "r320_flip"; num_train 46 (both splits trimmed to whole batches), batch 4, 2 epochs of
train + valid."""
import io
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_loader_golden as mlg  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "loader_bev.npz")
COUNT, MAX_NAME = 2535, 3625
NUM_TRAIN, BATCH, EPOCHS = 46, 4, 2
CASES = {"r256_noflip": (256, False, 1), "r256_flip": (256, True, 2), "r320_flip": (320, True, 3)}   # resize, flip_on, seed
NREAL = 8
# write_lsq_results(nclasses, all_branches_ready, horizon_on, resize, no_ortho, test_phase)
LSQ_ARGS = [(4, False, False, 256, False, False), (4, False, False, 256, True, False), (4, True, True, 320, False, False),
            (4, True, False, 256, True, False)]


def _ref_path():
    from oracle import reference_import as ri
    return os.path.join(ri.REFERENCE_ROOT, "Birds_Eye_View_Loss", "Dataloader", "Load_Data_new.py")


def install_loader():
    """Copy the reference's BEV Dataloader/Load_Data_new.py verbatim into oracle/_ref/ (git-ignored), so
    tools/bench_loader_bev.py can time the reference's own loader where the checkout is absent.  Called by
    __graft_entry__.build(); no-op (False) when the checkout is absent or unreadable."""
    from oracle import reference_import as ri
    src = os.path.join(ri.SOURCE_ROOT, "Birds_Eye_View_Loss", "Dataloader", "Load_Data_new.py")
    if not os.access(src, os.R_OK):
        return False
    dst = os.path.join(ri.INSTALLED_ROOT, "Birds_Eye_View_Loss", "Dataloader", "Load_Data_new.py")
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    shutil.copyfile(src, dst)
    return True


def load_reference():
    import importlib.util
    from oracle import reference_import as ri
    ri._stub_matplotlib()
    if not hasattr(np, "RankWarning"):
        np.RankWarning = np.exceptions.RankWarning
    spec = importlib.util.spec_from_file_location("_ref_bev_load_data_new", _ref_path())
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


class _HflipShim(types.ModuleType):
    """torchvision.transforms.functional, except that hflip mirrors numpy arrays along their width."""

    def __init__(self, F):
        super().__init__("F_hflip_shim")
        self._F = F

    def __getattr__(self, name):
        return getattr(self._F, name)

    def hflip(self, img):
        return np.flip(img, 1) if isinstance(img, np.ndarray) else self._F.hflip(img)


def maps():
    """Three 1280x720 BEV label maps (PNG bytes) and their arrays."""
    from oracle.make_png_golden import lane_map, pil_png
    out = []
    for k, seed in enumerate((81, 82, 83)):
        m = lane_map(720, 1280, seed)                      # 1..4 from row ~216 down; 1 / 2 on the left half
        if k == 2:
            m = np.ascontiguousarray(m[:, ::-1])           # 1 / 2 on the right half
        m[120:140, 300:340] = 3                            # classes 3 / 4 above the first lane row
        m[150:170, 800:860] = 4
        m[500:520, 900:940] = 1 if k != 2 else 2           # the other class on the other half
        m[540:560, 980:1030] = 2 if k != 2 else 1
        m[600:620, 100:140] = 7                            # values >= 5
        m[640:660, 1100:1150] = 12 if k == 1 else 250
        if k == 1:
            m[180:190, 600:640] = 9                        # the first labelled row holds a value >= 5
        out.append(m)
    png = [pil_png(out[0], compress_level=6), pil_png(out[1], "P", 16), pil_png(out[2], compress_level=1)]
    return png, out


def base_rows():
    """(Curve_parameters rows, label_new rows): NREAL real rows (one with an all-zero lane), then the edge rows."""
    from oracle import reference_import as ri
    lab = os.path.join(ri.REFERENCE_ROOT, "Birds_Eye_View_Loss", "Labels")
    rd = lambda n: [json.loads(line) for line in open(os.path.join(lab, n))]
    params, lines = rd("Curve_parameters.json"), rd("label_new.json")
    zero = [i for i, r in enumerate(params) if any(all(x == 0 for x in p) for p in r["poly_params"])]
    pick = [0, 1, 2, 1500, 3000, zero[0], zero[len(zero) // 2], 3625]
    assert len(pick) == NREAL
    P = [params[i] for i in pick]
    C = [lines[i] for i in pick]
    ints = json.loads(json.dumps(params[3]))
    ints["poly_params"] = [[0, 0, 0], [0, 0, 1], [0, -1, 0], [0, 0, 0]]        # integers only: int64 arithmetic on a flip
    P += [ints, json.loads(json.dumps(params[4]))]
    C += [{"lines": [-1] * 10}, {"lines": [-1, 0, 1, -1, -1, 1, 0, -1, 1, -1]}]
    return P, C


def build_dir(d, fr, mp, params, lines, names, frame_of, map_of):
    """The synthetic BEV directory under `d`: img/, gt/, Labels/ (links to d/files/)."""
    os.makedirs(os.path.join(d, "files"))
    for k, b in enumerate(fr):
        open(os.path.join(d, "files", "f%d.jpg" % k), "wb").write(b)
    for k, b in enumerate(mp):
        open(os.path.join(d, "files", "m%d.png" % k), "wb").write(b)
    for sub in ("img", "gt", "Labels"):
        os.makedirs(os.path.join(d, sub))
    for n, f, m in zip(names, frame_of, map_of):
        os.symlink(os.path.join(d, "files", "f%d.jpg" % f), os.path.join(d, "img", "%d.jpg" % n))
        os.symlink(os.path.join(d, "files", "m%d.png" % m), os.path.join(d, "gt", "%d.png" % n))
    T = len(params)
    for name, rows in (("Curve_parameters.json", params), ("label_new.json", lines)):
        with open(os.path.join(d, "Labels", name), "w") as f:
            for r in range(MAX_NAME):
                f.write(json.dumps(rows[r % T]) + "\n")


def from_fixture(z, d):
    """Rebuild the directory of a fixture `z` (np.load of the npz) under `d`; returns the paths the loader takes."""
    fr = [z["jpeg/%d" % k].tobytes() for k in range(int(z["n_jpeg"]))]
    mp = [z["png/%d" % k].tobytes() for k in range(int(z["n_png"]))]
    rows = lambda key: [json.loads(line) for line in z[key].tobytes().decode().splitlines()]
    build_dir(d, fr, mp, rows("params_jsonl"), rows("lines_jsonl"), z["names"], z["frame_of"], z["map_of"])
    return {"image_dir": os.path.join(d, "img"), "gt_dir": os.path.join(d, "gt"),
            "json_file": os.path.join(d, "Labels", "Curve_parameters.json"), "line_file": os.path.join(d, "Labels", "label_new.json"),
            "root": d}


def lsq_source(params):
    """A write_lsq_results input: rows with lanes, h_samples, fitted params (2 and 3 coefficients), line_id, horizon_est."""
    rng = np.random.default_rng(7)
    rows = []
    for k, r in enumerate(params[:6]):
        row = {"lanes": r["lanes"], "h_samples": r["h_samples"], "raw_file": r["raw_file"]}
        pp = [list(p) for p in r["poly_params"]]
        if k % 3 == 1:
            pp[1] = pp[1][1:]                              # two coefficients: left-padded with 0
        row["params"] = pp
        row["line_id"] = [[0, 1, 1, 1], [1, 1, 1, 0], [1, 1, 1, 1]][k % 3]
        row["horizon_est"] = rng.integers(0, 2, 40).tolist()
        if k == 2:
            row["run_time"] = 5
        rows.append(row)
    return rows


def run_reference(mod, paths, resize, flip_on, seed):
    """The reference's batches {(epoch, split): [batch tuples]}, the flip draws per (epoch, split), and valid_idx."""
    import torch
    import torchvision.transforms.functional as F
    torch.manual_seed(seed)
    train, valid, valid_idx = mod.get_loader(NUM_TRAIN, paths["json_file"], paths["image_dir"], paths["gt_dir"], flip_on, BATCH,
                                             True, 0, True, resize)
    out, draws = {}, {}
    real_uniform = np.random.uniform
    mod.F = _HflipShim(F) if flip_on else F
    try:
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
    finally:
        mod.F = F
    return out, draws, valid_idx


def main():
    params, lines = base_rows()
    fr = mlg.frames()
    mp, _ = maps()
    rng = np.random.default_rng(2535)
    names = np.sort(rng.choice(np.arange(1, MAX_NAME + 1), COUNT, replace=False)).astype(np.int32)
    frame_of = (names % len(fr)).astype(np.int32)
    map_of = ((names // 3) % len(mp)).astype(np.int32)
    jl = lambda rows: np.frombuffer("".join(json.dumps(r) + "\n" for r in rows).encode(), np.uint8)
    lsq_rows = lsq_source(params)
    z = {"n_jpeg": len(fr), "n_png": len(mp), "names": names, "frame_of": frame_of, "map_of": map_of, "params_jsonl": jl(params),
         "lines_jsonl": jl(lines), "lsq_src": jl(lsq_rows), "cases": np.array(sorted(CASES))}
    for k, b in enumerate(fr):
        z["jpeg/%d" % k] = np.frombuffer(b, np.uint8)
    for k, b in enumerate(mp):
        z["png/%d" % k] = np.frombuffer(b, np.uint8)
    mod = load_reference()
    for resize in (256, 320):
        z["homography/%d" % resize] = mod.get_homography(resize)
    cwd = os.getcwd()
    d = tempfile.mkdtemp()
    try:
        paths = from_fixture(z, d)
        os.chdir(d)                                   # the reference reads Labels/label_new.json, Labels/Curve_parameters.json
        for k, a in enumerate(LSQ_ARGS):
            src, dst = os.path.join(d, "lsq_src.json"), os.path.join(d, "lsq_dst.json")
            open(src, "wb").write(z["lsq_src"].tobytes())
            mod.write_lsq_results(src, dst, a[0], a[1], a[2], a[3], no_ortho=a[4], test_phase=a[5])
            z["lsq/%d" % k] = np.frombuffer(open(dst, "rb").read(), np.uint8)
        used_rows = set()
        for case, (resize, flip_on, seed) in sorted(CASES.items()):
            batches, draws, valid_idx = run_reference(mod, paths, resize, flip_on, seed)
            z["valid_idx/" + case] = np.array(valid_idx, np.int64)
            for (e, split), bl in batches.items():
                key = "%s/e%d/%s/" % (case, e, split)
                z[key + "idx"] = np.stack([b[3].numpy() for b in bl])
                used_rows.update(z[key + "idx"].ravel().tolist())
                if split == "valid":
                    assert all(len(b) == 7 for b in bl)
                    z[key + "index"] = np.stack([b[6].numpy() for b in bl])
                z[key + "params"] = np.stack([b[2].numpy() for b in bl])
                z[key + "line_lst"] = np.stack([b[4].numpy() for b in bl])
                z[key + "horizon"] = np.stack([b[5].numpy() for b in bl])
                z[key + "image_sha"] = np.array([mlg.digest(b[0]) for b in bl])
                z[key + "gt_sha"] = np.array([mlg.digest(b[1]) for b in bl])
                z[key + "draws"] = draws[(e, split)]
            if case == "r256_flip":
                mod.load_valid_set_file_all(valid_idx, os.path.join(d, "valid_set.json"), paths["image_dir"])
                z["valid_set_all"] = np.frombuffer(open(os.path.join(d, "valid_set.json"), "rb").read(), np.uint8)
        T = len(params)
        missing = set(range(T)) - {r % T for r in used_rows}
        assert not missing, ("base rows not reached by any batch", missing)
    finally:
        os.chdir(cwd)
        shutil.rmtree(d)
    np.savez_compressed(GOLDEN, **z)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN))


if __name__ == "__main__":
    main()
