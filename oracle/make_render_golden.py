"""Write tests/golden/render_testset.npz: test-set overlays drawn by the reference's own drawing lines (the im_path ...
img.save body of test_model's draw_testset branch, BP/test.py:111-121: Pillow decode, cv2.circle per point, Pillow save)
on synthetic frames.  CPU only; needs the reference checkout (oracle/reference_import.py) and cv2.

    python -m oracle.make_render_golden [--out tests/golden/render_testset.npz]

The lines are taken out of the reference's test_model with ast and run unmodified in a namespace that holds what the loop
has at that point (json_line, lanes_to_write, im_id, args, colormap, and the reference module's np / cv2 / Image / os).
The branch's first lines, which save the weight-map image {im_id}_vis.jpg, are not run: Pillow cannot write that float
image as a JPEG.

Contents (K frames of 1280x720):
  rows_json    uint8, the K ground-truth rows as UTF-8 JSON lines (raw_file, h_samples)
  frame{k}     uint8, the JPEG file of frame k (Pillow, quality 75)
  lanes        [K, 4, S] int32, the lanes drawn (-2 = no point); h_samples [K, S] int32
  overlay{k}   uint8, the JPEG file the reference writes for frame k
"""
import argparse
import ast
import io
import json
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

H, W = 720, 1280
S = 56
TUSIMPLE_ROWS = list(range(160, 720, 10))


def reference_draw_lines():
    """(colormap statement, drawing statements) of the reference's test_model, compiled from its source."""
    from oracle import reference_import as ri
    path = os.path.join(ri.REFERENCE_ROOT, "Backprojection_Loss", "test.py")
    with open(path) as f:
        tree = ast.parse(f.read(), path)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "test_model")
    cmap = next(n for n in fn.body if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", None) == "colormap")
    branch = next(n for n in ast.walk(fn) if isinstance(n, ast.If) and ast.unparse(n.test) == "args.draw_testset")
    start = next(i for i, n in enumerate(branch.body) if isinstance(n, ast.Assign) and getattr(n.targets[0], "id", None) == "im_path")
    mod = lambda nodes: compile(ast.fix_missing_locations(ast.Module(body=nodes, type_ignores=[])), path, "exec")
    return mod([cmap]), mod(branch.body[start:])


def make_frame(k):
    """A road-like synthetic frame: smooth gradients, a few soft blobs and faint seeded noise."""
    rng = np.random.default_rng(100 + k)
    y, x = np.mgrid[:H, :W].astype(np.float64)
    img = np.stack([60 + 80 * y / H + 20 * np.sin(x / (90 + 20 * k)), 70 + 60 * y / H + 15 * np.cos(y / 70),
                    90 + 40 * (1 - y / H) + 10 * np.sin((x + y) / 150)], -1)
    for _ in range(6):
        cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(30, 150)
        img += rng.uniform(-40, 40, 3) * np.exp(-((y - cy) ** 2 + (x - cx) ** 2) / (2 * r * r))[..., None]
    img += rng.normal(0, 0.5, img.shape)
    return np.clip(np.round(img), 0, 255).astype(np.uint8)


def make_lanes(k, rng):
    """Lanes of frame k: straight lanes with gaps, overlapping neighbours, and points at and past the frame borders."""
    if k < 2:
        h = list(TUSIMPLE_ROWS)
    else:   # rows at the top and bottom borders and past them
        h = [0, 1, 2, 3, 715, 716, 717, 718, 719, 720, 722, -1, -3] + list(range(40, 40 + 10 * (S - 13), 10))
    y = np.asarray(h, np.float64)
    lanes = np.full((4, S), -2, np.int64)
    for j in range(4):
        x = 200 + 300 * j + (j - 1.5) * 0.8 * (y - 160) + rng.normal(0, 1.5, S)
        lanes[j] = np.round(x)
        lanes[j, rng.random(S) < 0.15] = -2
    if k == 0:      # lane 1 overlaps lane 0 on a stretch: lane 1's stamps win there
        lanes[1, 10:30] = lanes[0, 10:30] + rng.integers(-4, 5, 20)
    if k == 1:      # points at the left and right borders and beyond them
        lanes[0, :12] = [0, 1, 2, 3, -1, -3, -4, 0, 1, -2, 2, 0]
        lanes[3, :12] = [1279, 1278, 1277, 1276, 1280, 1282, 1283, 1279, 1278, -2, 1277, 1279]
        lanes[2, 20:40] = lanes[3, 20:40] + 2
    if k == 2:      # the corners
        lanes[0, :6] = [0, 1279, 2, 1277, 0, 1279]
        lanes[3, 4:11] = [0, 1279, 3, 1276, 0, 1279, 1]
    return h, lanes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "render_testset.npz"))
    a = ap.parse_args()
    import cv2
    from PIL import Image
    cmap_code, draw_code = reference_draw_lines()
    rng = np.random.default_rng(2026)
    out, rows, lanes_all, h_all = {}, [], [], []
    with tempfile.TemporaryDirectory() as d:
        test_dir, save_path = os.path.join(d, "test"), os.path.join(d, "save")
        os.makedirs(os.path.join(test_dir, "clips"))
        os.makedirs(os.path.join(save_path, "example", "testset"))
        args = types.SimpleNamespace(test_dir=test_dir, save_path=save_path, draw_testset=True)
        for k in range(a.frames):
            bio = io.BytesIO()
            Image.fromarray(make_frame(k)).save(bio, "JPEG", quality=75)
            raw = "clips/%d.jpg" % k
            with open(os.path.join(test_dir, raw), "wb") as f:
                f.write(bio.getvalue())
            h, lanes = make_lanes(k, rng)
            row = {"raw_file": raw, "h_samples": h}
            ns = {"np": np, "cv2": cv2, "Image": Image, "os": os}
            exec(cmap_code, ns)
            ns.update(json_line=dict(row, lanes=lanes.tolist()), lanes_to_write=lanes.tolist(), im_id=k, args=args)
            exec(draw_code, ns)
            with open(os.path.join(save_path, "example", "testset", "%d.jpg" % k), "rb") as f:
                out["overlay%d" % k] = np.frombuffer(f.read(), np.uint8)
            out["frame%d" % k] = np.frombuffer(bio.getvalue(), np.uint8)
            rows.append(row)
            lanes_all.append(lanes)
            h_all.append(h)
    text = "".join(json.dumps(r) + "\n" for r in rows)
    np.savez_compressed(a.out, rows_json=np.frombuffer(text.encode(), np.uint8), lanes=np.asarray(lanes_all, np.int32),
                        h_samples=np.asarray(h_all, np.int32), **out)
    print("wrote %s: %d frames, %.1f kB" % (a.out, a.frames, os.path.getsize(a.out) / 1024))


if __name__ == "__main__":
    main()
