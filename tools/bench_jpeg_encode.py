"""JPEG encode on the GPU (csrc/jpeg_enc.cu) against Pillow on one host core, and inference.render_testset against the
reference's host drawing loop.  Writes profiles/h100/bench_jpeg_encode.json (or --out).

    python tools/bench_jpeg_encode.py [--out PATH] [--frames 2782] [--host-frames 300]

Arms, all in one process with the card's name / power limit / max SM clock read at the start:
  encode   batches of 32 and 128 synthetic 1280x720 frames (oracle/make_jpeg_golden.make_frame) at q75 and q95, 4:2:0:
           device ms per batch over >= 1 s of back-to-back encode_async calls (CUDA events, after a warm-up; the number of
           calls is recorded), the split between the four kernels from torch.profiler, and the mean file size;
  pillow   Image.fromarray(a).save(buf, "JPEG", quality=q) per frame on one host core, at q75 and q95;
  render   render_testset over --frames synthetic test frames (32 distinct 1280x720 JPEGs under distinct names, four seeded
           lanes each, batches of 32): wall time including the file reads and writes, against the host loop of the
           reference (Pillow decode, cv2.circle per point, Pillow save) over the first --host-frames of them."""
import argparse
import io
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def synthetic_frames(n):
    from oracle.make_jpeg_golden import make_frame
    return np.stack([make_frame(720, 1280, 1000 + s) for s in range(n)])


def time_encode(enc, frames):
    import torch
    for _ in range(3):
        enc.encode_async(frames)
    torch.cuda.synchronize()
    calls, ms = 0, 0.0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while ms < 1000.0:
        k = max(1, 2 * calls)
        e0.record()
        for _ in range(k):
            enc.encode_async(frames)
        e1.record()
        torch.cuda.synchronize()
        calls, ms = k, e0.elapsed_time(e1)
    _, _, lengths = enc.encode_async(frames)
    return {"ms_per_batch": round(ms / calls, 4), "images_per_s": round(frames.shape[0] * calls * 1000.0 / ms, 1),
            "calls_timed": calls, "mean_kb_per_file": round(float(lengths.double().mean()) / 1024, 1)}


def kernel_split(enc, frames):
    """device ms per batch of each kernel, from torch.profiler's kernel times"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            enc.encode_async(frames)
        torch.cuda.synchronize()
    t = {}
    for ev in prof.key_averages():
        if "enc_" in ev.key and "_kernel" in ev.key:
            name = ev.key.split("enc_")[1].split("_kernel")[0]
            t[name] = round(ev.device_time_total / 5 / 1000.0, 4)
    return t


def pillow_arm(frames, q):
    from PIL import Image
    t0 = time.perf_counter()
    for a in frames:
        Image.fromarray(a).save(io.BytesIO(), "JPEG", quality=q)
    return (time.perf_counter() - t0) / len(frames) * 1e3


def render_arm(n_frames, host_frames, frames):
    import cv2
    import torch
    from PIL import Image
    from lanedetection_end2end_b200.inference import COLORMAP, render_testset
    rng = np.random.default_rng(5)
    h = list(range(160, 720, 10))
    y = np.asarray(h, np.float64)
    lanes = np.full((n_frames, 4, 56), -2, np.int32)
    for j in range(4):
        x = 250 + 260 * j + (j - 1.5) * (0.6 + 0.4 * rng.random((n_frames, 1))) * (y - 160) + rng.normal(0, 2, (n_frames, 56))
        lanes[:, j] = np.where((x >= 0) & (x <= 1279) & (rng.random((n_frames, 56)) > 0.1), np.round(x), -2)
    datas = []
    for a in frames:
        bio = io.BytesIO()
        Image.fromarray(a).save(bio, "JPEG", quality=90)
        datas.append(bio.getvalue())
    with tempfile.TemporaryDirectory() as d:
        rows = []
        for i in range(n_frames):
            raw = "clips/%d/20.jpg" % i
            os.makedirs(os.path.join(d, "test", os.path.dirname(raw)), exist_ok=True)
            with open(os.path.join(d, "test", raw), "wb") as f:
                f.write(datas[i % len(datas)])
            rows.append({"raw_file": raw, "h_samples": h})
        dl = torch.from_numpy(lanes).cuda()
        render_testset(dl[:64], rows[:64], os.path.join(d, "test"), os.path.join(d, "warm"))     # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        render_testset(dl, rows, os.path.join(d, "test"), os.path.join(d, "gpu"))
        gpu_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        for i in range(host_frames):
            with open(os.path.join(d, "test", rows[i]["raw_file"]), "rb") as f:
                img = np.array(Image.open(f).convert("RGB"))
            for l, lane in enumerate(lanes[i].tolist()):
                for x, yy in zip(lane, h):
                    if x != -2:
                        img = cv2.circle(img, (x, yy), thickness=-1, color=COLORMAP[l], radius=3)
            Image.fromarray(np.uint8(img)).save(os.path.join(d, "host_%d.jpg" % i))
        host_s = time.perf_counter() - t0
        same = all(open(os.path.join(d, "gpu", "%d.jpg" % i), "rb").read() == open(os.path.join(d, "host_%d.jpg" % i), "rb").read()
                   for i in range(host_frames))
    return {"frames": n_frames, "batch": 32, "gpu_wall_s": round(gpu_s, 3), "gpu_ms_per_frame": round(gpu_s / n_frames * 1e3, 3),
            "host_frames": host_frames, "host_wall_s": round(host_s, 3), "host_ms_per_frame": round(host_s / host_frames * 1e3, 3),
            "files_identical_on_host_frames": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_jpeg_encode.json"))
    ap.add_argument("--frames", type=int, default=2782)
    ap.add_argument("--host-frames", type=int, default=300)
    a = ap.parse_args()
    import torch
    from bench_modes import gpu_info
    from lanedetection_end2end_b200.jpeg import JpegEncoder
    assert torch.cuda.is_available(), "bench_jpeg_encode.py times the GPU; there is no CPU fallback"
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "frame": "1280x720 synthetic (oracle/make_jpeg_golden.make_frame), 4:2:0",
           "encode": {}, "pillow_ms_per_frame_one_core": {}}
    frames = synthetic_frames(32)
    dev = torch.from_numpy(np.concatenate([frames] * 4)).cuda()      # the batch of 128 repeats the 32 frames
    for q in (75, 95):
        enc = JpegEncoder("cuda", quality=q)
        for n in (32, 128):
            key = "q%d_b%d" % (q, n)
            r = time_encode(enc, dev[:n])
            r["kernel_ms_per_batch"] = kernel_split(enc, dev[:n])
            rec["encode"][key] = r
            print(key, r, flush=True)
        rec["pillow_ms_per_frame_one_core"]["q%d" % q] = round(pillow_arm(frames, q), 3)
    print("pillow", rec["pillow_ms_per_frame_one_core"], flush=True)
    rec["render"] = render_arm(a.frames, a.host_frames, frames)
    print("render", rec["render"], flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
