"""Label-map decode throughput on the GPU (csrc/png.cu + LabelPreprocessor) against Pillow's label path on one host core,
and the overlap of the next batch's JPEG + PNG decode and both preprocessors with the graphed config-2 training step.
Writes profiles/h100/bench_labels.json (or --out).

    python tools/bench_labels.py [--out PATH]

Arms, all in one process with the card's name / power limit / max SM clock read at the start:
  decode   batches of 32 and 128 seeded synthetic 1280x720 label maps (oracle/make_png_golden.lane_map) written by Pillow
           (L, compress level 6), by OpenCV (8-bit gray, its default level) and by Pillow as a 4-bit palette image:
           decode + LabelPreprocessor(256, 4) in ms per batch over >= 1 s of back-to-back calls (CUDA events, after a
           warm-up), the split between the inflate launch and unfilter + label transform from torch.profiler's kernel
           times, and the host parse + blob build in us per image;
  pillow   the reference loader's label path per image on one host core (open + convert('P'), crop, NEAREST resize,
           class rules, flip, ToTensor * 255 .long()); nproc;
  overlap  the graphed config-2 step (tf32x3 and bf16) alone against the same step with the next batch's JPEG + PNG
           decode and FramePreprocessor + LabelPreprocessor on a side stream, alternated 3 times."""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def label_pngs(n, encoder):
    from oracle.make_png_golden import cv2_png, lane_map, pil_png
    out = []
    for s in range(n):
        m = lane_map(720, 1280, 2000 + s)
        if encoder == "pil_L6":
            out.append(pil_png(m, compress_level=6))
        elif encoder == "cv2":
            out.append(cv2_png(m))
        else:
            out.append(pil_png(m, "P", 16))
    return out


def time_decode(dec, pre, datas):
    import torch
    for _ in range(3):
        pre(dec(datas))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        dec.prepare(datas)
    host_us = (time.perf_counter() - t0) / 5 / len(datas) * 1e6
    calls, ms = 0, 0.0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while ms < 1000.0:
        k = max(1, 2 * calls)
        e0.record()
        for _ in range(k):
            pre(dec(datas))
        e1.record()
        torch.cuda.synchronize()
        calls, ms = k, e0.elapsed_time(e1)
    dec.check()
    return {"images_per_s": round(len(datas) * calls * 1000.0 / ms, 1), "ms_per_batch": round(ms / calls, 4),
            "host_parse_us_per_image": round(host_us, 1), "calls_timed": calls}


def split_kernels(dec, pre, datas):
    """device ms per batch of the inflate, unfilter and label-transform kernels, from torch.profiler's kernel times"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            pre(dec(datas))
        torch.cuda.synchronize()
    t = {}
    for ev in prof.key_averages():
        for name in ("png_inflate", "png_unfilter", "label_preprocess"):
            if name + "_kernel" in ev.key:
                t[name] = round(ev.device_time_total / 5 / 1000.0, 4)
    return t


def pillow_arm(datas, n=20):
    """the reference loader's label path (Load_Data_new.py:120-121,129,131,160-184) per image, flip on"""
    import torch
    from PIL import Image
    t0 = time.perf_counter()
    for d in datas[:n]:
        gt = Image.open(io.BytesIO(d)).convert("P").crop((0, 80, 1280, 720)).resize((512, 256), Image.NEAREST)
        gt = np.array(gt)
        idx3, idx4 = np.isin(gt, 3), np.isin(gt, 4)
        gt = np.flip(gt, axis=1)
        idx1, idx2 = np.isin(gt, 1), np.isin(gt, 2)
        gt[idx1], gt[idx2], gt[idx3], gt[idx4] = 2, 1, 4, 3
        gt = Image.fromarray(gt)
        (torch.from_numpy(np.array(gt, copy=True)).float().div(255)[None] * 255).long()
    return (time.perf_counter() - t0) / n * 1e3


def overlap_arm(jpegs, pngs, rounds=3, steps=30):
    import torch
    import bench
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor, LabelPreprocessor
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    from lanedetection_end2end_b200.png import PngDecoder
    cfg = bench.CONFIGS[2]
    args = bench.build_args(cfg)
    res = {}
    default = ops_net.CONV_MODE
    try:
        for mode in ("tf32x3", "bf16"):
            ops_net.set_conv_mode(mode)
            torch.manual_seed(0)
            model = Net(args)
            with contextlib.redirect_stdout(io.StringIO()):
                define_init_weights(model, "kaiming")
            model = model.cuda().train()
            crit = backprojection_loss(args)
            hx, hxgt, hvalid = bench.host_batch(cfg, 1234, pinned=False)
            g = GraphedTrainStep(model, crit, cfg["nclasses"], hx.cuda(), hxgt.cuda(), hvalid.cuda(), None, warmup=3)
            side = torch.cuda.Stream()
            resize = cfg.get("resize", 256)
            jd, pd = JpegDecoder("cuda"), PngDecoder("cuda")
            fp, lp = FramePreprocessor(resize), LabelPreprocessor(resize, cfg["nclasses"])
            jb, pb = jpegs[:cfg["batch"]], pngs[:cfg["batch"]]
            flip = torch.arange(len(jb), device="cuda") % 2 == 1
            alone, with_dec = [], []
            for _ in range(rounds):
                for arm in ("alone", "decode"):
                    for _ in range(3):
                        g()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        if arm == "decode":
                            side.wait_stream(torch.cuda.current_stream())
                            with torch.cuda.stream(side):
                                x, gt = fp(jd(jb), flip=flip), lp(pd(pb), flip=flip)
                        g()
                        if arm == "decode":
                            torch.cuda.current_stream().wait_stream(side)
                            x.record_stream(torch.cuda.current_stream())
                            gt.record_stream(torch.cuda.current_stream())
                    e1.record()
                    torch.cuda.synchronize()
                    (alone if arm == "alone" else with_dec).append(e0.elapsed_time(e1) / steps)
            jd.check()
            pd.check()
            res[mode] = {"step_ms_alone": [round(v, 3) for v in alone], "step_ms_with_decode": [round(v, 3) for v in with_dec],
                         "median_alone_ms": round(statistics.median(alone), 3),
                         "median_with_decode_ms": round(statistics.median(with_dec), 3), "batch": len(jb)}
            del g, model
    finally:
        ops_net.set_conv_mode(default)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_labels.json"))
    a = ap.parse_args()
    import torch
    from bench_decode import frames_jpeg
    from bench_modes import gpu_info
    from lanedetection_end2end_b200.input_pipeline import LabelPreprocessor
    from lanedetection_end2end_b200.png import PngDecoder
    assert torch.cuda.is_available(), "bench_labels.py times the GPU; there is no CPU fallback"
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "host_cpus_usable": len(os.sched_getaffinity(0)),
           "map": "1280x720 synthetic label map, 4 lanes of values 1-4 (oracle/make_png_golden.lane_map)", "decode": {}}
    dec, pre = PngDecoder("cuda"), LabelPreprocessor(256, 4)
    pil = None
    for enc in ("pil_L6", "cv2", "pil_P4"):
        datas = label_pngs(32, enc) * 4            # 32 distinct maps; the batch of 128 repeats them
        if enc == "pil_L6":
            pil = datas
        kb = sum(len(d) for d in datas) / len(datas) / 1024
        for n in (32, 128):
            key = "%s_b%d" % (enc, n)
            r = time_decode(dec, pre, datas[:n])
            r["kernel_ms_per_batch"] = split_kernels(dec, pre, datas[:n])
            r["mean_kb_per_map"] = round(kb, 2)
            rec["decode"][key] = r
            print(key, r, flush=True)
    rec["pillow_label_path_ms_per_image_one_core"] = round(pillow_arm(pil), 3)
    print("pillow", rec["pillow_label_path_ms_per_image_one_core"], flush=True)
    rec["overlap"] = overlap_arm(frames_jpeg(32, 75, 0), pil)
    print("overlap", rec["overlap"], flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
