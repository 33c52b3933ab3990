"""JPEG decode throughput on the GPU (csrc/jpeg.cu) against Pillow on one host core, and the overlap of the next batch's
decode + preprocess with the graphed config-2 training step.  Writes profiles/h100/bench_decode.json (or --out).

    python tools/bench_decode.py [--out PATH]

Arms, all in one process with the card's name / power limit / max SM clock read at the start:
  decode   batches of 32 and 128 synthetic 1280x720 4:2:0 frames (oracle/make_jpeg_golden.make_frame) at q75 / q90, with
           and without restart markers: images/s over >= 1 s of back-to-back calls (CUDA events, after a warm-up), the
           split between launch 1 (entropy decode) and launches 2-3 (IDCT, upsample + colour) from a per-launch event
           trace, and the host parse + blob build in us per image;
  pillow   Image.open().convert('RGB') + crop + BILINEAR resize per image on one host core; nproc;
  overlap  the graphed config-2 step (tf32x3 and bf16) alone against the same step with the next batch's decode +
           FramePreprocessor on a side stream, alternated 3 times."""
import argparse
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def frames_jpeg(n, q, restart_rows):
    from PIL import Image
    from oracle.make_jpeg_golden import make_frame
    out = []
    for s in range(n):
        kw = {"quality": q, "subsampling": 2}
        if restart_rows:
            kw["restart_marker_rows"] = restart_rows
        bio = io.BytesIO()
        Image.fromarray(make_frame(720, 1280, 1000 + s)).save(bio, "JPEG", **kw)
        out.append(bio.getvalue())
    return out


def time_decode(dec, datas):
    import torch
    from lanedetection_end2end_b200 import _capi
    for _ in range(3):
        dec(datas)
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
            dec(datas)
        e1.record()
        torch.cuda.synchronize()
        calls, ms = k, e0.elapsed_time(e1)
    _capi.TRACE = []      # one traced call: events around lf_jpeg_decode (the pinned copy is outside them)
    dec(datas)
    torch.cuda.synchronize()
    whole = _capi.TRACE[0][1].elapsed_time(_capi.TRACE[0][2])
    _capi.TRACE = None
    dec.check()
    return {"images_per_s": round(len(datas) * calls * 1000.0 / ms, 1), "ms_per_batch": round(ms / calls, 4),
            "host_parse_us_per_image": round(host_us, 1), "traced_call_ms": round(whole, 4), "calls_timed": calls}


def split_entropy(dec, datas):
    """device ms per batch of each of the three kernels (entropy, idct, color), from torch.profiler's kernel times"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            dec(datas)
        torch.cuda.synchronize()
    t = {}
    for ev in prof.key_averages():
        if "jpeg_" in ev.key:
            name = ev.key.split("jpeg_")[1].split("_kernel")[0]
            t[name] = round(ev.device_time_total / 5 / 1000.0, 4)
    return t


def pillow_arm(datas, n=20):
    from PIL import Image
    t0 = time.perf_counter()
    for d in datas[:n]:
        Image.open(io.BytesIO(d)).convert("RGB").crop((0, 80, 1280, 720)).resize((512, 256), Image.BILINEAR)
    return (time.perf_counter() - t0) / n * 1e3


def overlap_arm(datas, rounds=3, steps=30):
    import contextlib
    import torch
    import bench
    from lanedetection_end2end_b200 import ops_net
    from lanedetection_end2end_b200.Networks.LSQ_layer import Net
    from lanedetection_end2end_b200.Networks.utils import define_init_weights
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.input_pipeline import FramePreprocessor
    from lanedetection_end2end_b200.jpeg import JpegDecoder
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
            dec, pre = JpegDecoder("cuda"), FramePreprocessor(cfg.get("resize", 256))
            batch = datas[:cfg["batch"]]
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
                                nxt = pre(dec(batch))
                        g()
                        if arm == "decode":
                            torch.cuda.current_stream().wait_stream(side)
                            nxt.record_stream(torch.cuda.current_stream())
                    e1.record()
                    torch.cuda.synchronize()
                    (alone if arm == "alone" else with_dec).append(e0.elapsed_time(e1) / steps)
            dec.check()
            res[mode] = {"step_ms_alone": [round(v, 3) for v in alone], "step_ms_with_decode": [round(v, 3) for v in with_dec],
                         "median_alone_ms": round(statistics.median(alone), 3),
                         "median_with_decode_ms": round(statistics.median(with_dec), 3), "batch": len(batch)}
            del g, model
    finally:
        ops_net.set_conv_mode(default)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100", "bench_decode.json"))
    a = ap.parse_args()
    import torch
    from bench_modes import gpu_info
    from lanedetection_end2end_b200.jpeg import JpegDecoder
    assert torch.cuda.is_available(), "bench_decode.py times the GPU; there is no CPU fallback"
    rec = {"gpu": gpu_info(), "nproc": os.cpu_count(), "frame": "1280x720 4:2:0 synthetic (oracle/make_jpeg_golden.make_frame)",
           "decode": {}}
    dec = JpegDecoder("cuda")
    q75 = None
    for q in (75, 90):
        for rst in (0, 2):
            datas = frames_jpeg(32, q, rst) * 4      # 32 distinct frames; the batch of 128 repeats them
            if q == 75 and rst == 0:
                q75 = datas
            kb = sum(len(d) for d in datas) / len(datas) / 1024
            for n in (32, 128):
                key = "q%d_%s_b%d" % (q, "rst2rows" if rst else "norst", n)
                r = time_decode(dec, datas[:n])
                r["kernel_ms_per_batch"] = split_entropy(dec, datas[:n])
                r["mean_kb_per_frame"] = round(kb, 1)
                rec["decode"][key] = r
                print(key, r, flush=True)
    rec["pillow_ms_per_image_one_core"] = round(pillow_arm(q75), 3)
    print("pillow", rec["pillow_ms_per_image_one_core"], flush=True)
    rec["overlap"] = overlap_arm(q75)
    print("overlap", rec["overlap"], flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
