"""Benchmark the GPU JPEG encoder (ops.jpeg.JpegEncodePlan, csrc/jpeg_encode.cu) on the files of the extraction step; prints
one JSON line.  Workloads, each one call:

  flow_L      the 512 x / y planes of the TV-L1 benchmark's 256-pair call, 340 x 256 'L' (flow-like planes), quality 95
  rgb_340     256 RGB frames at 340 x 256 (smooth textures), quality 95
  rgb_480     400 RGB frames at 480 x 360, quality 95

Per workload: the median and range of CUDA-event times over --windows windows of --calls calls after warm-up, images per
second, the device time per kernel from torch.profiler in a separate call, the bytes read (pixels) and written (files)
computed from shapes and lengths with their share of 3.35 TB/s HBM, and Pillow on one host core (--pillow images, timed
one by one) as the CPU column.  The card's name and power limit are read in the same run.  Needs a CUDA device.

    python tools/bench_jpeg_encode.py
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM = 3.35e12
WORKLOADS = (("flow_L", "L", 512, 256, 340), ("rgb_340", "RGB", 256, 256, 340), ("rgb_480", "RGB", 400, 360, 480))


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def images(mode, n, h, w, distinct=16):
    """n images of `distinct` seeded contents: flow-like planes for 'L', smooth textures for 'RGB'"""
    from oracle import jpeg_encode_oracle as E
    from oracle import tvl1_oracle as T
    if mode == "L":
        base = np.stack([E.fixture("flow", h, w, 1, s) for s in range(distinct)])
    else:
        ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
        base = np.stack([np.clip(np.rint(np.stack([T.texture(xs + s, ys - s, seed=3 * s + c, waves=6) for c in range(3)], -1)), 0, 255)
                         for s in range(distinct)]).astype(np.uint8)
    return base[np.arange(n) % distinct]


def pillow_s_per_image(arr, mode, count):
    from PIL import Image
    t = []
    for i in range(count):
        im = Image.fromarray(arr[i, ..., 0] if mode == "L" else arr[i], mode)
        t0 = time.perf_counter()
        im.save(io.BytesIO(), format="JPEG", quality=95)
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pillow", type=int, default=32)
    a = ap.parse_args()
    import torch
    from ops.jpeg import JpegEncodePlan
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_encode needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card_info()}
    for name, mode, n, h, w in WORKLOADS:
        arr = images(mode, n, h, w)
        x = torch.from_numpy(arr).to(dev)
        plan = JpegEncodePlan([(h, w)] * n, mode, 95, dev)
        for _ in range(a.warmup):
            plan.run(x)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.calls):
                plan.run(x)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3 / a.calls)
        t = float(np.median(times))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            plan.run(x)
            torch.cuda.synchronize()
        stage = {}
        for ev in prof.key_averages():
            if "enc_" in ev.key and "_kernel" in ev.key:
                k = ev.key.split("enc_")[1].split("_kernel")[0]
                stage[k] = round(stage.get(k, 0.0) + ev.device_time_total / 1e3, 3)
        lens = plan.lengths.cpu().numpy()
        read, written = int(arr.nbytes), int(lens.sum())
        cpu = pillow_s_per_image(arr, mode, min(a.pillow, n))
        res[name] = {"workload": "%d %s images of %dx%d (W x H), quality 95" % (n, mode, w, h), "s_per_call": round(t, 5),
                     "s_range": [round(min(times), 5), round(max(times), 5)], "images_per_s": round(n / t, 1), "stage_ms": stage,
                     "bytes_read": read, "bytes_written": written, "mean_file_bytes": round(written / n, 1),
                     "hbm_share": round((read + written) / t / HBM, 4), "pillow_1core_s_per_image": round(cpu, 6),
                     "pillow_1core_images_per_s": round(1.0 / cpu, 1)}
        del plan, x
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
