"""JPEG decode on the GPU (ops/jpeg.py, csrc/jpeg.cu) against Pillow on one CPU core.

Prints one JSON line.  Per workload:
  - the device time of the decode and of each stage (entropy decode, IDCT, upsample / colour), from CUDA events around each
    launch of `--iters` calls after `--warmup`, the median over `--reps` windows;
  - images/s and compressed MB/s over that device time;
  - the host side of a call: the plan (header parse, tables) and the whole decode_jpeg call (plan, one pinned copy, the
    kernels, the status read), wall clock, median;
  - Pillow's Image.open(f).convert(mode) on one core of the same host over a subset of the images, or "not measured" where
    Pillow is missing.
The streams are seeded smooth frames encoded by Pillow 4:2:0 q95 (RGB) or grayscale q95 (the L planes of Flow); their decode is
checked bitwise against Pillow (or the numpy oracle without Pillow) on a sample before timing.  The card name and power limit
are read in the same run.

    python tools/bench_jpeg.py [--iters 10] [--warmup 3] [--reps 5] [--no-cpu]
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "action-detection_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

# (name, images, H, W, mode): config [1]'s training batch (32 proposals x 9 segments), Flow's (the same 288 segments x 5 ticks
# x (x, y) planes), and 10-crop test calls of 40 and 100 ticks at 340x256 and 480x360
WORKLOADS = [
    ("train_rgb_340x256", 288, 256, 340, "RGB"),
    ("train_flow_340x256", 2880, 256, 340, "L"),
    ("test_340x256_40", 40, 256, 340, "RGB"),
    ("test_340x256_100", 100, 256, 340, "RGB"),
    ("test_480x360_40", 40, 360, 480, "RGB"),
    ("test_480x360_100", 100, 360, 480, "RGB"),
]
DISTINCT = 96        # distinct streams per workload, cycled
STAGES = ("jpeg_entropy_kernel", "jpeg_idct_kernel", "jpeg_colour_kernel")
# README's measured training rates (NVIDIA H100 80GB HBM3, 700 W): proposals/s, 32 proposals per step
STEP_MS = {"train_rgb_340x256": 32 / 818.0 * 1e3, "train_flow_340x256": 32 / 693.0 * 1e3}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "not read"


def streams(H, W, mode, seed):
    from oracle.gen_golden_jpeg import content, encode
    sub = "gray" if mode == "L" else "420"
    return [encode(content("smooth", W, H, 1 if mode == "L" else 3, seed + i), sub, quality=95) for i in range(DISTINCT)]


def reference(data, mode):
    try:
        from PIL import Image
    except ImportError:
        from oracle import jpeg_oracle as J
        return J.decode(data, mode)
    im = Image.open(io.BytesIO(data)).convert(mode)
    return np.asarray(im).reshape(im.size[1], im.size[0], -1)


def gpu_arm(blobs, mode, iters, warmup, reps):
    from ops.jpeg import JpegPlan, decode_jpeg
    from ssn_b200._lib import lib
    dev = torch.device("cuda:0")
    ends = np.cumsum([len(b) for b in blobs])
    buf = np.frombuffer(b"".join(blobs), np.uint8)
    t0 = time.perf_counter()
    plan = JpegPlan(buf, ends - [len(b) for b in blobs], ends, [3 if mode == "RGB" else 1] * len(blobs))
    plan_s = time.perf_counter() - t0
    d = plan.upload(dev)
    out = torch.empty(plan.out_bytes, dtype=torch.uint8, device=dev)
    ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=dev)
    status = torch.empty(len(blobs), dtype=torch.int32, device=dev)
    for _ in range(warmup):
        plan.run(d, out, status, ws)
    torch.cuda.synchronize()
    assert (status.cpu() == 0).all()
    for i in range(0, len(blobs), max(1, len(blobs) // 8)):
        im = plan.images[i]
        got = out[im.out_offset:im.out_offset + im.width * im.height * im.channels].cpu().numpy()
        assert got.tobytes() == reference(blobs[i], mode).tobytes(), "image %d differs from Pillow" % i
    totals, stages = [], {k: [] for k in STAGES}
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(reps):
        lib.ssnb_timing_begin(stream)
        for _ in range(iters):
            plan.run(d, out, status, ws)
        rows = [r.split("\t") for r in lib.ssnb_timing_launches().decode().splitlines()]
        per = {k: sum(float(r[3]) for r in rows if r[0] == k) / iters for k in STAGES}
        for k in STAGES:
            stages[k].append(per[k])
        totals.append(sum(per.values()))
    ms = statistics.median(totals)
    call = []
    for _ in range(max(3, reps)):
        t0 = time.perf_counter()
        decode_jpeg([blobs], mode=mode)
        call.append(time.perf_counter() - t0)
    mb = buf.size / 1e6
    return {"images": len(blobs), "compressed_MB": round(mb, 2), "device_ms": round(ms, 3),
            "images_per_s": round(len(blobs) / ms * 1e3, 1), "compressed_MB_per_s": round(mb / ms * 1e3, 1),
            "stage_ms": {k.replace("jpeg_", "").replace("_kernel", ""): round(statistics.median(v), 3) for k, v in stages.items()},
            "host_plan_ms": round(plan_s * 1e3, 2), "decode_jpeg_call_ms": round(statistics.median(call) * 1e3, 2),
            "workspace_MB": round(plan.workspace_bytes / 1e6, 1)}


def cpu_arm(blobs, mode, n=48):
    try:
        from PIL import Image
    except ImportError:
        return "not measured"
    torch.set_num_threads(1)
    sub = blobs[:n]
    for b in sub[:4]:
        Image.open(io.BytesIO(b)).convert(mode)
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        for b in sub:
            Image.open(io.BytesIO(b)).convert(mode).load()
        times.append(time.perf_counter() - t0)
    per = statistics.median(times) / len(sub)
    import PIL
    return {"images_per_s": round(1 / per, 1), "ms_per_image": round(per * 1e3, 3), "pillow": PIL.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg.py measures the GPU and needs a CUDA device")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "workloads": {}}
    for k, (wname, n, H, W, mode) in enumerate(WORKLOADS):
        distinct = streams(H, W, mode, 1000 * k)
        blobs = [distinct[i % DISTINCT] for i in range(n)]
        r = gpu_arm(blobs, mode, args.iters, args.warmup, args.reps)
        r["cpu_pillow_one_core"] = "not measured" if args.no_cpu else cpu_arm(distinct, mode)
        if isinstance(r["cpu_pillow_one_core"], dict):
            r["cpu_cores_to_match"] = round(r["images_per_s"] / r["cpu_pillow_one_core"]["images_per_s"], 1)
        if wname in STEP_MS:
            r["share_of_training_step"] = round(r["device_ms"] / STEP_MS[wname], 4)
        res["workloads"][wname] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
