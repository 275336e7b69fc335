"""Frame transforms on the GPU (ops/frame_transforms.py, csrc/frames.cu) against the reference's PIL transforms on one CPU core.

Prints one JSON line: per workload the network frames per second on the GPU (CUDA events around `--iters` calls after
`--warmup`, median of `--reps` windows), the bytes the call must move (uint8 source read, fp32 frames written, the GroupScale
scratch written and read back; computed from the shapes) as a share of the H100 SXM's 3.35 TB/s, and the CPU arm: the
reference's transforms.py (the copy build() vendors into oracle/_ref) + PIL + Stack / ToTorchFormatTensor / GroupNormalize, on one
core, over a smaller batch of the same shape.  Where that copy or PIL is missing the CPU arm reads "not measured".  The card
name and power limit are read in the same run.

    python tools/bench_frames.py [--iters 20] [--warmup 5] [--reps 5] [--no-cpu]
"""
import argparse
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

HBM_BYTES_PER_S = 3.35e12
RGB_MEAN, FLOW_MEAN = [104, 117, 128], [128]

# (name, kind, groups, images per group, H, W, channels of an image, channels of a network frame)
#   train_*: the bench shape of training, 32 proposals x 9 segments (RGB; Flow: 5 ticks x (x, y) planes per segment)
#   oversample_*: 10-crop test chunks of 40 and 100 ticks, from 340x256 (no resize) and 480x360 (GroupScale to 341x256)
#   center_340: 1-crop test / validation of the same 288 frames
WORKLOADS = [
    ("train_rgb_340x256", "train", 32, 9, 256, 340, 3, 3),
    ("train_flow_340x256", "train", 32, 90, 256, 340, 1, 10),
    ("oversample_340x256_40", "oversample", 1, 40, 256, 340, 3, 3),
    ("oversample_340x256_100", "oversample", 1, 100, 256, 340, 3, 3),
    ("oversample_480x360_40", "oversample", 1, 40, 360, 480, 3, 3),
    ("oversample_480x360_100", "oversample", 1, 100, 360, 480, 3, 3),
    ("center_340x256", "center", 32, 9, 256, 340, 3, 3),
]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "not read"


def bytes_moved(kind, G, n, H, W, c):
    from oracle.frames_oracle import scaled_size
    crops = 10 if kind == "oversample" else 1
    b = G * n * H * W * c + G * n * crops * c * 224 * 224 * 4
    if kind != "train":
        sh, sw = scaled_size(H, W, 256)
        if (sh, sw) != (H, W):
            b += 2 * G * n * sh * sw * c
    return b


def gpu_arm(wl, iters, warmup, reps):
    from ops.frame_transforms import FramePlan, sample_train_params
    from ssn_b200._lib import FRAMES_TRAIN, FRAMES_OVERSAMPLE, FRAMES_CENTER
    import random
    name, kind, G, n, H, W, c, fc = wl
    dev = torch.device("cuda:0")
    mode = {"train": FRAMES_TRAIN, "oversample": FRAMES_OVERSAMPLE, "center": FRAMES_CENTER}[kind]
    params = sample_train_params([(H, W)] * G, [1, .875, .75] if c == 1 else [1, .875, .75, .66], rng=random.Random(0)) \
        if kind == "train" else None
    plan = FramePlan(mode, [(n, H, W)] * G, c, 224, 256, FLOW_MEAN if c == 1 else RGB_MEAN, [1], c == 1, dev, params)
    src = torch.randint(0, 256, (G * n * H * W * c,), dtype=torch.uint8, device=dev)
    dst = torch.empty(plan.dst_floats, dtype=torch.float32, device=dev)
    for _ in range(warmup):
        plan.run(src, dst)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            plan.run(src, dst)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3 / iters)
    t = statistics.median(times)
    frames = plan.dst_floats // (fc * 224 * 224)
    moved = bytes_moved(kind, G, n, H, W, c)
    return {"ms_per_call": round(t * 1e3, 4), "frames": frames, "frames_per_s": round(frames / t, 1),
            "hbm_bytes": moved, "hbm_share": round(moved / t / HBM_BYTES_PER_S, 4)}


def cpu_arm(wl):
    """the reference pipeline on one core over one group (oversample: 4 ticks), in network frames per second"""
    name, kind, G, n, H, W, c, fc = wl
    path = os.path.join(ROOT, "oracle", "_ref", "transforms.py")
    try:
        from PIL import Image
        import importlib.util
        import torchvision
    except ImportError:
        return "not measured"
    if not os.path.exists(path):
        return "not measured"
    torchvision.transforms.Scale = torchvision.transforms.Resize      # the fifth patch (oracle/gen_golden_frames.py)
    spec = importlib.util.spec_from_file_location("reference_transforms", path)
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    torch.set_num_threads(1)
    n_cpu = 4 if kind == "oversample" else n
    rng = np.random.default_rng(0)
    imgs = [Image.fromarray(a) if c == 3 else Image.fromarray(a[:, :, 0], "L") for a in rng.integers(0, 256, (n_cpu, H, W, c), dtype=np.uint8)]
    if kind == "train":
        head = [T.GroupMultiScaleCrop(224, [1, .875, .75] if c == 1 else [1, .875, .75, .66]), T.GroupRandomHorizontalFlip(is_flow=c == 1)]
    elif kind == "oversample":
        head = [T.GroupOverSample(224, 256)]
    else:
        head = [T.GroupScale(256), T.GroupCenterCrop(224)]
    pipe = torchvision.transforms.Compose(head + [T.Stack(roll=True), T.ToTorchFormatTensor(div=False),
                                                  T.GroupNormalize(FLOW_MEAN if c == 1 else RGB_MEAN, [1])])
    pipe(imgs)
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        out = pipe(imgs)
        times.append(time.perf_counter() - t0)
    frames = out.shape[0] // fc
    return {"frames_per_s": round(frames / statistics.median(times), 1), "group_images": n_cpu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames.py measures the GPU and needs a CUDA device")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "workloads": {}}
    for wl in WORKLOADS:
        r = gpu_arm(wl, args.iters, args.warmup, args.reps)
        r["cpu_reference_one_core"] = "not measured" if args.no_cpu else cpu_arm(wl)
        if isinstance(r["cpu_reference_one_core"], dict):
            r["speedup_vs_one_core"] = round(r["frames_per_s"] / r["cpu_reference_one_core"]["frames_per_s"], 1)
        res["workloads"][wl[0]] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
