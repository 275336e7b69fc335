"""Benchmark the GPU frame resize (ops.optical_flow.ResizePlan, csrc/frame_resize.cu): DenseFlow's cv::resize of every
decoded frame to 340 x 256 (INTER_LINEAR), many videos per call; prints one JSON line.  Workloads, 2,048 frames each, one call:

  thumos     8 videos x 256 frames of 320 x 240 (THUMOS14; an upscale)
  anet       3 videos of 640 x 360, 3 of 854 x 480 and 2 of 1280 x 720, 256 frames each (ActivityNet's YouTube sizes;
             downscales of three source sizes in one call)

Per workload: the median and range of CUDA-event times of plan.run() (the kernel alone, sources already packed) over
--windows windows of --calls calls after warm-up, and of resize_frames (which also packs the videos into one buffer);
frames per second; bytes read (whole source frames) plus written, from shapes, with their share of 3.35 TB/s HBM; the
device time per kernel from torch.profiler in a separate run; and cv2.resize per frame on one CPU core for each source
size.  The first frame of every video is checked bitwise against the oracle.  The card's name and power limit are read in
the same run.  Needs a CUDA device.

    python tools/bench_frame_resize.py
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_jpeg_encode import HBM, card_info  # noqa: E402
from bench_jpeg_roundtrip import kernel_ms, timed  # noqa: E402

DST_W, DST_H = 340, 256
WORKLOADS = [("thumos", [(256, 240, 320)] * 8),
             ("anet", [(256, 360, 640)] * 3 + [(256, 480, 854)] * 3 + [(256, 720, 1280)] * 2)]


def cv2_ms_per_frame(h, w, frames=64):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    src = np.random.default_rng(h * w).integers(0, 256, (frames, h, w, 3), dtype=np.uint8)
    for f in src[:4]:
        cv2.resize(f, (DST_W, DST_H), interpolation=cv2.INTER_LINEAR)
    t0 = time.perf_counter()
    for f in src:
        cv2.resize(f, (DST_W, DST_H), interpolation=cv2.INTER_LINEAR)
    return round((time.perf_counter() - t0) / frames * 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from oracle import frame_resize_oracle as R
    from ops.optical_flow import ResizePlan, resize_frames
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_resize needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card_info()}
    for name, shapes in WORKLOADS:
        g = torch.Generator(device=dev).manual_seed(0)
        videos = [torch.randint(0, 256, s + (3,), dtype=torch.uint8, device=dev, generator=g) for s in shapes]
        plan = ResizePlan(shapes, DST_W, DST_H, dev)
        got = plan.run(videos)
        for v, o in zip(videos, plan.offsets[:-1]):
            assert got[o].cpu().numpy().tobytes() == R.resize(v[0].cpu().numpy(), DST_W, DST_H).tobytes(), name + ": differs from the oracle"
        t, r = timed(lambda: plan.run(), a.calls, a.windows, a.warmup)
        t_rf, r_rf = timed(lambda: resize_frames(videos), a.calls, a.windows, a.warmup)
        n = int(plan.offsets[-1])
        moved = int(plan.src.numel()) + int(plan.frames.numel())
        sizes = sorted({s[1:] for s in shapes})
        res[name] = {"workload": "%d frames: %s (W x H) -> %dx%d" % (n, ", ".join("%d x %dx%d" % (sum(s[0] for s in shapes if s[1:] == hw), hw[1], hw[0])
                                                                              for hw in sizes), DST_W, DST_H),
                     "s_per_call": round(t, 6), "s_range": r, "frames_per_s": round(n / t, 1),
                     "resize_frames_s_per_call": round(t_rf, 6), "resize_frames_s_range": r_rf,
                     "bytes_read_plus_written": moved, "hbm_share": round(moved / t / HBM, 4),
                     "kernel_ms": kernel_ms(lambda: plan.run()),
                     "cv2_ms_per_frame_one_core": {"%dx%d" % (hw[1], hw[0]): cv2_ms_per_frame(*hw) for hw in sizes}}
        del videos, plan, got
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
