"""Benchmark the GPU JPEG round trip (ops.jpeg.JpegRoundtripPlan, csrc/jpeg_roundtrip.cu) against encode -> decode on the
GPU (ops.jpeg.JpegEncodePlan, then decode_jpeg's JpegPlan on the files) on the same images in the same run; prints one JSON
line.  Workloads, each one call, quality 95:

  flow_L      the 512 x / y planes of the TV-L1 benchmark's 256-pair call, 340 x 256 'L' (flow-like planes)
  rgb_340     256 RGB frames at 340 x 256 (smooth textures)
  rgb_480     400 RGB frames at 480 x 360

Per workload: the median and range of CUDA-event times over --windows windows of --calls calls after warm-up for the round
trip, for the encode alone and for the decode alone (the decode's plan is made on the host once, outside the window, as its
entropy decode needs the files' bytes), the round trip's outputs checked bitwise against decode(encode); the round trip's
bytes read (pixels) and written (pixels) from shapes with their share of 3.35 TB/s HBM; and the device time per kernel
from torch.profiler in a separate run.  The card's name and power limit are read in the same run.  Needs a CUDA device.

    python tools/bench_jpeg_roundtrip.py
"""
import argparse
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_jpeg_encode import HBM, WORKLOADS, card_info, images  # noqa: E402


def timed(fn, calls, windows, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3 / calls)
    return float(np.median(times)), [round(min(times), 5), round(max(times), 5)]


def kernel_ms(fn):
    import torch
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        m = re.search(r"(\w+_kernel)(<\d+>)?", ev.key)
        if m and ev.device_time_total > 0:
            out[m.group(0)] = round(out.get(m.group(0), 0.0) + ev.device_time_total / 1e3, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from ops.jpeg import JpegEncodePlan, JpegPlan, JpegRoundtripPlan
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_roundtrip needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card_info()}
    for name, mode, n, h, w in WORKLOADS:
        arr = images(mode, n, h, w)
        x = torch.from_numpy(arr).to(dev)
        rt = JpegRoundtripPlan([(h, w)] * n, mode, 95, dev)
        enc = JpegEncodePlan([(h, w)] * n, mode, 95, dev)
        enc.run(x)
        files = enc.files()
        lens = np.array([len(f) for f in files], np.int64)
        ends = np.cumsum(lens)
        dec = JpegPlan(np.frombuffer(b"".join(files), np.uint8), ends - lens, ends, [arr.shape[3]] * n)
        dec_in = dec.upload(dev)
        dec_out = torch.empty(dec.out_bytes, dtype=torch.uint8, device=dev)
        dec_ws = torch.empty(max(dec.workspace_bytes, 1), dtype=torch.uint8, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        got = rt.run(x)
        dec.run(dec_in, dec_out, status, dec_ws)
        torch.cuda.synchronize()
        assert not status.any() and torch.equal(got.reshape(-1), dec_out), name + ": round trip differs from decode(encode)"
        t_rt, r_rt = timed(lambda: rt.run(x), a.calls, a.windows, a.warmup)
        t_enc, r_enc = timed(lambda: enc.run(x), a.calls, a.windows, a.warmup)
        t_dec, r_dec = timed(lambda: dec.run(dec_in, dec_out, status, dec_ws), a.calls, a.windows, a.warmup)
        moved = 2 * int(arr.nbytes)
        res[name] = {"workload": "%d %s images of %dx%d (W x H), quality 95" % (n, mode, w, h),
                     "roundtrip_s_per_call": round(t_rt, 5), "roundtrip_s_range": r_rt, "images_per_s": round(n / t_rt, 1),
                     "encode_s_per_call": round(t_enc, 5), "encode_s_range": r_enc,
                     "decode_s_per_call": round(t_dec, 5), "decode_s_range": r_dec,
                     "speedup_vs_encode_plus_decode": round((t_enc + t_dec) / t_rt, 2),
                     "bytes_read_plus_written": moved, "hbm_share": round(moved / t_rt / HBM, 4),
                     "roundtrip_kernel_ms": kernel_ms(lambda: rt.run(x)),
                     "encode_kernel_ms": kernel_ms(lambda: enc.run(x)),
                     "decode_kernel_ms": kernel_ms(lambda: dec.run(dec_in, dec_out, status, dec_ws))}
        del rt, enc, dec, dec_in, dec_out, dec_ws, x, got
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
