"""Benchmark restart intervals in the GPU JPEG path: what restart_marker_rows / restart_marker_blocks cost the encoder
(ops.jpeg.JpegEncodePlan, csrc/jpeg_encode.cu) and what they save the decoder (ops.jpeg.decode_jpeg, csrc/jpeg.cu), whose
entropy stage runs one thread per interval.  Prints one JSON line.

Encode: bench_jpeg_encode's three workloads (512 flow planes at 340 x 256 'L', 256 RGB frames at 340 x 256, 400 at 480 x 360,
quality 95), with no markers, restart_marker_rows=1 and restart_marker_blocks=1.  The arms alternate window by window in one
run: per arm the median and range of CUDA-event times over --windows windows of --calls calls after warm-up, the device time
per kernel from torch.profiler in a separate call, and the mean file size.

Decode: bench_jpeg's training batches, 288 RGB frames and 2,880 Flow planes at 340 x 256 (smooth seeded content, 96 distinct
images cycled), encoded by our encoder at quality 95 with no markers, rows=1 and rows=2.  Per arm, alternating: the device
time of each decode stage (jpeg_entropy_kernel, jpeg_idct_kernel, jpeg_colour_kernel) from the library's per-launch CUDA
events, median over --windows windows of --calls calls; the whole decode_jpeg call (host plan, copy, kernels, status read),
wall clock, median; the intervals per image; and whether every arm decodes to the same bytes in this run.  The card's name
and power limit are read in the same run.  Needs a CUDA device.

    python tools/bench_jpeg_restart.py
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

ENC_ARMS = (("none", {}), ("rows1", {"restart_marker_rows": 1}), ("blocks1", {"restart_marker_blocks": 1}))
DEC_ARMS = (("none", {}), ("rows1", {"restart_marker_rows": 1}), ("rows2", {"restart_marker_rows": 2}))
DEC_WORKLOADS = (("train_rgb_340x256", 288, 256, 340, "RGB"), ("train_flow_340x256", 2880, 256, 340, "L"))
STAGES = ("jpeg_entropy_kernel", "jpeg_idct_kernel", "jpeg_colour_kernel")


def _rng(v):
    return [round(min(v), 5), round(max(v), 5)]


def encode_bench(a, dev):
    import torch
    from ops.jpeg import JpegEncodePlan
    from bench_jpeg_encode import WORKLOADS, images
    res = {}
    for name, mode, n, h, w in WORKLOADS:
        x = torch.from_numpy(images(mode, n, h, w)).to(dev)
        plans = {arm: JpegEncodePlan([(h, w)] * n, mode, 95, dev, **kw) for arm, kw in ENC_ARMS}
        for p in plans.values():
            for _ in range(a.warmup):
                p.run(x)
        torch.cuda.synchronize()
        times = {arm: [] for arm in plans}
        for _ in range(a.windows):
            for arm, p in plans.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.calls):
                    p.run(x)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1) / a.calls)
        out = {}
        for arm, p in plans.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                p.run(x)
                torch.cuda.synchronize()
            stage = {}
            for ev in prof.key_averages():
                if "enc_" in ev.key and "_kernel" in ev.key:
                    k = ev.key.split("enc_")[1].split("_kernel")[0]
                    stage[k] = round(stage.get(k, 0.0) + ev.device_time_total / 1e3, 3)
            p.run(x)
            lens = p.lengths.cpu().numpy()
            out[arm] = {"ms_per_call": round(statistics.median(times[arm]), 4), "ms_range": _rng(times[arm]), "stage_ms": stage,
                        "mean_file_bytes": round(float(lens.mean()), 1)}
        for arm in ("rows1", "blocks1"):
            out[arm]["vs_none"] = round(out[arm]["ms_per_call"] / out["none"]["ms_per_call"], 3)
        res[name] = {"workload": "%d %s images of %dx%d (W x H), quality 95" % (n, mode, w, h), "arms": out}
        del plans, x
        torch.cuda.empty_cache()
    return res


def decode_bench(a, dev):
    import torch
    from oracle.gen_golden_jpeg import content
    from ops.jpeg import JpegPlan, decode_jpeg, encode_jpeg
    from ssn_b200._lib import lib
    res = {}
    stream = torch.cuda.current_stream().cuda_stream
    for k, (name, n, H, W, mode) in enumerate(DEC_WORKLOADS):
        C = 3 if mode == "RGB" else 1
        distinct = torch.from_numpy(np.stack([content("smooth", W, H, C, 1000 * k + i) for i in range(96)])).to(dev)
        arms = {}
        for arm, kw in DEC_ARMS:
            files = encode_jpeg(distinct, mode=mode, quality=95, **kw)
            blobs = [files[i % len(files)] for i in range(n)]
            ends = np.cumsum([len(b) for b in blobs])
            buf = np.frombuffer(b"".join(blobs), np.uint8)
            plan = JpegPlan(buf, ends - [len(b) for b in blobs], ends, [C] * n)
            d = plan.upload(dev)
            out = torch.empty(plan.out_bytes, dtype=torch.uint8, device=dev)
            ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=dev)
            status = torch.empty(n, dtype=torch.int32, device=dev)
            arms[arm] = dict(blobs=blobs, plan=plan, d=d, out=out, ws=ws, status=status, mb=buf.size / 1e6,
                             intervals=int(plan.images[0].intervals), stages={s: [] for s in STAGES}, device=[], call=[])
        for r in arms.values():
            for _ in range(a.warmup):
                r["plan"].run(r["d"], r["out"], r["status"], r["ws"])
        torch.cuda.synchronize()
        assert all(bool((r["status"] == 0).all()) for r in arms.values())
        same = all(torch.equal(r["out"], arms["none"]["out"]) for r in arms.values())
        for _ in range(a.windows):
            for r in arms.values():
                lib.ssnb_timing_begin(stream)
                for _ in range(a.calls):
                    r["plan"].run(r["d"], r["out"], r["status"], r["ws"])
                rows = [x.split("\t") for x in lib.ssnb_timing_launches().decode().splitlines()]
                per = {s: sum(float(x[3]) for x in rows if x[0] == s) / a.calls for s in STAGES}
                for s in STAGES:
                    r["stages"][s].append(per[s])
                r["device"].append(sum(per.values()))
            for r in arms.values():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                decode_jpeg([r["blobs"]], mode=mode)
                r["call"].append((time.perf_counter() - t0) * 1e3)
        out = {}
        for arm, r in arms.items():
            out[arm] = {"intervals_per_image": r["intervals"], "compressed_MB": round(r["mb"], 3),
                        "device_ms": round(statistics.median(r["device"]), 3), "device_ms_range": _rng(r["device"]),
                        "stage_ms": {s.replace("jpeg_", "").replace("_kernel", ""): round(statistics.median(v), 3) for s, v in r["stages"].items()},
                        "decode_jpeg_call_ms": round(statistics.median(r["call"]), 2), "decode_jpeg_call_ms_range": _rng(r["call"])}
        for arm in ("rows1", "rows2"):
            out[arm]["entropy_speedup"] = round(out["none"]["stage_ms"]["entropy"] / out[arm]["stage_ms"]["entropy"], 2)
        res[name] = {"workload": "%d %s images of %dx%d (W x H), quality 95, our encoder" % (n, mode, W, H),
                     "outputs_bitwise_equal_across_arms": bool(same), "arms": out}
        del arms, distinct
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg_restart needs a CUDA device")
    from bench_jpeg_encode import card_info
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card_info(), "encode": encode_bench(a, dev), "decode": decode_bench(a, dev)}))


if __name__ == "__main__":
    main()
