#!/usr/bin/env python
"""Per-launch times of the tensor-core kernels (umma_conv_kernel, umma_wgrad_kernel) on one H100; prints ONE JSON line.

  python tools/bench_conv.py [--frames 288] [--reps 2] [--table FILE]

One eager forward + backward of the BNInception backbone at `frames` frames (288 = bench.py's 32 proposals x 9 segments)
in EXACT_TC and in FAST, after one warm-up pass, with every library launch timed by CUDA events on its stream
(ssnb_timing_begin / ssnb_timing_launches).  For each umma_conv_kernel launch the table lists op, pass, tile count, tile
width, microseconds, algorithmic TFLOP/s, the epilogue's HBM bytes and the GB/s they imply, next to a data-sheet model of
the same launch: issued MMAs (padding included; EXACT_TC issues three per product) at 989 TFLOP/s dense fp16, and epilogue
bytes at 3.35 TB/s HBM3 (H100 SXM data sheet, 700 W).  The model's epilogue bytes per output element: EXACT_TC forward 8
(fp32 + hi + lo planes), data gradient 12 (also the old gradient or the fp32 mask); FAST forward 2, data gradient 4.
For each umma_wgrad_kernel launch a second table lists op, CTAs, splits, microseconds, algorithmic TFLOP/s, the product
MMAs the kernel issues (m64nNk16 units of 64 x 64 x 16, padding included: every 128-row co tile issues for each 64-row half
that holds an output channel, over all block_n columns of all taps of its tap group, stale taps of a short last group
included; three per product in EXACT_TC) and the bytes its TMA loads move into shared memory (every box of every pixel tile,
each plane once), next to the model: those MMAs at 989 TFLOP/s.  Not counted: the bias-gradient m64n16k16 MMAs of layers
whose bias gradient rides on the kernel (per pixel tile, 4 in FAST and 8 in EXACT_TC for each such 64-row half of the CTAs of
the first ci tile and tap group, a quarter of a unit each), because which layers carry them is decided by the engine's mask
fusion, not by the plan.  The plan comes from oracle/tile_plan.py, which restates the kernel's planner.
The table goes to stdout (or FILE); the JSON line carries the totals per precision and pass.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

PEAK_F16 = 989e12       # dense fp16 tensor FLOP/s, H100 SXM data sheet
HBM = 3.35e12           # B/s, H100 SXM data sheet
EPI_BYTES = {"exact_tc": (8, 12), "fast": (2, 4)}
PHASES = {0: "fwd", 1: "dgrad"}
MMA_UNIT = 64 * 64 * 16         # multiply-adds of one 64 x 64 x 16 slice of a wgmma
BOX_BYTES = 64 * 128            # one [64 px][64 ch] fp16 TMA box


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def launch_model(op, phase, flop, tiles, block_n, spec, precision):
    """(epilogue bytes, model MMA seconds, model epilogue seconds) of one launch; conv1 (space-to-depth taps) has no MMA model"""
    convs = [spec[n] for n in op.split("+")]
    if phase == 0:          # output elements: pixels x cout of every fused sibling
        elems = sum(flop_c / (2.0 * ci * k * k) for flop_c, (ci, co, k, s) in zip(_split(flop, convs), convs))
        kred, taps = convs[0][0], convs[0][2] ** 2
    else:                   # input-resolution pixels x cin (stride-2 layers: the zero-upsampled dz has 4x the pixels)
        elems = sum(flop_c / (2.0 * co * k * k) * s * s for flop_c, (ci, co, k, s) in zip(_split(flop, convs), convs)) / len(convs)
        kred, taps = sum(c[1] for c in convs), convs[0][2] ** 2
    b = elems * EPI_BYTES[precision][phase]
    nseg = 3 if precision == "exact_tc" else 1
    t_mma = None if op == "conv1_7x7_s2" else 2.0 * tiles * 128 * block_n * math.ceil(kred / 16) * 16 * taps * nseg / PEAK_F16
    return b, t_mma, b / HBM


def wgrad_counts(plan, co, precision):
    """(issued 64 x 64 x 16 product MMA units, TMA bytes) of one umma_wgrad_kernel launch (tile_plan.wgrad_plan's dict); the
    bias-gradient MMAs are not included (module docstring)"""
    nseg, planes = (3, 2) if precision == "exact_tc" else (1, 1)
    nb, tpc, taps = plan["block_n"] // 64, plan["taps_per_cta"], plan["ntaps"]
    mma = tma = 0
    for mt in range(plan["m_tiles"]):
        halves = sum(1 for h in range(2) if mt * 128 + h * 64 < co)       # 64-row halves holding an output channel
        for g in range(plan["tap_groups"]):
            ntap = min(tpc, taps - g * tpc)
            mma += plan["n_tiles"] * halves * tpc * nb * 4 * nseg          # 4 k-steps of 16 pixels per tile
            tma += plan["n_tiles"] * planes * (halves + ntap * nb) * BOX_BYTES
    return mma * plan["ptiles"], tma * plan["ptiles"]


def _split(flop, convs):
    w = [ci * co * k * k for (ci, co, k, s) in convs]
    return [flop * x / sum(w) for x in w]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=288)
    ap.add_argument("--reps", type=int, default=2, help="timed forward + backward passes per precision (times are averaged)")
    ap.add_argument("--table", default=None, help="write the per-launch table here instead of stdout")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_conv.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    from ssn_b200 import _lib
    from ssn_b200.engine import BackboneEngine
    from oracle import ssn_oracle as O
    from oracle import synth
    from oracle import tile_plan as T
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    spec = {n: (ci, co, k, s) for (n, ci, co, k, s, _p) in O.conv_layers(3)}
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    x = synth.synth_frames(args.frames, 3, seed=1).to(dev)
    table = open(args.table, "w") if args.table else sys.stdout
    result = {"metric": "umma_conv_kernel and umma_wgrad_kernel per-launch time, backbone fwd + bwd", "frames": args.frames, "card": card_info(), "modes": {}}
    names = list(spec)
    for precision, prec in (("exact_tc", _lib.EXACT_TC), ("fast", _lib.FAST_FP16)):
        # the engine is driven from this thread: the timing session is per thread, and autograd would run the backward on
        # a worker thread of its own
        e = BackboneEngine(3, args.frames, prec, True, 1024.0, dev)
        e.pack([bb[n + ".weight"].to(dev) for n in names], [bb[n + ".bias"].to(dev) for n in names],
               [bb[n + "_bn.weight"].to(dev) for n in names], [bb[n + "_bn.bias"].to(dev) for n in names],
               [bb[n + "_bn.running_mean"].to(dev) for n in names], [bb[n + "_bn.running_var"].to(dev) for n in names])
        dw = [torch.zeros(bb[n + ".weight"].shape, device=dev) for n in names]
        db = [torch.zeros(bb[n + ".bias"].shape, device=dev) for n in names]
        g = torch.randn(args.frames, 1024, device=dev, generator=torch.Generator(device=dev).manual_seed(0)) * 1e-3

        def step():
            e.forward(x)
            e.backward(g, dw, db)
        step()
        torch.cuda.synchronize()
        acc, wacc = {}, {}
        for _ in range(args.reps):
            _lib.lib.ssnb_timing_begin(C.c_void_p(torch.cuda.current_stream().cuda_stream))
            step()
            for i, ln in enumerate(_lib.lib.ssnb_timing_launches().decode().splitlines()):
                c = ln.split("\t")
                if c[0] == "umma_wgrad_kernel":
                    a = wacc.setdefault((i, c[2]), {"ms": 0.0, "flop": float(c[4]), "ctas": int(c[5]), "splits": int(c[6])})
                    a["ms"] += float(c[3]) / args.reps
                    continue
                if c[0] != "umma_conv_kernel" or int(c[1]) not in PHASES:
                    continue
                key = (i, c[2], int(c[1]))
                a = acc.setdefault(key, {"ms": 0.0, "flop": float(c[4]), "tiles": int(c[5]), "block_n": int(c[6])})
                a["ms"] += float(c[3]) / args.reps
        print("# %s, %d frames, %s" % (precision, args.frames, result["card"]), file=table)
        print("%-62s %5s %6s %5s %9s %8s %9s %8s %9s %9s" % ("op", "pass", "tiles", "bn", "us", "TFLOP/s", "epi MB", "epi GB/s",
                                                              "mdl mma", "mdl epi"), file=table)
        tot = {}
        for (i, op, ph), a in sorted(acc.items()):
            b, t_mma, t_epi = launch_model(op, ph, a["flop"], a["tiles"], a["block_n"], spec, precision)
            s = a["ms"] / 1e3
            print("%-62s %5s %6d %5d %9.1f %8.1f %9.1f %8.0f %9s %9.1f" % (
                op[:62], PHASES[ph], a["tiles"], a["block_n"], s * 1e6, a["flop"] / s / 1e12, b / 1e6, b / s / 1e9,
                "-" if t_mma is None else "%.1f" % (t_mma * 1e6), t_epi * 1e6), file=table)
            t = tot.setdefault(PHASES[ph], {"launches": 0, "ms": 0.0, "flop": 0.0, "epi_bytes": 0.0, "model_mma_ms": 0.0, "model_epi_ms": 0.0,
                                            "model_serial_ms": 0.0, "model_overlap_ms": 0.0})
            t["launches"] += 1; t["ms"] += a["ms"]; t["flop"] += a["flop"]; t["epi_bytes"] += b
            if t_mma is not None:
                t["model_mma_ms"] += t_mma * 1e3; t["model_epi_ms"] += t_epi * 1e3
                t["model_serial_ms"] += (t_mma + t_epi) * 1e3; t["model_overlap_ms"] += max(t_mma, t_epi) * 1e3
        plans = {l["op"]: l["plan"] for l in T.schedule(3, args.frames, precision, torch.cuda.get_device_properties(dev).multi_processor_count)
                 if l["phase"] == 2}
        print(file=table)
        print("%-24s %5s %6s %9s %8s %10s %9s %9s %8s" % ("op (wgrad)", "ctas", "splits", "us", "TFLOP/s", "MMAs", "TMA MB", "TMA GB/s",
                                                          "mdl mma"), file=table)
        w = tot.setdefault("wgrad", {"launches": 0, "ms": 0.0, "flop": 0.0, "mmas": 0, "tma_bytes": 0.0, "model_mma_ms": 0.0})
        for (i, op), a in sorted(wacc.items()):
            mmas, tma = wgrad_counts(plans[op], spec[op][1], precision)
            s = a["ms"] / 1e3
            t_mma = 2.0 * mmas * MMA_UNIT / PEAK_F16
            print("%-24s %5d %6d %9.1f %8.1f %10d %9.1f %9.0f %8.1f" % (op[:24], a["ctas"], a["splits"], s * 1e6, a["flop"] / s / 1e12, mmas,
                                                                    tma / 1e6, tma / s / 1e9, t_mma * 1e6), file=table)
            w["launches"] += 1; w["ms"] += a["ms"]; w["flop"] += a["flop"]; w["mmas"] += mmas; w["tma_bytes"] += tma
            w["model_mma_ms"] += t_mma * 1e3
        for t in tot.values():
            t["tflops"] = t["flop"] / (t["ms"] / 1e3) / 1e12
        print(file=table)
        result["modes"][precision] = tot
        del e
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
