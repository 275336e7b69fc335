#!/usr/bin/env python
"""Benchmark of the InceptionV3 backbone at test time on one H100; prints ONE JSON line.

  python tools/bench_inception_v3.py [--calls K] [--warmup W] [--ticks 40] [--crops 10]

SSN.test_scores (the loop body of ssn_test.py:80-84 with the crop mean folded into the test FC) and BinaryClassifier
scoring (`rst, _ = net(frames, None)`, binary_test.py:84-88) at `ticks` x `crops` frames per call (40 x 10 = 400 by
default), RGB, seeded synthetic weights and frames (oracle/inception_v3_oracle.py, oracle/synth.py), in EXACT_TC (split
fp16 operands on the tensor cores, fp32-grade), FAST_FP16 (fp16 operands) and EXACT_FP32 (fp32 SIMT).  CUDA events around
each call after `warmup` calls, median reported.  FLOP/s from the network's 5.711 GMAC (11.42 GFLOP) per frame:
`conv_tflops` is that algorithmic rate, `tensor_pipe_tflops` what the tensor cores issue (EXACT_TC: three MMAs per product;
FAST: one; EXACT_FP32 uses no tensor core).  The card's name, power limit and SM clocks are read in the same run.  Needs a
CUDA device: without one it fails.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

GMAC_PER_FRAME = 5.711


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def _time(fn, calls, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], ms[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--crops", type=int, default=10)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_inception_v3.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    import binary_model
    import ssn_models
    from oracle import inception_v3_oracle as IV
    from oracle import synth, binary_oracle as B
    dev = torch.device("cuda:0")
    F = args.ticks * args.crops
    w = IV.synth_weights(3, seed=0)
    x = synth.synth_frames(F, 3, IV.INPUT_SIZE, seed=3).to(dev)

    from ssn_b200 import _lib
    ssn = ssn_models.SSN(20, 2, 5, 2, "RGB", base_model="InceptionV3", dropout=0, test_mode=True)
    sd = ssn.state_dict()
    with torch.no_grad():
        for k, v in w.items():
            sd["base_model." + k].copy_(v)
        for k, v in synth.synth_heads(20, ssn.stpp.feat_multiplier, feat_dim=IV.FEAT_DIM, seed=0, std=0.02, bias_std=0.1).items():
            sd[k].copy_(v)
    ssn.prepare_test_fc()
    ssn = ssn.to(dev).eval()
    bc = binary_model.BinaryClassifier(2, 5, "RGB", base_model="InceptionV3", dropout=0, test_mode=True)
    bsd = bc.state_dict()
    with torch.no_grad():
        for k, v in w.items():
            bsd["base_model." + k].copy_(v)
        for k, v in B.synth_classifier(2, feat_dim=IV.FEAT_DIM, seed=0).items():
            bsd[k].copy_(v)
    bc.prepare_test_fc()
    bc = bc.to(dev).eval()

    def score_ssn():
        ssn.test_scores(x, num_crop=args.crops)

    def score_binary():
        with torch.no_grad():
            bc(x, None)

    line = {"workload": "inception_v3_test_time", "frames_per_call": F, "ticks": args.ticks, "crops": args.crops,
            "gmac_per_frame": GMAC_PER_FRAME}
    for pname, prec, mmas in (("exact_tc", _lib.EXACT_TC, 3), ("fast", _lib.FAST_FP16, 1), ("exact_fp32", _lib.EXACT_FP32, 0)):
        res = {}
        for name, model, fn in (("ssn_test_scores", ssn, score_ssn), ("binary_scores", bc, score_binary)):
            ssn.set_precision(prec); bc.set_precision(prec)    # drops both models' engines: one planned engine on the card at a time
            torch.cuda.empty_cache()
            med, best = _time(fn, args.calls, args.warmup)
            tf = 2 * GMAC_PER_FRAME * 1e9 * F / (med * 1e-3) / 1e12
            res[name] = {"ms_per_call": round(med, 3), "ms_best": round(best, 3), "frames_per_s": round(F / med * 1e3, 1),
                         "conv_tflops": round(tf, 2), "tensor_pipe_tflops": round(tf * mmas, 2)}
            res["workspace_bytes"] = model.base_model.engine_for(F, dev).workspace_bytes
        line[pname] = res
    line["card"] = card_info()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
