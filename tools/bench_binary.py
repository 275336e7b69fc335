#!/usr/bin/env python
"""Benchmark of the TAG actionness classifier (BinaryClassifier) on one H100; prints ONE JSON line.

  python tools/bench_binary.py [--steps K] [--warmup W] [--ticks 40] [--crops 10]

Training: BinaryClassifier.fused_step + ssn_b200.optim.FusedSGD captured in one CUDA graph at the reference's training
shape (binary_train.py:25,91 and load_binary_score.py:84-92): 4 videos x 12 proposals x 5 segments = 48 proposals = 240 RGB
frames per step, K=2 (THUMOS14), dropout 0.8, frozen BN.  Measured in EXACT_TC (the headline, fp32-grade) and FAST (fp16
operands).  CUDA events around each replayed step, the L2 flushed (256 MiB write) outside the event pairs, as bench.py does.
Scoring: the loop body of binary_test.py:84-88, `rst, _ = net(frames, None)` after prepare_test_fc, at `ticks` x `crops`
frames per call (40 x 10 = 400 by default), in EXACT_TC and FAST.  Synthetic seeded weights and frames (oracle/synth.py).
The card's name, power limit and SM clocks are read in the same run.  Needs a CUDA device: without one it fails.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

VIDEOS, PROPS, SEG, K, DROPOUT = 4, 12, 5, 2, 0.8


def _bench_module():
    spec = importlib.util.spec_from_file_location("bench_main", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], "--query-gpu=" + q,
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    c = [t.strip() for t in out.split(",")]
    if len(c) < 4:
        return {"nvidia_smi": out or None}
    return {"name": c[0], "power_limit_w": c[1], "sm_mhz_idle": c[2], "sm_max_mhz": c[3]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--crops", type=int, default=10)
    ap.add_argument("--score-calls", type=int, default=20)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_binary.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    import binary_model
    from ssn_b200 import _lib
    from ssn_b200.optim import FusedSGD
    from oracle import binary_oracle as B
    from oracle import synth
    bench = _bench_module()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    prec = {"exact_tc": _lib.EXACT_TC, "fast": _lib.FAST_FP16}
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    l2_flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def make(precision, test_mode=False):
        torch.manual_seed(0)
        m = binary_model.BinaryClassifier(K, SEG, "RGB", base_model="BNInception", dropout=DROPOUT, test_mode=test_mode)
        sd = m.state_dict()
        for k, v in bb.items():
            sd["base_model." + k].copy_(v)
        m = m.to(dev)
        m.set_precision(prec[precision], 4096.0)
        return m

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * steps)]
        out = None
        with bench.ClockSampler(0) as clocks:
            for i in range(steps):
                l2_flush.zero_()
                ev[2 * i].record()
                out = fn()
                ev[2 * i + 1].record()
            torch.cuda.synchronize()
        return sum(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(steps)) / steps, clocks.summary(), out

    batches = [tuple(t.to(dev) for t in B.synth_binary_batch(VIDEOS, PROPS, K, 3, SEG, seed=i)) for i in range(2)]
    frames = VIDEOS * PROPS * SEG
    train = {}
    for precision in ("exact_tc", "fast"):
        m = make(precision).train()
        order = [p for p in m.parameters() if p.requires_grad]
        opt = FusedSGD(m.get_optim_policies(), lr=1e-5, momentum=0.9, weight_decay=5e-4, order=order,
                       on_step=[m.base_model.invalidate_packed])
        static = tuple(torch.empty_like(t) for t in batches[0])

        def step():
            opt.flat_grad.zero_()
            loss = m.fused_step(*static)
            opt.step()
            return loss
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(3):
                for d_, s_ in zip(static, batches[i % 2]):
                    d_.copy_(s_)
                step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_loss = step()
        it = [0]

        def replay():
            for d_, s_ in zip(static, batches[it[0] % 2]):
                d_.copy_(s_)
            it[0] += 1
            graph.replay()
            return static_loss
        ms, clocks, loss = timed(replay, args.steps, args.warmup)
        l0 = _lib.lib.ssnb_global_launch_count()
        step()
        torch.cuda.synchronize()
        train[precision] = {"ms_per_step": ms, "proposals_per_s": VIDEOS * PROPS / (ms / 1e3), "frames_per_s": frames / (ms / 1e3),
                            "loss": float(loss.item()), "library_launches_per_step": int(_lib.lib.ssnb_global_launch_count() - l0),
                            "clocks": clocks}
        del m, opt, graph
        torch.cuda.empty_cache()

    score = {}
    nf = args.ticks * args.crops
    chunk = synth.synth_frames(nf, 3, seed=9).to(dev)
    for precision in ("exact_tc", "fast"):
        net = make(precision, test_mode=True)
        net.prepare_test_fc()
        net.eval()

        def call():
            with torch.no_grad():
                rst, _ = net(chunk, None)
            return rst
        ms, clocks, rst = timed(call, args.score_calls, 3)
        score[precision] = {"ms_per_call": ms, "frames_per_s": nf / (ms / 1e3), "clocks": clocks,
                            "scores_finite": bool(torch.isfinite(rst).all())}
        del net
        torch.cuda.empty_cache()

    line = {"metric": "binary_classifier_train_proposals_per_s", "value": train["exact_tc"]["proposals_per_s"], "unit": "proposals/s",
            "higher_is_better": True, "precision": "exact_tc", "steps": args.steps, "warmup": args.warmup,
            "config": {"videos": VIDEOS, "proposals_per_video": PROPS, "segments": SEG, "frames_per_step": frames, "num_class": K,
                       "dropout": DROPOUT, "modality": "RGB", "bn_mode": "frozen", "cuda_graph": True,
                       "l2": "flushed between timed steps (256 MiB write)", "score_frames_per_call": nf, "data": "synthetic"},
            "train": train, "score": score, "card": card_info(), "torch": torch.__version__}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
