"""What the rest of the training step costs around SSN.fused_step at config [1]'s shape (4 videos x 8 proposals x 9 segments,
K=20; 288 frames), EXACT_TC and FAST_FP16, as the median over windows of the per-step time:

  reference   the loop of ssn_train.py:207-250 on the module surface: fused_step, torch.nn.utils.clip_grad_norm_ over
              model.parameters() with its `if total_norm > clip` check, the loop's .item() meters (four losses and three
              accuracies), FusedSGD.step(); eager
  device      fused_step(meters=StepMeters) + FusedSGD.step(max_norm=...) in one CUDA graph, replayed
  plain       fused_step + FusedSGD.step() in one CUDA graph (bench.py's step: no clip, no meters)
  eval_fused  SSN.fused_eval, eager (validate()'s body)
  eval_module the module path under torch.no_grad(): model(...) and the three criteria, eager

One JSON line.  The card's name, power limit and SM clocks are read in the same run.  Needs a CUDA device: without one it
fails."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

VIDEOS, K, CLIP = 4, 20, 10.0           # the gradient norm of this batch is about 12: the device loop clips


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10, help="steps per window")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_train_loop.py measures the H100 path and needs a CUDA device; there is no CPU fallback")
    import ssn_models
    from bench_binary import card_info
    from ops.ssn_ops import ClassWiseRegressionLoss, CompletenessLoss
    from ssn_b200 import _lib
    from ssn_b200.meters import StepMeters
    from ssn_b200.optim import FusedSGD
    from oracle import synth
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    batch = tuple(t.to(dev) for t in synth.synth_batch(VIDEOS, K, seed=0))
    act_crit, comp_crit, reg_crit = torch.nn.CrossEntropyLoss(), CompletenessLoss(), ClassWiseRegressionLoss()

    def make(precision):
        torch.manual_seed(0)
        m = ssn_models.SSN(K, 2, 5, 2, "RGB", base_model="BNInception", dropout=0.8)
        sd = m.state_dict()
        for k, v in bb.items():
            sd["base_model." + k].copy_(v)
        m = m.to(dev).train()
        m.set_precision(precision, 4096.0)
        order = [p for p in m.parameters() if p.requires_grad]
        opt = FusedSGD(m.get_optim_policies(), lr=1e-6, momentum=0.9, weight_decay=5e-4, order=order,
                       on_step=[m.base_model.invalidate_packed])
        return m, opt

    def windows(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        per_step = []
        for _ in range(args.windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                fn()
            b.record()
            torch.cuda.synchronize()
            per_step.append(a.elapsed_time(b) / args.steps)
        return round(statistics.median(per_step), 3)

    def graphed(fn):
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g

    def accuracy(output, target):
        _, pred = output.topk(1, 1, True, True)
        return pred.t().eq(target.view(1, -1)).view(-1).float().sum(0).mul_(100.0 / target.size(0))

    res = {}
    for name, prec in (("exact_tc", _lib.EXACT_TC), ("fast", _lib.FAST_FP16)):
        m, opt = make(prec)
        r = {}

        def reference():
            opt.flat_grad.zero_()
            losses = m.fused_step(*batch)
            total_norm = torch.nn.utils.clip_grad_norm_(m.parameters(), CLIP)
            if float(total_norm) > CLIP:
                pass                                     # the reference prints here
            for v in losses:
                v.item()
            tp = batch[4].view(-1)
            sel = ((tp == 0) | (tp == 2)).nonzero().view(-1)
            act, tg = m.last_fused["raw_act"][sel], batch[2].view(-1)[sel]
            accuracy(act, tg).item()
            accuracy(act.view(-1, 2, act.size(1))[:, 0, :].contiguous(), tg.view(-1, 2)[:, 0].contiguous()).item()
            accuracy(act.view(-1, 2, act.size(1))[:, 1, :].contiguous(), tg.view(-1, 2)[:, 1].contiguous()).item()
            opt.step()
        r["reference_ms"] = windows(reference)

        meters = StepMeters("ssn", dev)

        def device():
            opt.flat_grad.zero_()
            m.fused_step(*batch, meters=meters)
            opt.step(max_norm=CLIP)
        g = graphed(device)
        r["device_ms"] = windows(g.replay)
        del g

        def plain():
            opt.flat_grad.zero_()
            m.fused_step(*batch)
            opt.step()
        g = graphed(plain)
        r["plain_ms"] = windows(g.replay)
        del g

        m.eval()
        r["eval_fused_ms"] = windows(lambda: m.fused_eval(*batch))

        def module_eval():
            with torch.no_grad():
                a, at, c, ct, rg, rl, rt = m(*batch)
                return act_crit(a, at) + 0.1 * comp_crit(c, ct, 1, 7) + 0.1 * reg_crit(rg, rl, rt)
        r["eval_module_ms"] = windows(module_eval)
        r["norm"] = float(opt.norm)
        res[name] = r
        del m, opt
        torch.cuda.empty_cache()
    line = {"bench": "train_loop", "shape": {"videos": VIDEOS, "proposals": 8, "segments": 9, "frames": VIDEOS * 72, "K": K},
            "clip": CLIP, "windows": args.windows, "steps_per_window": args.steps, "results": res, "card": card_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
