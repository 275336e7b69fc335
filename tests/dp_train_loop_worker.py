"""torchrun worker of tests/test_dp_train_loop.py (2 ranks, NCCL): BinaryClassifier.fused_step on each rank's half of a
4-video batch with GradSync, then FusedSGD.step(max_norm=...) after sync.finish(); rank 0 also runs the single-GPU step on
the global batch and compares the norms."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "action-detection_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def make(dev, bb):
    import binary_model
    from oracle import binary_oracle as B
    from ssn_b200 import _lib
    from ssn_b200.optim import FusedSGD
    m = binary_model.BinaryClassifier(2, 5, "RGB", base_model="BNInception", dropout=0)
    sd = m.state_dict()
    for k, v in bb.items():
        sd["base_model." + k].copy_(v)
    for k, v in B.synth_classifier(2, seed=0).items():
        sd[k].copy_(v)
    m = m.to(dev).train()
    m.set_precision(_lib.EXACT_TC, 1024.0)
    order = [p for p in m.parameters() if p.requires_grad]
    opt = FusedSGD(m.get_optim_policies(), lr=1e-3, momentum=0.9, weight_decay=5e-4, order=order)
    return m, opt, order


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    import datetime
    dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=180))
    from oracle import binary_oracle as B
    from oracle import synth
    from ssn_b200.dp import GradSync
    bb = synth.synth_backbone(3, seed=0, calib_frames=2)
    x, target = B.synth_binary_batch(4, 4, 2, 3, seed=9)
    half = x.shape[0] // world
    m, opt, order = make(dev, bb)
    sync = GradSync(opt.flat_grad, order, m)
    m.fused_step(x[rank * half:(rank + 1) * half].to(dev), target[rank * half:(rank + 1) * half].to(dev), loss_scale=1.0 / world,
                 grad_sync=sync)
    sync.finish()
    norm = opt.step(max_norm=1e-3).clone()
    norms = [torch.zeros_like(norm) for _ in range(world)]
    dist.all_gather(norms, norm)
    if rank == 0:
        m1, opt1, _ = make(dev, bb)
        m1.fused_step(x.to(dev), target.to(dev))
        ref = opt1.step(max_norm=1e-3)
        r = {"rank_norms": [float(n) for n in norms], "rank_norms_bitwise_equal": all(torch.equal(norms[0], n) for n in norms),
             "global_norm": float(ref), "rel_vs_global": abs(float(norms[0]) - float(ref)) / float(ref)}
        print("DP_TRAIN_LOOP_RESULT " + json.dumps(r), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
