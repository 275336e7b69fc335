"""Generate tests/golden/binary.npz from the REAL reference BinaryClassifier (binary_model.py of yjxiong/action-detection).

Run where a checkout of the reference exists:  python -m oracle.gen_golden_binary
The four external patches of oracle/gen_golden.py are applied (no reference file is edited), plus one more:
binary_model.py:120 uses `Identity` without importing it, so ops.ssn_ops.Identity is injected into the module's namespace
from outside.  The model is built with dropout=0 and seeded synthetic weights (oracle/synth.py, oracle/binary_oracle.py).

Cases: RGB with K=2 at 2 videos x 4 proposals x 5 segments, Flow (2x5 channels) with K=100 at 2 x 2 x 5.  Stored per case:
state_dict keys (before and after prepare_test_fc), optimiser group sizes, raw scores, targets, the CrossEntropyLoss, every
convolution / classifier_fc gradient (sum and absolute sum; conv1 and classifier_fc in full) and test_forward outputs of the
first 4 frames.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
CASES = (("rgb", "RGB", 3, 2, 2, 4), ("flow", "Flow", 10, 100, 2, 2))     # tag, modality, channels, K, videos, proposals
SEG = 5


def main():
    sys.path.insert(0, os.path.dirname(HERE))
    from oracle import gen_golden, synth, binary_oracle as B
    _ssn_models, R, _pl = gen_golden.import_reference()
    import binary_model
    binary_model.Identity = R.Identity          # patch 5: binary_model.py:120 uses Identity without importing it
    torch.manual_seed(0)
    out = {}
    for tag, modality, C, K, V, P in CASES:
        with contextlib.redirect_stdout(io.StringIO()):
            model = binary_model.BinaryClassifier(K, SEG, modality, base_model="BNInception", dropout=0, bn_mode="frozen")
        sd = model.state_dict()
        with torch.no_grad():
            for k, v in synth.synth_backbone(C, seed=0).items():
                assert sd["base_model." + k].shape == v.shape, k
                sd["base_model." + k].copy_(v)
            for k, v in B.synth_classifier(K, seed=0).items():
                sd[k].copy_(v)
        t = tag + "_"
        out[t + "sd_keys"] = np.array(list(model.state_dict().keys()))
        out[t + "policy_sizes"] = np.array([len(g["params"]) for g in model.get_optim_policies()])
        model.train()
        x, target = B.synth_binary_batch(V, P, K, C, SEG, seed=0)
        raw, tgt = model(x, target)
        loss = torch.nn.CrossEntropyLoss()(raw, tgt)
        loss.backward()
        names, gsum, gabs = [], [], []
        for n_, p_ in model.named_parameters():
            if p_.grad is None or "_bn." in n_:           # frozen BatchNorm2d weights get a gradient only through :214's typo
                continue
            names.append(n_); gsum.append(p_.grad.double().sum().item()); gabs.append(p_.grad.double().abs().sum().item())
        out.update({t + "raw": raw.detach().numpy(), t + "target": tgt.numpy(), t + "loss": np.float64(loss.item()),
                    t + "grad_names": np.array(names), t + "grad_sum": np.array(gsum), t + "grad_abs": np.array(gabs),
                    t + "g_conv1_w": model.base_model.conv1_7x7_s2.weight.grad.numpy(),
                    t + "g_conv1_b": model.base_model.conv1_7x7_s2.bias.grad.numpy(),
                    t + "g_cls_w": model.classifier_fc.weight.grad.numpy(),
                    t + "g_cls_b": model.classifier_fc.bias.grad.numpy()})
        model.prepare_test_fc()
        out[t + "sd_keys_test"] = np.array(list(model.state_dict().keys()))
        out[t + "test_shares_storage"] = np.bool_(model.test_fc.weight.data_ptr() == model.classifier_fc.weight.data_ptr())
        model.eval()
        model.test_mode = True
        with torch.no_grad():
            scores, base_out = model(x.view(-1, C, 224, 224)[:4], None)
        out[t + "test_scores"], out[t + "test_base"] = scores.numpy(), base_out.numpy()
    np.savez_compressed(os.path.join(GOLD, "binary.npz"), **out)
    print("golden written to", os.path.join(GOLD, "binary.npz"))


if __name__ == "__main__":
    main()
