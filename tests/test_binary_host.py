"""BinaryClassifier (TAG actionness) without a GPU: the CPU oracle against the reference's own outputs
(tests/golden/binary.npz, oracle/gen_golden_binary.py), and the drop-in module's surface against the reference's."""
import os

import numpy as np
import pytest
import torch

from oracle import binary_oracle as B
from oracle import synth

CASES = [("rgb", "RGB", 3, 2, 2, 4), ("flow", "Flow", 10, 100, 2, 2)]       # tag, modality, channels, K, videos, proposals


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "binary.npz"), allow_pickle=False)


@pytest.mark.parametrize("tag,modality,C,K,V,P", CASES)
def test_oracle_matches_reference(golden_dir, tag, modality, C, K, V, P):
    """oracle: backbone -> segment mean -> classifier_fc -> CrossEntropyLoss, forward and backward, at the bars
    test_oracle_golden uses for the whole-SSN case"""
    z, t = _golden(golden_dir), tag + "_"
    bb = synth.synth_backbone(C, seed=0)
    hd = B.synth_classifier(K, seed=0)
    for d in (bb, hd):
        for k in d:
            if "_bn." not in k:
                d[k].requires_grad_(True)
    x, target = B.synth_binary_batch(V, P, K, C, seed=0)
    raw, tgt = B.binary_train_forward(bb, hd, x, target, in_channels=C)
    loss = B.cross_entropy(raw, tgt)
    np.testing.assert_allclose(raw.detach().numpy(), z[t + "raw"], rtol=2e-4, atol=2e-5)
    np.testing.assert_array_equal(tgt.numpy(), z[t + "target"])
    np.testing.assert_allclose(loss.item(), float(z[t + "loss"]), rtol=2e-5)
    loss.backward()
    np.testing.assert_allclose(bb["conv1_7x7_s2.weight"].grad.numpy(), z[t + "g_conv1_w"], rtol=2e-3, atol=2e-6)
    np.testing.assert_allclose(hd["classifier_fc.weight"].grad.numpy(), z[t + "g_cls_w"], rtol=2e-4, atol=1e-7)
    np.testing.assert_allclose(hd["classifier_fc.bias"].grad.numpy(), z[t + "g_cls_b"], rtol=2e-4, atol=1e-7)
    names = [str(s) for s in z[t + "grad_names"]]
    assert len(names) == 2 * 69 + 2
    for n_, ga in zip(names, z[t + "grad_abs"]):
        p = bb[n_[len("base_model."):]] if n_.startswith("base_model.") else hd[n_]
        assert abs(p.grad.double().abs().sum().item() - ga) <= 2e-4 * ga + 1e-9, n_
    with torch.no_grad():
        scores, base = B.binary_test_forward(bb, hd, x.view(-1, C, 224, 224)[:4], C)
    np.testing.assert_allclose(base.numpy(), z[t + "test_base"], rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(scores.numpy(), z[t + "test_scores"], rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize("tag,modality,C,K,V,P", CASES)
def test_module_surface_matches_reference(golden_dir, tag, modality, C, K, V, P):
    """state_dict keys (also after prepare_test_fc, whose test_fc shares classifier_fc's tensors), optimiser group sizes
    and the attributes binary_train.py / binary_test.py read"""
    import binary_model
    z, t = _golden(golden_dir), tag + "_"
    m = binary_model.BinaryClassifier(K, 5, modality, base_model="BNInception", dropout=0)
    assert list(m.state_dict().keys()) == [str(k) for k in z[t + "sd_keys"]]
    assert [len(g["params"]) for g in m.get_optim_policies()] == z[t + "policy_sizes"].tolist()
    assert m.num_segments == m.course_segment == 5 and m.new_length == (1 if modality == "RGB" else 5)
    assert m.base_model.in_channels() == C and m.feature_dim == 1024 and m.test_fc is None
    assert (m.crop_size, m.scale_size, m.input_std) == (224, 256, [1])
    assert m.input_mean == ([104, 117, 128] if modality == "RGB" else [128])
    assert m.train() is m
    assert all(not b.training and not b.weight.requires_grad and not b.bias.requires_grad
               for b in m.base_model.modules() if isinstance(b, torch.nn.BatchNorm2d))
    m.prepare_test_fc()
    assert list(m.state_dict().keys()) == [str(k) for k in z[t + "sd_keys_test"]]
    assert bool(z[t + "test_shares_storage"])
    assert m.test_fc.weight.data_ptr() == m.classifier_fc.weight.data_ptr()
    assert m.test_fc.bias.data_ptr() == m.classifier_fc.bias.data_ptr()
    # a training checkpoint loads the way binary_test.py:126 loads one (DataParallel's `module.` prefix stripped)
    ckpt = {"module." + k: v for k, v in m.state_dict().items() if not k.startswith("test_fc.")}
    m2 = binary_model.BinaryClassifier(K, 5, modality, base_model="BNInception", test_mode=True)
    m2.load_state_dict({'.'.join(k.split('.')[1:]): v for k, v in ckpt.items()})
    assert torch.equal(m2.classifier_fc.weight, m.classifier_fc.weight)


def test_unsupported_configurations_raise():
    import binary_model
    with pytest.raises(ValueError):
        binary_model.BinaryClassifier(2, 5, "RGB", base_model="resnet101")
    with pytest.raises(ValueError):
        binary_model.BinaryClassifier(2, 5, "RGB")                         # the reference's default base model
    for modality in ("RGBDiff", "Depth"):
        with pytest.raises(ValueError):
            binary_model.BinaryClassifier(2, 5, modality, base_model="BNInception")
    with pytest.raises(ValueError):
        binary_model.BinaryClassifier(2, 5, "RGB", base_model="BNInception", bn_mode="nope")
    full = binary_model.BinaryClassifier(2, 5, "RGB", base_model="BNInception", bn_mode="full").train()
    with pytest.raises(NotImplementedError):
        full.base_model.bn1_training()
    m = binary_model.BinaryClassifier(2, 5, "RGB", base_model="BNInception")
    with pytest.raises(RuntimeError):                                      # no CPU fallback
        m(torch.zeros(1, 5 * 3, 224, 224), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(RuntimeError):
        m.fused_step(torch.zeros(1, 5 * 3, 224, 224), torch.zeros(1, dtype=torch.int64))


def test_classifier_ce_arguments_are_validated():
    """the CE entry point rejects bad shapes and NULL buffers with an error code before touching the device"""
    from ssn_b200 import _lib
    lib = _lib.lib
    assert lib.ssnb_classifier_ce_workspace_bytes(48, 2) >= 48 * 2 * 4 + 48 * 8
    assert lib.ssnb_classifier_ce_workspace_bytes(0, 2) == 0
    p = 256                                                                # never dereferenced: validation fails first
    assert lib.ssnb_classifier_ce_fwd_bwd(p, p, p, p, 0, 1024, 2, 1.0, p, p, p, p, p, p, None) == 1
    assert lib.ssnb_classifier_ce_fwd_bwd(p, p, p, p, 4, 1024, 5000, 1.0, p, p, p, p, p, p, None) == 1
    assert lib.ssnb_classifier_ce_fwd_bwd(p, p, p, p, 4, 1024, 2, 1.0, p, p, p, p, p, None, None) == 1
    assert b"classifier_ce" in lib.ssnb_last_error(None)
    # zero STPP parts: a course-only call must still name the course output (and, backward, d_course)
    assert lib.ssnb_stpp_bwd(None, None, None, 1, 5, 1024, 0, None, None, None, None, 0, 5, p, None) == 1
    assert lib.ssnb_stpp_fwd(p, None, 1, 5, 1024, 0, None, None, None, None, 0, 5, None, None, None) == 1
