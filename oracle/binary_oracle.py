"""CPU oracle for the TAG actionness classifier (BinaryClassifier).  TEST INFRASTRUCTURE ONLY (same rules as
oracle/ssn_oracle.py: tests/, smoke() and the benchmarks may import it; the product never does).

A restatement, on CPU (torch CPU ops, fp32), of binary_model.py of yjxiong/action-detection:
    train_forward :226-234   BNInception -> fc (Dropout / Identity) -> view(-1, course_segment, 1024).mean(1) -> classifier_fc
    test_forward  :237-240   (test_fc(base_out), base_out) per frame, test_fc sharing classifier_fc's tensors (:245-254)
and of the loss of binary_train.py:135,162 (torch.nn.CrossEntropyLoss(), mean).  Pinned against the reference's own
outputs by oracle/gen_golden_binary.py -> tests/golden/binary.npz.
"""
import torch
import torch.nn.functional as F

from . import ssn_oracle as O
from . import synth


def synth_classifier(num_class, feat_dim=1024, seed=0, std=0.02, bias_std=0.1):
    """classifier_fc, N(0, std) weights like binary_model.py:127-128 (larger std and a bias give the tests non-trivial values)"""
    g = torch.Generator().manual_seed(5000 + seed)
    return {"classifier_fc.weight": torch.randn(num_class, feat_dim, generator=g) * std,
            "classifier_fc.bias": torch.randn(num_class, generator=g) * bias_std}


def synth_binary_batch(n_videos, props, num_class, in_channels=3, course_segment=5, size=224, seed=0):
    """One batch shaped like BinaryDataSet's (load_binary_score.py:223-262): x [videos, props*S*C, H, W], target [videos,
    props] -- the first quarter of each video's proposals foreground (class >= 1 when num_class > 2, else 1), the rest 0."""
    g = torch.Generator().manual_seed(6000 + seed)
    frames = synth.synth_frames(n_videos * props * course_segment, in_channels, size, seed=seed)
    x = frames.view(n_videos, props * course_segment * in_channels, size, size)
    target = torch.zeros(n_videos, props, dtype=torch.int64)
    n_fg = max(1, props // 4)
    target[:, :n_fg] = torch.randint(1, num_class, (n_videos, n_fg), generator=g) if num_class > 2 else 1
    return x, target


def binary_train_forward(params, head, x, target, course_segment=5, in_channels=3, mask=None, taps=None, bn_train_first=False):
    """BinaryClassifier.train_forward: returns (raw scores [n, K], target.view(-1)).  mask: the dropout mask (already divided
    by the keep probability) applied to the backbone output, as nn.Dropout(p) in training mode does.  bn_train_first:
    bn_mode='partial' (see ssn_oracle.backbone_forward)."""
    frames = x.view((-1, in_channels) + tuple(x.shape[-2:]))
    base_out = O.backbone_forward(params, frames, in_channels, bn_train_first=bn_train_first)
    if mask is not None:
        base_out = base_out * mask
    course_ft = base_out.view(-1, course_segment, base_out.size(1)).mean(dim=1)
    if taps is not None:
        taps["base_out"], taps["course_ft"] = base_out, course_ft
    return F.linear(course_ft, head["classifier_fc.weight"], head["classifier_fc.bias"]), target.view(-1)


def cross_entropy(raw, target):
    """torch.nn.CrossEntropyLoss() (binary_train.py:135): mean over rows"""
    return F.cross_entropy(raw, target)


def binary_test_forward(params, head, frames, in_channels=3):
    """BinaryClassifier.test_forward after prepare_test_fc: (per-frame scores [F, K], base_out [F, 1024])"""
    base_out = O.backbone_forward(params, frames.view((-1, in_channels) + tuple(frames.shape[-2:])), in_channels)
    return F.linear(base_out, head["classifier_fc.weight"], head["classifier_fc.bias"]), base_out
