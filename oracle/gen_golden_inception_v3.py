"""Write tests/golden/inception_v3.json and tests/golden/inception_v3.npz from the REAL reference InceptionV3
(model_zoo/bninception/pytorch_load.py:64-67 with inceptionv3.yaml, ssn_models.py:133-139, binary_model.py:175-178) and
its transforms.py, vendored under oracle/_ref (oracle/ref_harness.py).  No weights are stored: they are regenerated from
the seed (oracle/inception_v3_oracle.synth_weights, oracle/synth.synth_heads, oracle/binary_oracle.synth_classifier).

Patches, all applied from outside the reference: the four of oracle/gen_golden.py (among them BNInception.load_state_dict
-> no-op, which InceptionV3 inherits: load_url returns None offline), Identity injected into binary_model
(oracle/gen_golden_binary.py) and torchvision.transforms.Scale = Resize (oracle/gen_golden_frames.py).

json: the yaml's layer list as the reference parsed it, the backbone's children in order and its state_dict keys / shapes
for RGB and Flow.  npz, per modality (rgb: K = 4, Flow: 2x5 channels, K = 3), 10 seeded 299x299 frames through
SSN(..., 'InceptionV3', test_mode=True) after prepare_test_fc: base_out [10, 2048] and the test_fc output; BinaryClassifier
(K = 2) test_forward scores; and the SHA-256 of the reference's GroupOverSample(299, 341) and GroupScale(341) +
GroupCenterCrop(299) outputs on seeded 340x256 RGB and Flow frames.

    python oracle/gen_golden_inception_v3.py
"""
import contextlib
import hashlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, "tests", "golden")
# tag, modality, in_channels, SSN num_class, frames seed
CASES = (("rgb", "RGB", 3, 4, 11), ("flow", "Flow", 10, 3, 12))
N_FRAMES = 10
# frame-transform cases: (name, kind, seed, (images, h, w, c), mean)
FRAME_CASES = (("oversample_rgb", "oversample", 2300, (2, 256, 340, 3), [104, 117, 128]),
               ("oversample_flow", "oversample", 2301, (4, 256, 340, 1), [128]),
               ("center_rgb", "center", 2302, (2, 256, 340, 3), [104, 117, 128]),
               ("center_flow", "center", 2303, (4, 256, 340, 1), [128]))


def main():
    sys.path.insert(0, ROOT)
    from oracle import ref_harness
    if not ref_harness.available():
        ref_harness.vendor()
    from oracle import gen_golden, gen_golden_frames as GF, synth, binary_oracle as B, inception_v3_oracle as IV
    T = GF.load_reference_transforms()
    frames_out = {}
    for name, kind, seed, shape, mean in FRAME_CASES:
        out, _ = GF.run_reference(T, kind, GF.frames_for(seed, *shape), dict(out=299, scale=341, mean=mean))
        frames_out[name] = dict(kind=kind, seed=seed, shape=list(shape), mean=mean, out_shape=list(out.shape),
                                sha256=hashlib.sha256(np.ascontiguousarray(out, np.float32).tobytes()).hexdigest())
    cwd = os.getcwd()
    ssn_models, R, pl = gen_golden.import_reference()
    import binary_model
    binary_model.Identity = R.Identity
    torch.manual_seed(0)

    with contextlib.redirect_stdout(io.StringIO()):
        net = pl.InceptionV3()
    import yaml
    manifest = yaml.load(open("model_zoo/bninception/inceptionv3.yaml"))
    layer_list = []
    for l in manifest["layers"]:
        out, op, ins = l["expr"].split("<=")
        layer_list.append([l["id"], op, out, ins.split(","), l.get("attrs", {})])
    graph = {"layers": layer_list, "children": [n for n, _ in net.named_children()], "state_dict": {}}

    arrays = {}
    for tag, modality, C, K, fseed in CASES:
        with contextlib.redirect_stdout(io.StringIO()):
            model = ssn_models.SSN(K, 2, 5, 2, modality, base_model="InceptionV3", dropout=0, test_mode=True)
        sd = model.state_dict()
        graph["state_dict"][tag] = [[k, list(v.shape)] for k, v in sd.items()]
        graph["input_" + tag] = dict(input_size=model.input_size, input_mean=model.input_mean, input_std=model.input_std,
                                     crop_size=model.crop_size, scale_size=model.scale_size)
        bb = IV.synth_weights(C, seed=0)
        hd = synth.synth_heads(K, model.stpp.feat_multiplier, feat_dim=IV.FEAT_DIM, seed=0, std=0.02, bias_std=0.1)
        with torch.no_grad():
            for k, v in bb.items():
                assert sd["base_model." + k].shape == v.shape, k
                sd["base_model." + k].copy_(v)
            for k, v in hd.items():
                sd[k].copy_(v)
        model.prepare_test_fc()
        model.eval()
        x = synth.synth_frames(N_FRAMES, C, IV.INPUT_SIZE, seed=fseed)
        with torch.no_grad():
            out, base_out = model(x, None, None, None, None)
        arrays[tag + "_base_out"], arrays[tag + "_test_fc"] = base_out.numpy(), out.numpy()

        with contextlib.redirect_stdout(io.StringIO()):
            bc = binary_model.BinaryClassifier(2, 5, modality, base_model="InceptionV3", dropout=0, test_mode=True)
        bsd = bc.state_dict()
        with torch.no_grad():
            for k, v in bb.items():
                bsd["base_model." + k].copy_(v)
            for k, v in B.synth_classifier(2, feat_dim=IV.FEAT_DIM, seed=0).items():
                bsd[k].copy_(v)
        bc.prepare_test_fc()
        bc.eval()
        with torch.no_grad():
            scores, bbase = bc(x, None)
        arrays[tag + "_binary_scores"], arrays[tag + "_binary_base"] = scores.numpy(), bbase.numpy()
    graph["frames"] = frames_out
    os.chdir(cwd)
    with open(os.path.join(GOLD, "inception_v3.json"), "w") as f:
        json.dump(graph, f, indent=0, sort_keys=True)
    np.savez_compressed(os.path.join(GOLD, "inception_v3.npz"), **arrays)
    print("golden written to", GOLD)


if __name__ == "__main__":
    main()
