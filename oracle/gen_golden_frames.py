"""Write tests/golden/frames.npz from the reference's own transforms.py and PIL (the vendored copy under oracle/_ref, see
oracle/ref_harness.py).  tests/test_frames_host.py checks oracle/frames_oracle.py against it and tests/test_gpu_frames.py
checks the GPU against the golden cases directly.

transforms.py is loaded unmodified.  Besides the four patches of oracle/ref_harness.py, it needs a fifth, applied here from
outside the reference:
  5. torchvision.transforms.Scale = torchvision.transforms.Resize   (transforms.py:93; Scale was removed from torchvision)

Small cases are stored whole (input frames, the parameters the reference drew, its output).  Full-size cases (340x256 and
480x360 frames -> 224) are stored as the seed of their input frames plus the SHA-256 of the reference output bytes, which keeps
the file small.  `draws` holds the (crop_w, crop_h, offset_w, offset_h, flip) sequences the reference drew for fixed seeds.

    python oracle/gen_golden_frames.py
"""
import hashlib
import importlib.util
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "frames.npz")
RGB_MEAN, FLOW_MEAN = [104, 117, 128], [128]


def frames_for(seed, n, h, w, c):
    """the input frames of a hashed case: uint8 [n, h, w, c] from numpy's default_rng(seed)"""
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, c), dtype=np.uint8)


def load_reference_transforms():
    import torchvision
    torchvision.transforms.Scale = torchvision.transforms.Resize          # patch 5
    path = os.path.join(HERE, "_ref", "transforms.py")
    if not os.path.exists(path):
        raise SystemExit("oracle/_ref/transforms.py is missing: run __graft_entry__.build() where the reference is checked out")
    spec = importlib.util.spec_from_file_location("reference_transforms", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pil(frames):
    from PIL import Image
    return [Image.fromarray(f) if f.shape[2] == 3 else Image.fromarray(f[:, :, 0], "L") for f in frames]


def run_reference(T, kind, frames, case):
    """-> (output fp32 [planes, out, out], drawn params or None) of one group through the reference composition"""
    import torchvision
    drawn = {}

    class Recording(T.GroupMultiScaleCrop):
        def _sample_crop_size(self, im_size):
            drawn["crop"] = super()._sample_crop_size(im_size)
            return drawn["crop"]

    out = case["out"]
    if kind == "train":
        crop = Recording(out, case["scales"], fix_crop=case.get("fix_crop", True))
        flip = T.GroupRandomHorizontalFlip(is_flow=case["is_flow"])
        cropped = crop(_pil(frames))
        imgs = flip(cropped)                 # the same list unless it flipped (transforms.py:56-64)
        params = list(drawn["crop"]) + [int(imgs is not cropped)]
    elif kind == "oversample":
        imgs = T.GroupOverSample(out, case["scale"])(_pil(frames))
        params = None
    else:
        imgs = torchvision.transforms.Compose([T.GroupScale(case["scale"]), T.GroupCenterCrop(out)])(_pil(frames))
        params = None
    tail = torchvision.transforms.Compose([T.Stack(roll=True), T.ToTorchFormatTensor(div=False), T.GroupNormalize(case["mean"], [1])])
    return tail(imgs).numpy(), params


def main():
    T = load_reference_transforms()
    arrays, cases = {}, []
    rgb_scales, flow_scales = [1, .875, .75, .66], [1, .875, .75]

    def add(name, kind, frames=None, seed=None, shape=None, **case):
        case.update(name=name, kind=kind)
        case.setdefault("mean", FLOW_MEAN if case.get("is_flow") or (frames is not None and frames.shape[3] == 1)
                        or (shape is not None and shape[3] == 1) else RGB_MEAN)
        if frames is None:
            frames = frames_for(seed, *shape)
            case.update(seed=seed, shape=list(shape))
        random.seed(case.pop("rseed", 0))
        out, params = run_reference(T, kind, frames, case)
        case["params"] = params
        if seed is None:
            arrays["in_" + name] = frames
            arrays["out_" + name] = out
        else:
            case["sha256"] = hashlib.sha256(np.ascontiguousarray(out, np.float32).tobytes()).hexdigest()
            case["out_shape"] = list(out.shape)
        cases.append(case)

    rng = np.random.default_rng(12345)
    small = lambda n, h, w, c: rng.integers(0, 256, (n, h, w, c), dtype=np.uint8)
    for s in range(6):
        add("train_rgb_%d" % s, "train", small(2, 40, 52, 3), out=32, scales=rgb_scales, is_flow=False, rseed=s)
        add("train_flow_%d" % s, "train", small(4, 45, 30, 1), out=24, scales=flow_scales, is_flow=True, rseed=100 + s)
    for s in range(3):
        add("train_randint_%d" % s, "train", small(2, 37, 50, 3), out=24, scales=rgb_scales, is_flow=False, fix_crop=False, rseed=200 + s)
    for s in range(6):       # a shorter edge of 31: crops of 31 snap up to 32 and reach outside the frame
        add("train_snap_%d" % s, "train", small(2, 31, 44, 3), out=32, scales=rgb_scales, is_flow=False, rseed=300 + s)
    add("train_upsample", "train", small(2, 20, 17, 3), out=32, scales=rgb_scales, is_flow=False, rseed=3)
    add("oversample_resize", "oversample", small(2, 29, 21, 3), out=16, scale=20)
    add("oversample_plain", "oversample", small(2, 20, 27, 3), out=16, scale=20)
    add("oversample_flow", "oversample", small(4, 23, 34, 1), out=16, scale=19)
    for h, w in ((41, 60), (36, 45), (59, 36), (36, 36)):
        add("center_%dx%d" % (h, w), "center", small(2, h, w, 3), out=32, scale=36)
    # full size: 340x256 RGB and Flow frames (the bench shape) and 480x360 (GroupScale resizes)
    for s in range(3):
        add("full_train_rgb_%d" % s, "train", seed=1000 + s, shape=(3, 256, 340, 3), out=224, scales=rgb_scales, is_flow=False, rseed=s)
        add("full_train_flow_%d" % s, "train", seed=1100 + s, shape=(4, 256, 340, 1), out=224, scales=flow_scales, is_flow=True, rseed=s)
    add("full_oversample_340", "oversample", seed=1200, shape=(2, 256, 340, 3), out=224, scale=256)
    add("full_oversample_480", "oversample", seed=1201, shape=(2, 360, 480, 3), out=224, scale=256)
    add("full_center_480", "center", seed=1202, shape=(2, 360, 480, 3), out=224, scale=256)

    # the reference's draws for fixed seeds: groups of the given (H, W) in sequence
    sizes = [(256, 340), (240, 320), (360, 480), (223, 300), (256, 256)]
    draws = []
    for seed in range(4):
        for modality, scales in (("RGB", rgb_scales), ("Flow", flow_scales)):
            for fix_crop in (True, False):
                random.seed(seed)
                seq = []
                # randint offsets need the crop inside the image: not for a shorter edge that snaps up to 224
                sz = sizes if fix_crop else [x for x in sizes if min(x) >= 224]
                for h, w in sz:
                    c = 3 if modality == "RGB" else 1
                    _, p = run_reference(T, "train", np.zeros((2, h, w, c), np.uint8) + np.arange(w, dtype=np.uint8)[None, None, :, None],
                                         dict(out=224, scales=scales, is_flow=modality == "Flow", fix_crop=fix_crop, mean=[0]))
                    seq.append(p)
                draws.append(dict(seed=seed, scales=scales, fix_crop=fix_crop, sizes=sz, params=seq))
    arrays["cases"] = np.array(json.dumps(cases))
    arrays["draws"] = np.array(json.dumps(draws))
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(cases), "cases")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
