"""Write tests/golden/optical_flow.npz: what OpenCV computes for the two stages of oracle/tvl1_oracle.py that have a CPU
counterpart in cv2, after checking the oracle against it:

  grey     cv2.cvtColor(COLOR_RGB2GRAY) of a seeded random 64 x 64 RGB image (Pillow's 'L' rule differs on a few pixels of
           such an image) and of all 2^24 colours (checked here, too large to store)
  resize   cv2.resize(INTER_LINEAR) of a float32 grey frame down the pyramid of oracle.level_sizes at the default scale_step, and
           of a two-plane float32 flow up one level: the oracle's R3 within 1e-6 relative L2

The tests read only the npz, so OpenCV is needed only to regenerate it:  python -m oracle.gen_golden_flow
"""
import os

import numpy as np

from oracle import tvl1_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "optical_flow.npz")


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-300))


def main():
    import cv2
    rng = np.random.default_rng(0)
    out = {}
    a = np.arange(1 << 24, dtype=np.uint32)
    every = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert (O.grey(every) == cv2.cvtColor(every, cv2.COLOR_RGB2GRAY)).all(), "grey rule vs OpenCV on all colours"
    rgb = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    out["grey_rgb"], out["grey_cv2"] = rgb, cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)
    assert (O.grey(rgb) == out["grey_cv2"]).all()
    # a 96 x 128 frame down every level, each level from the previous cv2 level
    g = cv2.cvtColor(rng.integers(0, 256, (96, 128, 3), dtype=np.uint8), cv2.COLOR_RGB2GRAY).astype(np.float32)
    sizes = O.level_sizes(96, 128)
    out["pyr_sizes"] = np.array(sizes, np.int32)
    out["pyr_0"] = g
    for l, (h, w) in enumerate(sizes[1:], 1):
        out["pyr_%d" % l] = cv2.resize(out["pyr_%d" % (l - 1)], (w, h), interpolation=cv2.INTER_LINEAR)
        e = rel(O.resize(out["pyr_%d" % (l - 1)], h, w), out["pyr_%d" % l])
        assert e <= 1e-6, ("pyramid level", l, e)
    flow = (rng.standard_normal((2, 39, 52)) * 3).astype(np.float32)
    out["up_src"] = flow
    out["up_cv2"] = np.stack([cv2.resize(f, (65, 49), interpolation=cv2.INTER_LINEAR) for f in flow])
    e = rel(O.resize(flow, 49, 65), out["up_cv2"])
    assert e <= 1e-6, ("upsampling", e)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
