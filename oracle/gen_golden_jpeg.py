"""Write tests/golden/jpeg.npz: seeded images encoded by Pillow, and what Image.open(f).convert('RGB' | 'L') decodes them to.

    python oracle/gen_golden_jpeg.py

Sizes 1x1 .. 37x23 store Pillow's pixels; 341x255, 340x256 and 480x360 store the SHA-256 of them.  Subsampling 4:4:4, 4:2:2,
4:2:0 and grayscale; quality 5 .. 100, optimize=True, restart_marker_blocks / restart_marker_rows; flat, saturated,
checkerboard, noise and smooth content; both modes for every stream (grayscale -> 'RGB', colour -> 'L'); and a progressive
stream, which the decoder refuses.  content() needs only numpy, so tests and benchmarks make the same images without PIL.
"""
import hashlib
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg.npz")

SMALL = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (37, 23)]          # (width, height)
LARGE = [(341, 255), (340, 256), (480, 360)]
SUBSAMPLING = {"444": 0, "422": 1, "420": 2, "gray": None}
QUALITIES = [5, 50, 75, 90, 95, 100]
CONTENTS = ["flat", "saturated", "checker", "noise", "smooth"]


def content(kind, w, h, channels, seed):
    """seeded uint8 [h, w, channels] test content"""
    rng = np.random.default_rng(seed)
    if kind == "flat":
        a = np.broadcast_to(rng.integers(0, 256, channels), (h, w, channels))
    elif kind == "saturated":
        a = np.where(rng.random((h, w, channels)) < 0.5, 0, 255)
    elif kind == "checker":
        a = np.repeat(((np.indices((h, w)).sum(0) % 2) * 255)[..., None], channels, -1)
    elif kind == "noise":
        a = rng.integers(0, 256, (h, w, channels))
    else:                       # smooth gradients with a little noise, like video frames
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        ph = rng.random(3) * 6.28
        a = np.stack([127 + 100 * np.sin(x / (17 + 5 * c) + y / (23 + 3 * c) + ph[c]) for c in range(channels)], -1)
        a = a + rng.normal(0, 6, a.shape)
    return np.ascontiguousarray(np.clip(a, 0, 255).astype(np.uint8))


def encode(arr, sub, **kw):
    from PIL import Image
    b = io.BytesIO()
    if sub == "gray":
        Image.fromarray(arr[..., 0], "L").save(b, "JPEG", **kw)
    else:
        Image.fromarray(arr, "RGB").save(b, "JPEG", subsampling=SUBSAMPLING[sub], **kw)
    return b.getvalue()


def pil_decode(data, mode):
    from PIL import Image
    im = Image.open(io.BytesIO(data)).convert(mode)
    return np.asarray(im).reshape(im.size[1], im.size[0], -1)


def specs():
    """(name, width, height, subsampling, content, seed, encoder keywords)"""
    out, seed = [], 0
    for w, h in SMALL:
        for sub in SUBSAMPLING:
            for ci, kind in enumerate(CONTENTS[:4]):
                q = QUALITIES[(seed + ci) % len(QUALITIES)]
                out.append(("%dx%d_%s_%s_q%d" % (w, h, sub, kind, q), w, h, sub, kind, seed, dict(quality=q)))
                seed += 1
    for sub in SUBSAMPLING:
        out.append(("37x23_%s_noise_opt" % sub, 37, 23, sub, "noise", seed, dict(quality=90, optimize=True)))
        out.append(("37x23_%s_smooth_rst_blocks" % sub, 37, 23, sub, "smooth", seed + 1, dict(quality=75, restart_marker_blocks=1)))
        out.append(("37x23_%s_smooth_rst_rows" % sub, 37, 23, sub, "smooth", seed + 2, dict(quality=95, restart_marker_rows=1)))
        seed += 3
    for i, (w, h) in enumerate(LARGE):
        for j, sub in enumerate(SUBSAMPLING):
            q = [50, 90, 95][(i + j) % 3]
            out.append(("%dx%d_%s_smooth_q%d" % (w, h, sub, q), w, h, sub, "smooth", seed, dict(quality=q)))
            seed += 1
    out.append(("340x256_420_smooth_q95_opt_rst", 340, 256, "420", "smooth", seed, dict(quality=95, optimize=True, restart_marker_rows=2)))
    out.append(("480x360_444_checker_q100", 480, 360, "444", "checker", seed + 1, dict(quality=100)))
    return out


def main():
    import PIL
    arrays, cases = {}, []
    for name, w, h, sub, kind, seed, kw in specs():
        data = encode(content(kind, w, h, 1 if sub == "gray" else 3, seed), sub, **kw)
        case = dict(name=name, width=w, height=h, subsampling=sub, content=kind, seed=seed, encoder=kw, bytes=len(data))
        arrays["jpg_" + name] = np.frombuffer(data, np.uint8)
        for mode in ("RGB", "L"):
            px = pil_decode(data, mode)
            if w * h <= 64 * 64:
                arrays["px_%s_%s" % (mode, name)] = px
            else:
                case["sha256_" + mode] = hashlib.sha256(px.tobytes()).hexdigest()
        cases.append(case)
    prog = encode(content("smooth", 16, 16, 3, 999), "420", quality=90, progressive=True)
    arrays["jpg_progressive"] = np.frombuffer(prog, np.uint8)
    arrays["cases"] = np.array(json.dumps(dict(pillow=PIL.__version__, cases=cases)))
    np.savez_compressed(OUT, **arrays)
    print("wrote %s: %d cases, %d bytes" % (OUT, len(cases), os.path.getsize(OUT)))


if __name__ == "__main__":
    sys.exit(main())
