"""Dual TV-L1 optical flow in float64 numpy: every stage of csrc/optical_flow.cu restated, one frame pair at a time.

The solver is OpenCV's CUDA OpticalFlowDual_TVL1 (the solver DenseFlow calls, which the reference README's "Extract Frames
and Optical Flow Images" uses), with the following rules.  The kernels follow them; each function below cites the one it
restates.

  R1 grey      cv2.cvtColor(x, COLOR_RGB2GRAY) on uint8: Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15, then float in [0, 255].
  R2 sizes     level l + 1 has size (cvRound(h_l * scale_step), cvRound(w_l * scale_step)) (round half to even, as
               saturate_cast<int>(double)); the pyramid stops before the first level narrower or shorter than 16 pixels, and
               after nscales levels.
  R3 resize    bilinear, half-pixel centres: output index d of an n -> m axis samples source coordinate
               (d + 0.5) * (n / m) - 0.5; taps floor(x) and floor(x) + 1 with weights 1 - a and a (a = x - floor(x)); indices
               clamped to 0 .. n - 1 (replicated border).  cv2.resize(src, (m_w, m_h), interpolation=INTER_LINEAR) on float32
               is this rule (oracle/gen_golden_flow.py pins it).  The pyramid downscales with it; the flow is upsampled with it
               to the next finer level and multiplied by 1 / scale_step.
  R4 gradient  centred differences of I1 with replicated borders: Ix = 0.5 (I(y, min(x+1, w-1)) - I(y, max(x-1, 0))), Iy alike.
  R5 warp      at (x, y) with flow (u1, u2): wx = x + u1, wy = y + u2, clamped to [-3, w + 2] x [-3, h + 2] (beyond that
               every tap reads the border pixel, so the value does not change); taps cx = ceil(wx - 2) .. floor(wx + 2),
               cy alike, weight k(wx - cx) k(wy - cy) with Keys' bicubic kernel (a = -0.5):
               k(t) = |t|^2 (1.5 |t| - 2.5) + 1 for |t| <= 1, |t| (|t| (-0.5 |t| + 2.5) - 4) + 2 for 1 < |t| < 2, else 0;
               reads clamped to the image (replicated border); the weighted sums of I1, Ix, Iy are divided by the summed
               weight.  grad = Ixw^2 + Iyw^2, rho_c = I1w - Ixw u1 - Iyw u2 - I0.
  R6 primal    rho = rho_c + Ixw u1 + Iyw u2; l_t = lambda theta; (d1, d2) = l_t (Ixw, Iyw) if rho < -l_t grad,
               -l_t (Ixw, Iyw) if rho > l_t grad, -rho / grad (Ixw, Iyw) if grad > FLT_EPSILON, else 0;
               u_i <- u_i + d_i + theta div(p_i1, p_i2) with div(a, b) = a(y, x) - a(y, x-1) + b(y, x) - b(y-1, x), the term at
               x - 1 (y - 1) dropped in the first column (row).
  R7 dual      taut = tau / theta; ux = u(y, min(x+1, w-1)) - u(y, x), uy alike; g = hypot(ux, uy);
               p_i1 <- (p_i1 + taut ux) / (1 + taut g), p_i2 <- (p_i2 + taut uy) / (1 + taut g).  p is zero at the start of
               each level; the flow is zero at the start of the coarsest level.
  R8 stopping  each iteration is one primal and one dual update.  error = the sum over the level's pixels of the squared
               primal change of u1 and u2; a warp stops after the first iteration whose error <= epsilon^2 * w * h, and after
               `iterations` iterations.  fixed_iterations ignores the error.  Warps 0 .. warps - 1 re-linearise around the
               current flow; the levels run from the coarsest to the finest.
  R9 planes    DenseFlow's convertFlowToImage with bound b: v < -b -> 0, v > b -> 255, else cvRound(255 (v + b) / (2 b)) in
               double from the fp32 value (half to even).

Parity with a built OpenCV CUDA or DenseFlow is not checked anywhere (neither is part of this project); this module is the
reference the kernels are held to.  gamma (the illumination term) is not implemented and is refused.
"""
import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)
DEFAULTS = dict(tau=0.25, lambda_=0.15, theta=0.3, nscales=5, warps=5, epsilon=0.01, iterations=300, scale_step=0.8, gamma=0.0)


def grey(rgb):
    """R1: uint8 [..., 3] RGB -> uint8 [...]"""
    r = rgb.astype(np.int64)
    return ((r[..., 0] * 9798 + r[..., 1] * 19235 + r[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def level_sizes(h, w, nscales=5, scale_step=0.8):
    """R2: [(h_0, w_0), (h_1, w_1), ...] finest first"""
    sizes = [(h, w)]
    while len(sizes) < nscales:
        ph, pw = sizes[-1]
        nh, nw = int(np.rint(ph * scale_step)), int(np.rint(pw * scale_step))
        if nh < 16 or nw < 16:
            break
        sizes.append((nh, nw))
    return sizes


def _axis(n, m):
    x = (np.arange(m, dtype=np.float64) + 0.5) * (n / m) - 0.5
    x0 = np.floor(x)
    a = x - x0
    x0 = x0.astype(np.int64)
    return np.clip(x0, 0, n - 1), np.clip(x0 + 1, 0, n - 1), a


def resize(img, h, w):
    """R3: [..., H, W] -> [..., h, w]"""
    y0, y1, ay = _axis(img.shape[-2], h)
    x0, x1, ax = _axis(img.shape[-1], w)
    img = np.asarray(img, np.float64)
    rows = img[..., y0, :] * (1 - ay)[:, None] + img[..., y1, :] * ay[:, None]
    return rows[..., x0] * (1 - ax) + rows[..., x1] * ax


def pyramid(g, sizes):
    """R2 + R3: grey level 0 [H, W] -> list of levels, finest first, each downscaled from the previous one"""
    levels = [np.asarray(g, np.float64)]
    for h, w in sizes[1:]:
        levels.append(resize(levels[-1], h, w))
    return levels


def gradient(I):
    """R4: -> (Ix, Iy)"""
    h, w = I.shape
    xs, ys = np.arange(w), np.arange(h)
    Ix = 0.5 * (I[:, np.minimum(xs + 1, w - 1)] - I[:, np.maximum(xs - 1, 0)])
    Iy = 0.5 * (I[np.minimum(ys + 1, h - 1), :] - I[np.maximum(ys - 1, 0), :])
    return Ix, Iy


def cubic(t):
    t = np.abs(t)
    return np.where(t <= 1, t * t * (1.5 * t - 2.5) + 1, np.where(t < 2, t * (t * (-0.5 * t + 2.5) - 4) + 2, 0.0))


def warp(I0, I1, Ix, Iy, u):
    """R5: u [2, h, w] -> (Ixw, Iyw, grad, rho_c)"""
    h, w = I0.shape
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    wx = np.clip(xs + u[0], -3.0, w + 2.0)
    wy = np.clip(ys + u[1], -3.0, h + 2.0)
    x0, y0 = np.ceil(wx - 2), np.ceil(wy - 2)
    acc = np.zeros((3, h, w))
    wsum = np.zeros((h, w))
    for j in range(5):
        cy = y0 + j
        ky = np.where(cy <= np.floor(wy + 2), cubic(wy - cy), 0.0)
        ry = np.clip(cy, 0, h - 1).astype(np.int64)
        for i in range(5):
            cx = x0 + i
            k = ky * np.where(cx <= np.floor(wx + 2), cubic(wx - cx), 0.0)
            rx = np.clip(cx, 0, w - 1).astype(np.int64)
            for c, src in enumerate((I1, Ix, Iy)):
                acc[c] += k * src[ry, rx]
            wsum += k
    I1w, Ixw, Iyw = acc / wsum
    grad = Ixw * Ixw + Iyw * Iyw
    rho_c = I1w - Ixw * u[0] - Iyw * u[1] - I0
    return Ixw, Iyw, grad, rho_c


def divergence(a, b):
    d = a.copy()
    d[:, 1:] -= a[:, :-1]
    d += b
    d[1:, :] -= b[:-1, :]
    return d


def primal(Ixw, Iyw, grad, rho_c, p, u, lambda_=0.15, theta=0.3):
    """R6: p [4, h, w] (p11, p12, p21, p22), u [2, h, w] -> (new u, error)"""
    l_t = lambda_ * theta
    rho = rho_c + Ixw * u[0] + Iyw * u[1]
    lo, hi = rho < -l_t * grad, rho > l_t * grad
    mid = ~lo & ~hi & (grad > FLT_EPSILON)
    fi = np.where(lo, l_t, np.where(hi, -l_t, np.where(mid, -rho / np.where(mid, grad, 1.0), 0.0)))
    nu = np.stack([u[0] + fi * Ixw + theta * divergence(p[0], p[1]), u[1] + fi * Iyw + theta * divergence(p[2], p[3])])
    return nu, float(((nu - u) ** 2).sum())


def dual(u, p, tau=0.25, theta=0.3):
    """R7: -> new p"""
    taut = tau / theta
    h, w = u.shape[1:]
    xs, ys = np.minimum(np.arange(w) + 1, w - 1), np.minimum(np.arange(h) + 1, h - 1)
    out = np.empty_like(p)
    for i in range(2):
        ux = u[i][:, xs] - u[i]
        uy = u[i][ys, :] - u[i]
        ng = 1 + taut * np.hypot(ux, uy)
        out[2 * i] = (p[2 * i] + taut * ux) / ng
        out[2 * i + 1] = (p[2 * i + 1] + taut * uy) / ng
    return out


def tvl1(g0, g1, counts=None, fixed_iterations=False, trace=None, **params):
    """R2 .. R8 for one pair of grey frames [H, W] -> (flow [2, H, W] float64, iterations int32 [levels, warps]).
    counts [levels, warps] (level 0 the finest): run exactly that many iterations (replaying another run's stopping rule).
    trace: a dict that receives trace[(level, warp)] = [error of iteration 1, 2, ...], R8's error as computed (replayed or not)."""
    prm = dict(DEFAULTS, **params)
    if prm["gamma"] != 0:
        raise ValueError("gamma != 0 is not implemented")
    sizes = level_sizes(*np.shape(g0), prm["nscales"], prm["scale_step"])
    P0, P1 = pyramid(g0, sizes), pyramid(g1, sizes)
    L, W = len(sizes), prm["warps"]
    its = np.zeros((L, W), np.int32)
    u = np.zeros((2,) + sizes[-1])
    for lv in range(L - 1, -1, -1):
        h, w = sizes[lv]
        Ix, Iy = gradient(P1[lv])
        p = np.zeros((4, h, w))
        thr = prm["epsilon"] * prm["epsilon"] * h * w
        for wp in range(W):
            Ixw, Iyw, grad, rho_c = warp(P0[lv], P1[lv], Ix, Iy, u)
            n = 0
            errs = []
            if trace is not None:
                trace[(lv, wp)] = errs
            while True:
                u, err = primal(Ixw, Iyw, grad, rho_c, p, u, prm["lambda_"], prm["theta"])
                p = dual(u, p, prm["tau"], prm["theta"])
                errs.append(err)
                n += 1
                if counts is not None:
                    if n >= counts[lv][wp]:
                        break
                elif n >= prm["iterations"] or (not fixed_iterations and err <= thr):
                    break
            its[lv, wp] = n
        if lv > 0:
            u = resize(u, *sizes[lv - 1]) * (1.0 / prm["scale_step"])
    return u, its


def planes(flow, bound=20.0):
    """R9: flow [..., 2, H, W] (fp32 values) -> uint8 [..., 2, H, W]"""
    v = np.asarray(flow, np.float32).astype(np.float64)
    q = np.rint(255.0 * (np.nan_to_num(v) + bound) / (2.0 * bound))
    return np.where(v > bound, 255, np.where((v < -bound) | np.isnan(v), 0, q)).astype(np.uint8)


def texture(x, y, seed=0, waves=12):
    """a smooth seeded grey texture in [~28, ~228] at real coordinates (sums of plane waves of 4 .. 16 px period)"""
    rng = np.random.default_rng(seed)
    out = np.full(np.broadcast(x, y).shape, 128.0)
    for _ in range(waves):
        k = 2 * np.pi / rng.uniform(4, 16)
        a = rng.uniform(0, 2 * np.pi)
        out += (100.0 / waves) * 2 * np.sin(k * (np.cos(a) * x + np.sin(a) * y) + rng.uniform(0, 2 * np.pi))
    return out


def moving_pair(h, w, motion, seed=0):
    """-> (I0, I1 float64 [h, w], true flow [2, h, w]) with I1(x + u(x)) = I0(x): motion ('shift', dx, dy) or ('rotate', degrees),
    the rotation about the image centre"""
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    if motion[0] == "shift":
        u = np.stack([np.full((h, w), motion[1]), np.full((h, w), motion[2])])
    else:
        t = np.deg2rad(motion[1])
        cx, cy = (w - 1) / 2, (h - 1) / 2
        u = np.stack([np.cos(t) * (xs - cx) - np.sin(t) * (ys - cy) + cx - xs, np.sin(t) * (xs - cx) + np.cos(t) * (ys - cy) + cy - ys])
    I0 = texture(xs, ys, seed)
    if motion[0] == "shift":
        I1 = texture(xs - motion[1], ys - motion[2], seed)
    else:
        t = np.deg2rad(motion[1])
        cx, cy = (w - 1) / 2, (h - 1) / 2
        I1 = texture(np.cos(t) * (xs - cx) + np.sin(t) * (ys - cy) + cx, -np.sin(t) * (xs - cx) + np.cos(t) * (ys - cy) + cy, seed)
    return I0, I1, u


def epe(flow, truth, border=8):
    """mean and max end-point error over the interior (border pixels dropped on every side)"""
    d = np.hypot(*(np.asarray(flow, np.float64) - truth))[border:-border, border:-border]
    return float(d.mean()), float(d.max())
