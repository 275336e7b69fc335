"""TV-L1 optical flow on the H100 at its edges (csrc/optical_flow.cu, ops/optical_flow.py): the stopping rule (R8) decided by
the in-kernel reduction, bracketed exactly from the GPU's own fixed-iteration trajectory at 1 .. 1,024 tiles per level; the
stopping decisions of the full pyramid against float64 within a measured band; fixed_iterations; shapes from 1 x 1 to
8192 x 16 and constant, black, identical, checkerboard and saturating contents through the whole solver; single-frame videos
and the grid limits (32,767 pairs, 65,535 frames); and ssnb_flow_planes bitwise at every rounding edge of R9.

Small shapes are height x width throughout."""
import time

import numpy as np
import pytest
import torch

from oracle import tvl1_oracle as O

pytestmark = pytest.mark.gpu

ABS_BAR, REL_BAR = 1e-2, 1e-4          # the whole-solver bars of tests/test_gpu_optical_flow.py (replayed counts vs float64)
# R8's decisions against float64: the GPU's error sum and the oracle's differ by the fp32 drift of the trajectory, so each
# GPU decision is held to thr (1 +- DELTA).  Measured on an H100 80GB HBM3 (700 W): worst ratio 0.146, at level 1, warp 2 of
# the 48 x 64 shift by (-2.3, 0.2), whose 2-3 px strip without a match drifts by 0.15 px; 0 for the 340 x 256 translation
# and the other 48 x 64 motions.  DELTA is twice the worst.
DELTA = 3e-1


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t = time.time()
    yield
    print("\ntest_gpu_optical_flow_edges.py wall time: %.1f s" % (time.time() - t))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _rel(a, b):
    a = np.asarray(a, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _rgb(g):
    """uint8 grey [..., h, w] -> RGB with R = G = B, whose R1 grey is g exactly (9798 + 19235 + 3735 = 2^15)"""
    return np.repeat(np.asarray(g, np.uint8)[..., None], 3, -1)


def _flow(grey, offsets, **prm):
    """uint8 grey frames [F, h, w] -> (flow fp32 [P, 2, h, w], iterations [P, levels, warps]) as numpy"""
    from ops.optical_flow import tvl1_flow
    f, its = tvl1_flow(torch.from_numpy(_rgb(grey)).to(_dev()), offsets, return_iterations=True, **prm)
    return f.cpu().numpy(), its.cpu().numpy()


def _tex(h, w, dx=0.0, dy=0.0, seed=0):
    """O.texture moved by (dx, dy), rounded to uint8 grey [h, w]"""
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    return np.clip(np.rint(O.texture(xs - dx, ys - dy, seed)), 0, 255).astype(np.uint8)


def _replay(flow, its, g0, g1, **prm):
    """the oracle run for exactly the GPU's counts -> (max |du|, rel-L2, float64 flow); a zero reference flow must be met
    exactly (rel-L2 is then 0 or inf)"""
    ref, rits = O.tvl1(np.asarray(g0, np.float64), np.asarray(g1, np.float64), counts=its, **prm)
    assert (rits == its).all()
    if not ref.any():
        return float(np.abs(flow).max()), 0.0 if not flow.any() else np.inf, ref
    return float(np.abs(flow - ref).max()), _rel(flow, ref), ref


def _within_bars(a, r):
    return a <= ABS_BAR and r <= REL_BAR


def _check_planes(got, ref, bound=20.0):
    """planes of the GPU flow vs O.planes of the float64 reference: equal, or one level apart next to a rounding tie"""
    from ops.optical_flow import flow_planes
    p = flow_planes(torch.from_numpy(np.ascontiguousarray(got[None])).to(_dev()), bound).cpu().numpy()[:, :, :, 0]
    d = p.astype(int) - O.planes(ref.astype(np.float32), bound)
    if (d != 0).any():
        v = 255.0 * (ref + bound) / (2 * bound)
        assert np.abs(d).max() <= 1 and (np.abs(v[d != 0] - np.floor(v[d != 0]) - 0.5) <= 1e-3 * 255 / (2 * bound)).all()
    return p


# ---------------------------------------------------------------------------------------------------------------------------
# R8's reduction, exactly: nscales=1, warps=1, so the returned flow is u after the last primal update and the GPU's error sum
# of iteration k is E_k = sum (u_k - u_{k-1})^2 up to the fp32 rounding of each pixel's squares (<~ 3e-7 relative).  A
# threshold 1e-5 above or below an E_k that is 1e-4 away from every other E_j has one right answer per pair: the first j with
# E_j <= T.  A dropped tile partial, partials of two pairs mixed, or '<' for '<=' changes some answer.

RED_SHAPES = [(256, 340), (16, 8192), (8192, 16), (8, 32), (9, 33), (1, 40)]
RED_N = 30


def _red_pairs(h, w):
    """four pairs of different content (they stop at different k) and a constant pair (E = 0 from the first iteration):
    grey [10, h, w] as five two-frame videos"""
    g = []
    for s, (dx, dy) in enumerate([(0.4, -0.3), (1.3, 0.6), (-0.8, 1.1), (2.1, -1.7)]):
        g += [_tex(h, w, seed=10 + s), _tex(h, w, dx, dy, seed=10 + s)]
    g += [np.full((h, w), 77, np.uint8)] * 2
    return np.stack(g), np.arange(0, 11, 2)


def _first_under(E, T, n):
    """E [P, n] (iteration 1 .. n) -> per pair the first iteration with E <= T, else n"""
    hit = E <= T
    return np.where(hit.any(1), hit.argmax(1) + 1, n)


@pytest.mark.parametrize("shape", RED_SHAPES, ids=["%dx%d" % s for s in RED_SHAPES])
def test_in_kernel_reduction_brackets_exactly(shape):
    from ops.optical_flow import tvl1_flow
    dev = _dev()
    h, w = shape
    g, off = _red_pairs(h, w)
    x = torch.from_numpy(_rgb(g)).to(dev)
    one = dict(nscales=1, warps=1)
    us = [torch.zeros(len(off) - 1, 2, h, w, device=dev)]
    for k in range(1, RED_N + 1):
        f, its = tvl1_flow(x, off, return_iterations=True, fixed_iterations=True, iterations=k, **one)
        assert (its == k).all()
        us.append(f)
    E = np.stack([((us[k].double() - us[k - 1].double()) ** 2).sum((1, 2, 3)).cpu().numpy() for k in range(1, RED_N + 1)], 1)
    tiles = ((w + 31) // 32) * ((h + 7) // 8)
    assert (E[-1] == 0).all() and (E[:-1] > 0).all()
    # brackets: E[p0, k] a new low of its pair (every earlier E of p0 more than 1e-4 above) and 1e-4 away from every other E
    flat = E[:-1].ravel()
    cands = []
    for p0 in range(E.shape[0] - 1):
        for k in range(1, RED_N):
            e = E[p0, k - 1]
            if (E[p0, :k - 1] > e * (1 + 1e-4)).all() and (np.abs(flat - e) > 1e-4 * e).sum() == flat.size - 1:
                cands.append((p0, k))
    assert len(cands) >= 3, cands
    picks = [cands[i] for i in sorted({0, len(cands) // 3, 2 * len(cands) // 3, len(cands) - 1})]
    differ = False
    for p0, k in picks:
        for sgn in (1, -1):
            T = E[p0, k - 1] * (1 + sgn * 1e-5)
            want = _first_under(E, T, RED_N)
            f, its = tvl1_flow(x, off, return_iterations=True, iterations=RED_N, epsilon=float(np.sqrt(T / (h * w))), **one)
            got = its[:, 0, 0].cpu().numpy()
            print("%dx%d (%d tiles): pair %d E_%d = %.9e, T = E (1 %+.0e): GPU counts %s, want %s" % (h, w, tiles, p0, k, E[p0, k - 1], sgn * 1e-5,
                                                                                                    got.tolist(), want.tolist()))
            assert (got == want).all()
            assert want[p0] == k if sgn > 0 else want[p0] > k
            differ |= len(set(want[:-1].tolist())) > 1
            for p, c in enumerate(got):                   # a stopped pair's flow is u after its last update, untouched since
                assert torch.equal(f[p], us[c][p]), (p, c)
    assert differ                                         # some bracket stopped the textured pairs at different k
    # E = 0 and epsilon = 0: '<=' stops the constant pair after one iteration, the textured ones run out
    _, its = tvl1_flow(x, off, return_iterations=True, iterations=RED_N, epsilon=0.0, **one)
    assert its[:, 0, 0].tolist() == [RED_N] * 4 + [1]


# ---------------------------------------------------------------------------------------------------------------------------
# R8 on the full pyramid against float64

def _band(its, trace, sizes, iterations, eps=0.01):
    """-> (worst ratio by which a GPU decision departs from the rule on the float64 trajectory, warps whose decision the rule
    would have taken otherwise)"""
    worst, flipped = 0.0, 0
    for (l, wp), errs in trace.items():
        c, thr = int(its[l, wp]), eps * eps * sizes[l][0] * sizes[l][1]
        r = np.asarray(errs) / thr
        over = r[-1] - 1 if c < iterations else -np.inf     # the GPU stopped after c: error at c <= thr
        under = (1 - r[:-1]).max(initial=-np.inf)           # and ran on before: every earlier error > thr
        worst = max(worst, over, under)
        flipped += int(over > 0 or under >= 0)
    return worst, flipped


def test_stopping_decisions_against_float64_band():
    """default parameters: a translation at 340 x 256 (five levels, 352 tiles at level 0; its flow held to the whole-solver
    bars and its planes to the tie rule) and the four known motions at 48 x 64.  (A 2 degree rotation at 340 x 256 is not held here: its corners turn out of the frame, and there fp32 and float64
    part by whole pixels and their errors by 6.5% of thr.)  The oracle replays the GPU's counts with trace; every GPU decision lies within thr (1 +- DELTA)
    of the float64 errors of its level's area, and the first warp where the oracle's own run counts differently is in the band"""
    worst = 0.0
    flipped = total = same = 0
    bars = []
    for (h, w), cases in (((256, 340), [("shift", 1.3, -0.7)]),
                          ((48, 64), [("shift", 0.37, -0.61), ("shift", 1.6, 0.85), ("shift", -2.3, 0.2), ("rotate", 2.0)])):
        g = []
        for s, m in enumerate(cases):
            I0, I1, _ = O.moving_pair(h, w, m, seed=s)
            g += [np.clip(np.rint(I0), 0, 255), np.clip(np.rint(I1), 0, 255)]
        g = np.stack(g).astype(np.uint8)
        flow, its = _flow(g, np.arange(0, 2 * len(cases) + 1, 2))
        sizes = O.level_sizes(h, w)
        for k, m in enumerate(cases):
            tr = {}
            a, r, ref = _replay(flow[k], its[k], g[2 * k], g[2 * k + 1], trace=tr)
            if h == 256:
                bars.append((m, a, r))
            wr, fl = _band(its[k], tr, sizes, 300)
            worst, flipped, total = max(worst, wr), flipped + fl, total + its[k].size
            line = "%dx%d %s: max |du| %.2e px, rel-L2 %.2e, band ratio %.2e, decisions the float64 rule takes otherwise %d" % (h, w, m, a, r, wr, fl)
            if h == 256:
                _check_planes(flow[k], ref)
            else:                                           # the oracle's own run: its first differing warp is in the band
                own_tr = {}
                _, own = O.tvl1(g[2 * k].astype(np.float64), g[2 * k + 1].astype(np.float64), trace=own_tr)
                same += int((own == its[k]).sum())
                order = [(l, wp) for l in range(len(sizes) - 1, -1, -1) for wp in range(5)]
                first = next((lw for lw in order if own[lw] != its[k][lw]), None)
                if first is not None:
                    c = min(own[first], its[k][first])
                    thr = 1e-4 * sizes[first[0]][0] * sizes[first[0]][1]
                    assert abs(tr[first][c - 1] / thr - 1) <= DELTA, (m, first)
                line += ", counts equal to the oracle's own run in %d of %d warps (first difference %s)" % (int((own == its[k]).sum()), own.size, first)
            print(line)
    print("stopping band: worst ratio %.2e, DELTA %.0e; %d of %d warps decided inside the band on the other side of thr; "
          "48x64 counts equal to the oracle's own run in %d of 100 warps" % (worst, DELTA, flipped, total, same))
    assert worst <= DELTA
    assert all(_within_bars(a, r) for _, a, r in bars), bars


# ---------------------------------------------------------------------------------------------------------------------------
# fixed_iterations

def _two_videos():
    """tests/test_gpu_optical_flow.py's whole-solver set: videos of 4 and 3 textured RGB frames at 40 x 56, as grey"""
    vids = []
    for (mx, my), n, seed in (((0.6, -0.35), 4, 5), ((-1.2, 0.5), 3, 9)):
        vids += [_tex(40, 56, k * mx, k * my, seed) for k in range(n)]
    return np.stack(vids), [0, 4, 7]


def test_fixed_iterations_on_the_gpu():
    g, off = _two_videos()
    pairs = [(0, 1), (1, 2), (2, 3), (4, 5), (5, 6)]
    flow, its = _flow(g, off, fixed_iterations=True, iterations=100)
    assert (its == 100).all()
    worst = [0.0, 0.0]
    for k, (i, j) in enumerate(pairs):
        ref, _ = O.tvl1(g[i].astype(np.float64), g[j].astype(np.float64), fixed_iterations=True, iterations=100)
        worst = [max(worst[0], float(np.abs(flow[k] - ref).max())), max(worst[1], _rel(flow[k], ref))]
    print("fixed 100 iterations vs float64: max |du| %.2e px, rel-L2 %.2e" % tuple(worst))
    assert worst[0] <= ABS_BAR and worst[1] <= REL_BAR
    fa, ia = _flow(g, off, fixed_iterations=True, iterations=40)
    fb, ib = _flow(g, off, epsilon=0.0, iterations=40)     # no textured warp reaches an error of exactly 0
    assert np.array_equal(fa, fb) and np.array_equal(ia, ib)
    c = np.stack([np.full((24, 32), v, np.uint8) for v in (90, 90, 140, 0)])   # equal constants, a brightness change, a fade
    for prm, n in ((dict(), 1), (dict(epsilon=0.0), 1), (dict(fixed_iterations=True, iterations=20), 20)):
        f, i = _flow(c, [0, 4], **prm)
        assert (i == n).all() and not f.any(), prm


# ---------------------------------------------------------------------------------------------------------------------------
# edge shapes and contents through the whole solver

def _checker(h, w, shift=0):
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return (((xs - shift + ys) & 1) * 255).astype(np.uint8)


CONTENTS = {
    "equal constants": lambda h, w: (np.full((h, w), 100, np.uint8), np.full((h, w), 100, np.uint8)),
    "brightness change": lambda h, w: (np.full((h, w), 60, np.uint8), np.full((h, w), 190, np.uint8)),
    "black to texture": lambda h, w: (np.zeros((h, w), np.uint8), _tex(h, w, seed=7)),
    "identical frames": lambda h, w: (_tex(h, w, seed=8), _tex(h, w, seed=8)),
    "checkerboard by 1 px": lambda h, w: (_checker(h, w), _checker(h, w, 1)),
    "shift 24 px": lambda h, w: (_tex(h, w, seed=9), _tex(h, w, 24.0, -3.0, seed=9)),
}
EDGE_SHAPES = [(1, 1), (1, 40), (40, 1), (15, 15), (16, 16), (19, 19), (20, 20), (16, 8192), (8192, 16)]


@pytest.mark.parametrize("shape", EDGE_SHAPES, ids=["%dx%d" % s for s in EDGE_SHAPES])
def test_edge_shapes_and_contents_replayed(shape):
    h, w = shape
    prm = dict(iterations=30, warps=2)
    g = np.stack([f for c in CONTENTS.values() for f in c(h, w)])
    flow, its = _flow(g, np.arange(0, 2 * len(CONTENTS) + 1, 2), **prm)
    assert ((its >= 1) & (its <= 30)).all()
    bad = []
    for k, name in enumerate(CONTENTS):
        a, r, ref = _replay(flow[k], its[k], g[2 * k], g[2 * k + 1], **prm)
        print("%dx%d %s (%d levels, %d iterations): max |du| %.2e px, rel-L2 %.2e" % (h, w, name, its.shape[1], its[k].sum(), a, r))
        if not _within_bars(a, r):
            bad.append((name, a, r))
            continue
        _check_planes(flow[k], ref)
        if name in ("equal constants", "brightness change", "identical frames"):
            assert not flow[k].any() and (its[k] == 1).all(), name    # no gradient or no change: exactly 0 after one iteration
    assert not bad, bad


def _smooth(x, y, seed):
    """a grey texture of 48 .. 128 px periods: still textured at 1/16 scale"""
    rng = np.random.default_rng(seed)
    out = np.full(np.broadcast(x, y).shape, 128.0)
    for _ in range(8):
        k, a = 2 * np.pi / rng.uniform(48, 128), rng.uniform(0, 2 * np.pi)
        out += 25.0 * np.sin(k * (np.cos(a) * x + np.sin(a) * y) + rng.uniform(0, 2 * np.pi))
    return out


def test_translation_above_the_bound_saturates_the_planes():
    """a 24 px translation at 340 x 256, found through a five-level pyramid at scale_step 0.5: the x planes saturate at 255
    over the interior, and flow and planes match the replayed float64 run"""
    h, w = 256, 340
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    g = np.stack([np.clip(np.rint(_smooth(xs - dx, ys - dy, 3)), 0, 255) for dx, dy in ((0, 0), (24, -3))]).astype(np.uint8)
    prm = dict(scale_step=0.5, iterations=50)
    flow, its = _flow(g, [0, 2], **prm)
    _, r, ref = _replay(flow[0], its[0], g[0], g[1], **prm)
    # max |du| where the displaced pixel stays in the frame (8 px beyond): the 24 columns that leave it have no match in the
    # second frame, and their flow is not determined closely enough for fp32 and float64 to agree to 1e-2 px
    a = float(np.abs(flow[0] - ref)[:, 11:-8, 8:w - 32].max())
    a_all = float(np.abs(flow[0] - ref).max())
    from ops.optical_flow import flow_planes
    p = flow_planes(torch.from_numpy(flow).to(_dev())).cpu().numpy()[:, :, :, 0]
    sat = float((p[0, 16:-16, 16:-16] == 255).mean())
    print("24 px translation: median flow (%.2f, %.2f) px, x planes at 255 over %.1f%% of the interior; max |du| %.2e px "
          "where matched (%.2e px over all), rel-L2 %.2e" % (np.median(flow[0, 0]), np.median(flow[0, 1]), 100 * sat, a, a_all, r))
    assert sat >= 0.9
    assert a <= 2 * ABS_BAR and r <= REL_BAR
    want = O.planes(ref.astype(np.float32))
    far = np.abs(ref) > 20 + 2 * ABS_BAR                    # beyond the bound by more than the flow error: saturated on both
    assert far[0, 16:-16, 16:-16].mean() >= 0.9 and (p[far] == want[far]).all()


STAGE_SHAPES = [(1, 1), (1, 33), (33, 1), (8, 8192)]


@pytest.mark.parametrize("shape", STAGE_SHAPES, ids=["%dx%d" % s for s in STAGE_SHAPES])
def test_stages_at_edge_shapes_against_float64(shape):
    from ssn_b200._lib import lib, check, ptr_array, TVL1_GREY, TVL1_RESIZE, TVL1_GRADIENT, TVL1_WARP, TVL1_PRIMAL, TVL1_DUAL
    from ops.optical_flow import tvl1_params, _stream
    dev = _dev()
    h, w = shape
    n = 2
    rng = np.random.default_rng(h * 10007 + w)

    def stage(s, ins, outs, oh=0, ow=0, mul=1.0):
        check(lib.ssnb_tvl1_stage(s, tvl1_params(), n, h, w, oh, ow, mul, ptr_array(ins), ptr_array(outs), _stream()), None, "tvl1_stage")
        torch.cuda.synchronize()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    E = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    rgb = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    gr = E(n, h, w)
    stage(TVL1_GREY, [T(rgb)], [gr])
    assert (gr.cpu().numpy() == O.grey(rgb).astype(np.float32)).all()
    I0 = np.stack([_tex(h, w, seed=s) for s in range(n)]).astype(np.float32)
    I1 = np.stack([_tex(h, w, 0.3, -0.7, seed=s) for s in range(n)]).astype(np.float32)
    errs = {}
    for oh, ow, mul in ((max(1, round(h * 0.8)), max(1, round(w * 0.8)), 1.0), (min(2 * h + 1, 8192), min(2 * w + 1, 8192), 1.25)):
        out = E(n, oh, ow)
        stage(TVL1_RESIZE, [T(I1)], [out], oh, ow, mul)
        errs["resize"] = max(errs.get("resize", 0.0), _rel(out.cpu(), O.resize(I1.astype(np.float64), oh, ow) * mul))
    u = (rng.standard_normal((n, 2, h, w)) * 2).astype(np.float32)
    u.reshape(-1)[:4] = [-40, 70, 1, -1]
    p = (rng.standard_normal((n, 4, h, w)) * 0.3).astype(np.float32)
    ix, iy = E(n, h, w), E(n, h, w)
    stage(TVL1_GRADIENT, [T(I1)], [ix, iy])
    ref = np.stack([np.stack(O.gradient(x)) for x in I1.astype(np.float64)], 1)
    errs["gradient"] = max(_rel(a.cpu(), b) for a, b in zip((ix, iy), ref))
    if h * w == 1:
        assert not ix.cpu().numpy().any() and not iy.cpu().numpy().any()
    Ix, Iy = ix.cpu().numpy().astype(np.float64), iy.cpu().numpy().astype(np.float64)
    outs = [E(n, h, w) for _ in range(4)]
    stage(TVL1_WARP, [T(I0), T(I1), ix, iy, T(u)], outs)
    ref = np.stack([np.stack(O.warp(I0[i].astype(np.float64), I1[i].astype(np.float64), Ix[i], Iy[i], u[i].astype(np.float64))) for i in range(n)], 1)
    errs["warp"] = max(_rel(o.cpu(), r) for o, r in zip(outs, ref))
    wx, wy, g2, rc = [o.cpu().numpy().astype(np.float64) for o in outs]
    un = E(n, 2, h, w)
    stage(TVL1_PRIMAL, outs + [T(p), T(u)], [un])
    ref = np.stack([O.primal(wx[i], wy[i], g2[i], rc[i], p[i].astype(np.float64), u[i].astype(np.float64))[0] for i in range(n)])
    errs["primal"] = _rel(un.cpu(), ref)
    pn = E(n, 4, h, w)
    stage(TVL1_DUAL, [un, T(p)], [pn])
    unh = un.cpu().numpy().astype(np.float64)
    errs["dual"] = _rel(pn.cpu(), np.stack([O.dual(unh[i], p[i].astype(np.float64)) for i in range(n)]))
    print("%dx%d stage rel-L2 vs float64:" % shape, {k: "%.2e" % v for k, v in errs.items()})
    assert max(errs.values()) <= 1e-6, errs


# ---------------------------------------------------------------------------------------------------------------------------
# single-frame videos and the grid limits

def test_single_frame_videos_in_a_ragged_call():
    """videos of one frame at the start, in the middle, back to back and at the end: every other video's pairs are bitwise
    those of the video alone, and the listed pairs match float64"""
    from ops.optical_flow import pair_offsets
    counts = [1, 4, 1, 1, 3, 2, 1, 5, 1]
    g = []
    for v, n in enumerate(counts):
        g += [_tex(24, 32, 0.7 * k, -0.4 * k, seed=30 + v) for k in range(n)]
    g = np.stack(g)
    off = np.concatenate([[0], np.cumsum(counts)])
    prm = dict(iterations=40, nscales=2)
    flow, its = _flow(g, off, **prm)
    pr = pair_offsets(off)
    assert flow.shape[0] == pr[-1] == 10
    for v in range(len(counts)):
        if counts[v] > 1:
            f1, i1 = _flow(g[off[v]:off[v + 1]], [0, counts[v]], **prm)
            assert np.array_equal(f1, flow[pr[v]:pr[v + 1]]) and np.array_equal(i1, its[pr[v]:pr[v + 1]]), v
    res = []
    # the first pair, after two single-frame videos, the 2-frame video, after the single-frame video before it, the last pair
    for k, fr in ((0, 1), (2, 3), (3, 7), (5, 10), (6, 13), (9, 16)):
        res.append(_replay(flow[k], its[k], g[fr], g[fr + 1], **prm)[:2])
    print("single-frame videos: listed pairs vs float64 (max |du| px, rel-L2):", ["%.2e %.2e" % ar for ar in res])
    assert all(_within_bars(*ar) for ar in res), res


def test_grid_limits_of_one_call():
    """20 x 20 (two levels), exactly 32,767 pairs and 65,535 frames in 32,768 videos of 1 .. 6 frames: grid.z of the pyramid
    resize is 65,535 and of the flow upsampling 65,534.  Every pair bitwise equals the same pair computed in calls of 512
    videos; 50 pairs (the first, the last, and around single-frame videos) match float64"""
    from ops.optical_flow import pair_offsets
    rng = np.random.default_rng(40)
    V, F = 32768, 65535
    n = rng.integers(1, 4, V)
    while n.sum() != F:                                      # move frames between videos until the total is exact
        i = rng.integers(V)
        if n.sum() > F and n[i] > 1:
            n[i] -= 1
        elif n.sum() < F and n[i] < 6:
            n[i] += 1
    off = np.concatenate([[0], np.cumsum(n)])
    big = np.clip(np.rint(O.texture(*np.meshgrid(np.arange(128.0), np.arange(128.0)), seed=41)), 0, 255).astype(np.uint8)
    base = np.repeat(rng.integers(8, 100, (V, 2)), n, 0)
    step = np.repeat(rng.integers(-1, 2, (V, 2)), n, 0)
    k = np.arange(F) - np.repeat(off[:-1], n)
    oy, ox = base[:, 0] + k * step[:, 0], base[:, 1] + k * step[:, 1]
    g = big[oy[:, None, None] + np.arange(20)[None, :, None], ox[:, None, None] + np.arange(20)[None, None, :]]
    prm = dict(nscales=2, warps=1, iterations=2)
    flow, its = _flow(g, off, **prm)
    P = F - V
    assert flow.shape == (P, 2, 20, 20) == (32767, 2, 20, 20) and its.shape == (P, 2, 1)
    pr = pair_offsets(off)
    for v0 in range(0, V, 512):
        v1 = min(V, v0 + 512)
        if pr[v1] == pr[v0]:
            continue
        f, i = _flow(g[off[v0]:off[v1]], off[v0:v1 + 1] - off[v0], **prm)
        assert np.array_equal(f, flow[pr[v0]:pr[v1]]) and np.array_equal(i, its[pr[v0]:pr[v1]]), v0
    single = np.flatnonzero(n == 1)
    around = [int(pr[v]) for v in single[1:] if v + 1 < V and n[v + 1] > 1][:24]            # first pair after a single-frame video
    around += [int(pr[v]) - 1 for v in single[1:] if n[v - 1] > 1][:24]                    # last pair before one
    sample = sorted({0, P - 1} | set(around))
    frame = np.arange(F)[np.concatenate([np.arange(off[v], off[v + 1] - 1) for v in range(V) if n[v] > 1])]
    worst = [0.0, 0.0]
    for q in sample:
        a, r, _ = _replay(flow[q], its[q], g[frame[q]], g[frame[q] + 1], **prm)
        worst = [max(worst[0], a), max(worst[1], r)]
    print("grid limits: %d pairs, %d frames, %d videos (%d of one frame); %d pairs vs float64: max |du| %.2e px, rel-L2 %.2e"
          % (P, F, V, len(single), len(sample), *worst))
    assert len(sample) >= 45 and _within_bars(*worst)


# ---------------------------------------------------------------------------------------------------------------------------
# R9 on the device, bitwise

def _edge_values(bound):
    """every fp32 within +-64 ULPs of R9's 255 rounding boundaries and of +-bound, +-0, subnormals, +-FLT_MAX, +-inf and NaNs of
    both signs with assorted payloads"""
    c = np.float32(((np.arange(255) + 0.5) * (2 * bound) / 255 - bound).tolist() + [bound, -bound])
    vals, up, dn = [c], c.copy(), c.copy()
    for _ in range(64):
        up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        vals += [up, dn]
    bits = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007fffff, 0x807fffff, 0x00400000, 0x80012345,
                     0x7f7fffff, 0xff7fffff, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fbfffff,
                     0xffbfffff, 0x7fffffff, 0xffffffff, 0x7fd2a5a5, 0xff912345], np.uint32)
    return np.concatenate(vals + [bits.view(np.float32)])


def test_flow_planes_bitwise_at_every_rounding_edge():
    from ops.optical_flow import flow_planes
    dev = _dev()
    rng = np.random.default_rng(50)
    rand = rng.integers(0, 1 << 32, 1 << 24, dtype=np.uint64).astype(np.uint32).view(np.float32)
    sweep = np.linspace(-21.0, 21.0, (1 << 22) + 1).astype(np.float32)
    cap = 148 * 32 * 256
    for bound in (20.0, 15.0, 1.0, 1e-3):
        edge = _edge_values(bound)
        for vals, (h, w) in ((edge, (7, 13)), (np.concatenate([edge, rand, sweep]), (37, 53))):
            P = -(-vals.size // (2 * h * w))
            flow = np.zeros(P * 2 * h * w, np.float32)
            flow[:vals.size] = vals
            flow = flow.reshape(P, 2, h, w)
            got = flow_planes(torch.from_numpy(flow).to(dev), bound).cpu().numpy().reshape(P, 2, h, w)
            with np.errstate(over="ignore", invalid="ignore"):
                want = O.planes(flow, bound)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (bound, flow.ravel()[bad[:5]], got.ravel()[bad[:5]], want.ravel()[bad[:5]])
            print("flow_planes bound %g: %d values in [%d, 2, %d, %d] (%s the %d-element grid cap) bitwise equal to O.planes"
                  % (bound, vals.size, P, h, w, "above" if flow.size > cap else "below", cap))
