"""TV-L1 optical flow on the H100 (csrc/optical_flow.cu, ops/optical_flow.py) against the float64 oracle
(oracle/tvl1_oracle.py): each stage on the operands the kernel consumed, the whole solver replaying the GPU's iteration
counts, known motions with the stopping rule, batching, repeatability, graph capture, and the planes through Flow scoring."""
import os

import numpy as np
import pytest
import torch

from oracle import tvl1_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "optical_flow.npz"))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _rel(a, b):
    a = np.asarray(a, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _stage(stage, n, h, w, ins, outs, oh=0, ow=0, mul=1.0):
    from ssn_b200._lib import lib, check, ptr_array
    from ops.optical_flow import tvl1_params, _stream
    check(lib.ssnb_tvl1_stage(stage, tvl1_params(), n, h, w, oh, ow, mul, ptr_array(ins), ptr_array(outs), _stream()), None, "tvl1_stage")
    torch.cuda.synchronize()


def _rgb_video(motion, n, h, w, seed):
    """n RGB frames of a texture moving by `motion` per frame (uint8 [n, h, w, 3]) and the per-pair true flow [2, h, w]"""
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    frames = []
    for k in range(n):
        ch = [O.texture(xs - k * motion[0], ys - k * motion[1], seed + c) for c in range(3)]
        frames.append(np.clip(np.rint(np.stack(ch, -1)), 0, 255).astype(np.uint8))
    return np.stack(frames), np.stack([np.full((h, w), motion[0]), np.full((h, w), motion[1])])


def test_grey_bitwise_against_opencv_golden():
    from ssn_b200._lib import TVL1_GREY
    dev = _dev()
    rgb = torch.from_numpy(GOLD["grey_rgb"]).to(dev)[None]
    out = torch.empty(1, 64, 64, dtype=torch.float32, device=dev)
    _stage(TVL1_GREY, 1, 64, 64, [rgb], [out])
    assert (out[0].cpu().numpy() == GOLD["grey_cv2"].astype(np.float32)).all()
    a = np.arange(1 << 24, dtype=np.uint32)              # every colour
    every = np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(1, 4096, 4096, 3)
    out = torch.empty(1, 4096, 4096, dtype=torch.float32, device=dev)
    _stage(TVL1_GREY, 1, 4096, 4096, [torch.from_numpy(every).to(dev)], [out])
    assert (out[0].cpu().numpy() == O.grey(every[0]).astype(np.float32)).all()


def test_pyramid_and_upsampling_stages_against_oracle_and_golden():
    from ssn_b200._lib import TVL1_RESIZE
    dev = _dev()
    sizes = [tuple(s) for s in GOLD["pyr_sizes"]]
    worst = 0.0
    for l in range(1, len(sizes)):
        src = torch.from_numpy(GOLD["pyr_%d" % (l - 1)]).to(dev)[None]
        out = torch.empty(1, *sizes[l], dtype=torch.float32, device=dev)
        _stage(TVL1_RESIZE, 1, *sizes[l - 1], [src], [out], *sizes[l])
        worst = max(worst, _rel(out[0].cpu(), O.resize(GOLD["pyr_%d" % (l - 1)], *sizes[l])))
        assert _rel(out[0].cpu(), GOLD["pyr_%d" % l]) <= 2e-6
    src = torch.from_numpy(GOLD["up_src"]).to(dev)
    out = torch.empty(2, 49, 65, dtype=torch.float32, device=dev)
    _stage(TVL1_RESIZE, 2, 39, 52, [src], [out], 49, 65, 1.25)
    worst = max(worst, _rel(out.cpu(), O.resize(GOLD["up_src"], 49, 65) * 1.25))
    print("resize rel-L2 vs float64: %.2e" % worst)
    assert worst <= 1e-6


def test_gradient_warp_primal_dual_stages_against_float64():
    from ssn_b200._lib import TVL1_GRADIENT, TVL1_WARP, TVL1_PRIMAL, TVL1_DUAL
    dev = _dev()
    rng = np.random.default_rng(3)
    n, h, w = 3, 37, 53
    I0 = np.stack([O.texture(*np.meshgrid(np.arange(w), np.arange(h)), seed=s) for s in range(n)]).astype(np.float32)
    I1 = np.stack([O.texture(*np.meshgrid(np.arange(w) + 0.3, np.arange(h) - 0.7), seed=s) for s in range(n)]).astype(np.float32)
    u = (rng.standard_normal((n, 2, h, w)) * 2).astype(np.float32)
    u[0, 0, 0, :5] = [-40, 70, 0, 1, -1]                       # far outside, and integer displacements (5 taps)
    p = (rng.standard_normal((n, 4, h, w)) * 0.3).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    E = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    ix, iy = E(n, h, w), E(n, h, w)
    _stage(TVL1_GRADIENT, n, h, w, [T(I1)], [ix, iy])
    errs = {"gradient": max(_rel(g.cpu(), r) for g, r in zip((ix, iy), np.stack([np.stack(O.gradient(x)) for x in I1.astype(np.float64)], 1)))}
    Ix, Iy = ix.cpu().numpy(), iy.cpu().numpy()
    outs = [E(n, h, w) for _ in range(4)]
    _stage(TVL1_WARP, n, h, w, [T(I0), T(I1), ix, iy, T(u)], outs)
    ref = np.stack([np.stack(O.warp(I0[i].astype(np.float64), I1[i].astype(np.float64), Ix[i].astype(np.float64), Iy[i].astype(np.float64),
                                    u[i].astype(np.float64))) for i in range(n)], 1)
    errs["warp"] = max(_rel(o.cpu(), r) for o, r in zip(outs, ref))
    wx, wy, gr, rc = [o.cpu().numpy().astype(np.float64) for o in outs]
    un = E(n, 2, h, w)
    _stage(TVL1_PRIMAL, n, h, w, outs + [T(p), T(u)], [un])
    ref = np.stack([O.primal(wx[i], wy[i], gr[i], rc[i], p[i].astype(np.float64), u[i].astype(np.float64))[0] for i in range(n)])
    errs["primal"] = _rel(un.cpu(), ref)
    pn = E(n, 4, h, w)
    _stage(TVL1_DUAL, n, h, w, [un, T(p)], [pn])
    unh = un.cpu().numpy().astype(np.float64)
    errs["dual"] = _rel(pn.cpu(), np.stack([O.dual(unh[i], p[i].astype(np.float64)) for i in range(n)]))
    print("stage rel-L2 vs float64:", {k: "%.2e" % v for k, v in errs.items()})
    assert max(errs.values()) <= 1e-6, errs


def _grey_np(frames):
    return O.grey(frames).astype(np.float64)


def test_whole_solver_replayed_against_oracle():
    """two videos of 4 and 3 frames at 40 x 56 (five pyramid levels), default parameters: the oracle run for exactly the
    GPU's iteration counts gives the GPU's flow within 1e-2 px and 1e-4 relative L2; the planes differ by one level at most,
    only next to a rounding tie"""
    from ops.optical_flow import tvl1_flow, flow_planes
    dev = _dev()
    a, _ = _rgb_video((0.6, -0.35), 4, 40, 56, seed=5)
    b, _ = _rgb_video((-1.2, 0.5), 3, 40, 56, seed=9)
    frames = np.concatenate([a, b])
    off = [0, 4, 7]
    flow, its = tvl1_flow(torch.from_numpy(frames).to(dev), off, return_iterations=True)
    flow, its = flow.cpu().numpy(), its.cpu().numpy()
    planes = flow_planes(torch.from_numpy(flow).to(dev)).cpu().numpy()
    g = _grey_np(frames)
    pairs = [(0, 1), (1, 2), (2, 3), (4, 5), (5, 6)]
    worst_abs = worst_rel = 0.0
    for k, (i, j) in enumerate(pairs):
        ref, rits = O.tvl1(g[i], g[j], counts=its[k])
        assert (rits == its[k]).all()
        worst_abs = max(worst_abs, float(np.abs(flow[k] - ref).max()))
        worst_rel = max(worst_rel, _rel(flow[k], ref))
        want = O.planes(ref.astype(np.float32))
        got = planes[2 * k:2 * k + 2, :, :, 0]
        d = got.astype(int) - want
        if (d != 0).any():
            v = 255.0 * (ref + 20.0) / 40.0
            assert np.abs(d).max() <= 1 and (np.abs(v[d != 0] - np.floor(v[d != 0]) - 0.5) <= 1e-3 * 255 / 40).all()
    print("replayed solver vs float64: max |du| %.2e px, rel-L2 %.2e, iterations per pair %s" % (worst_abs, worst_rel, its.sum((1, 2)).tolist()))
    assert worst_abs <= 1e-2 and worst_rel <= 1e-4


def test_known_motions_with_the_stopping_rule():
    """seeded sub-pixel translations and a 2 degree rotation of a texture: interior end-point error (8 px border) of the GPU
    flow, and how often its iteration counts equal the oracle's own stopping rule"""
    from ops.optical_flow import tvl1_flow
    dev = _dev()
    cases = [("shift", 0.37, -0.61), ("shift", 1.6, 0.85), ("shift", -2.3, 0.2), ("rotate", 2.0)]
    frames, truth = [], []
    for s, m in enumerate(cases):
        I0, I1, u = O.moving_pair(48, 64, m, seed=s)
        for I in (I0, I1):
            frames.append(np.repeat(np.clip(np.rint(I), 0, 255).astype(np.uint8)[..., None], 3, -1))
        truth.append(u)
    flow, its = tvl1_flow(torch.from_numpy(np.stack(frames)).to(dev), [0, 2, 4, 6, 8], return_iterations=True)
    flow, its = flow.cpu().numpy(), its.cpu().numpy()
    same = total = 0
    for k, m in enumerate(cases):
        mean, mx = O.epe(flow[k], truth[k])
        _, rits = O.tvl1(O.grey(frames[2 * k]).astype(np.float64), O.grey(frames[2 * k + 1]).astype(np.float64))
        same += int((rits == its[k]).sum())
        total += rits.size
        print("%s: interior EPE mean %.4f max %.4f px, iterations %d (oracle %d)" % (m, mean, mx, its[k].sum(), rits.sum()))
        assert mean <= 0.05 and mx <= 0.25, m
        assert its[k].max() < 300                              # the stopping rule stopped every warp
    print("iteration counts equal to the oracle's stopping rule: %d of %d warps" % (same, total))


def _ragged_frames(seed, counts, h, w):
    rng = np.random.default_rng(seed)
    vids = []
    for i, n in enumerate(counts):
        mo = rng.uniform(-1.5, 1.5, 2)
        vids.append(_rgb_video(mo, n, h, w, seed=100 + i)[0])
    return np.concatenate(vids), np.concatenate([[0], np.cumsum(counts)])


def test_ragged_batch_pairs_equal_alone_and_repeat_bitwise():
    """200 pairs of ragged videos (1 to 15 pairs each) in one call: every video's pairs are bitwise those of the video computed alone, and a
    repeat of the call is bitwise equal (stopping rule on, so pairs stop at different iterations)"""
    from ops.optical_flow import tvl1_flow
    dev = _dev()
    rng = np.random.default_rng(11)
    counts, left = [], 200
    while left:
        counts.append(min(int(rng.integers(2, 17)), left + 1))
        left -= counts[-1] - 1
    frames, off = _ragged_frames(12, counts, 24, 32)
    P = int(off[-1]) - len(counts)
    x = torch.from_numpy(frames).to(dev)
    prm = dict(iterations=40, nscales=2)
    flow, its = tvl1_flow(x, off, return_iterations=True, **prm)
    flow2, its2 = tvl1_flow(x, off, return_iterations=True, **prm)
    assert torch.equal(flow, flow2) and torch.equal(its, its2)
    assert len(set(its[:, 0, 0].tolist())) > 1
    pr = off - np.arange(len(off))
    for v in range(len(counts)):
        f1, i1 = tvl1_flow(x[off[v]:off[v + 1]], return_iterations=True, **prm)
        assert torch.equal(f1, flow[pr[v]:pr[v + 1]]) and torch.equal(i1, its[pr[v]:pr[v + 1]]), v
    print("ragged batch: %d pairs in %d videos, iterations %d .. %d" % (P, len(counts), int(its.sum((1, 2)).min()), int(its.sum((1, 2)).max())))


def test_poisoned_workspace_and_graph_replay():
    from ops.optical_flow import TVL1Plan
    dev = _dev()
    a, off = _ragged_frames(20, [5, 3, 6], 32, 40)
    b, _ = _ragged_frames(21, [5, 3, 6], 32, 40)
    plan = TVL1Plan(off, 32, 40, dev, iterations=50)
    src = torch.from_numpy(a).to(dev)
    plan.run(src)
    ref_a, its_a = plan.flow.clone(), plan.iterations.clone()
    plan.workspace.fill_(0xFF)
    plan.flow.fill_(float("nan"))
    plan.iterations.fill_(-1)
    plan.run(src)
    assert torch.equal(plan.flow, ref_a) and torch.equal(plan.iterations, its_a)
    plan.run(torch.from_numpy(b).to(dev))
    ref_b, its_b = plan.flow.clone(), plan.iterations.clone()
    static = src.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run(static)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run(static)
    static.copy_(torch.from_numpy(b).to(dev))
    plan.workspace.fill_(0xFF)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(plan.flow, ref_b) and torch.equal(plan.iterations, its_b)
    static.copy_(src)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(plan.flow, ref_a) and torch.equal(plan.iterations, its_a)


def test_planes_of_one_video_through_flow_scoring():
    """6 RGB frames -> 5 pairs (Flow's new_length) -> 10 planes x, y, ... -> oversample -> test_scores: one tick of scores, equal
    to the same planes given as decoded 'L' frames"""
    import ssn_models
    from oracle import synth
    from ssn_b200 import _lib
    from ops.optical_flow import tvl1_flow, flow_planes
    dev = _dev()
    frames, _ = _rgb_video((0.8, -0.4), 6, 256, 340, seed=2)
    planes = flow_planes(tvl1_flow(torch.from_numpy(frames).to(dev)))
    assert planes.shape == (10, 256, 340, 1) and planes.dtype == torch.uint8
    K = 4
    m = ssn_models.SSN(K, 2, 5, 2, "Flow", base_model="BNInception", dropout=0, test_mode=True)
    sd = m.state_dict()
    for k, v in synth.synth_backbone(10, seed=0, calib_frames=2).items():
        sd["base_model." + k].copy_(v)
    for k, v in synth.synth_heads(K, 5, seed=0, std=0.02, bias_std=0.1).items():
        if k in sd:
            sd[k].copy_(v)
    m = m.to(dev).eval()
    m.set_precision(_lib.EXACT_TC, 1024.0)
    m.prepare_test_fc()
    tf = m.frame_transforms()
    x = tf.oversample(planes)
    assert x.shape == (10, 10, 224, 224)
    sc = m.test_scores(x, 10)
    assert sc.shape[0] == 1 and torch.isfinite(sc).all()
    assert torch.equal(tf.oversample(planes.cpu()), x)
