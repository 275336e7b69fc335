"""Plain restatement of how the wgmma kernels split the backbone's work.  TEST INFRASTRUCTURE ONLY.

The tensor-core schedule (FAST and EXACT_TC) runs every convolution on two kernels whose work split depends on the frame
count F and on the GPU's SM count:

  umma_conv_kernel (csrc/umma_conv.cu: bind_common, umma_conv_launch), forward, data gradient and the fused sibling 1x1
    launches: a pick_box pixel box bw x bh x bf, tiles_w * tiles_h * tiles_f pixel tiles times n_tiles N tiles of block_n
    columns; grid = min(total, SMs), so CTA b runs my_tiles = ceil((total - b) / grid) tiles, handed alternately to two
    consumer warpgroups; the operand ring holds `stages` (tap, K chunk) stages, a tile takes ksteps = taps * kchunks;
  umma_wgrad_kernel (csrc/umma_wgrad.cu: umma_wgrad_bind_taps, umma_wgrad_splits), weight gradients: a 64-pixel box chosen
    by the layer width, ctas = m_tiles * n_tiles * tap_groups, splits = SMs / ctas (whole waves more where a split would sum
    more than MAX_PTILES pixel tiles) clamped to the planner's tsplits (engine.cu: plan) and to the pixel tile count,
    ptiles_per_split pixel tiles per split and a shorter last split.

`schedule(in_channels, frames, precision, sms)` lists the launches of one ssnb_backbone_fwd (+ ssnb_backbone_bwd for a
training engine) in launch order, each with the numbers above, and `log_key` reduces a launch to what
ssnb_timing_launches reports for it.  `CONV_REGIMES` / `WGRAD_REGIMES` name the regimes of the two kernels as predicates
on one launch's plan; `regimes(launch)` is the set a launch is in.

Every gated EXACT_TC plan passes UmmaConvParams::tc_ok in this network (engine.cu: ssnb_set_workspace), so the list is the
same for FAST and EXACT_TC except for `stages` (EXACT_TC stages hold both operand planes).  bn_mode='partial' runs the same
launches (conv1 raw changes its epilogue, not its tiles).  CPU only; nothing here touches a device.
"""
import functools

from . import schedule_check as S

SMS_H100_SXM = 132
SMS_H100_PCIE = 114

# The frame counts tests/test_gpu_tile_regimes.py runs the backbone at: greedy_cover(3, range(1, FRAME_RANGE + 1),
# SMS_H100_SXM, COVER_COST) in the order picked.  Together they reach every (precision, launch, regime) of the training
# schedule that some frame count in [1, FRAME_RANGE] reaches on a 132-SM H100 (tests/test_tile_regimes.py holds them to it).
# The cost is about what the per-launch check of one frame count takes: an engine and a float64 pass per frame plus a
# fixed part worth about 60 frames.
FRAME_RANGE = 640
COVER_COST = lambda f: f + 60          # noqa: E731
FRAME_SET = (1, 41, 73, 163, 17, 9, 325, 3, 518)

# umma_dev.cuh / umma_conv.cu / umma_wgrad.cu constants
BLOCK_M, BLOCK_K = 128, 64
MAX_STAGES = 8
PIPE_BYTES = 192 * 1024
A_BYTES = BLOCK_M * BLOCK_K * 2
MAX_BLOCK_N, N_STEP = 128, 16
MAX_PTILES = 768                 # UMMA_WGRAD_MAX_PTILES: longest pixel range of one weight-gradient split, in tiles


def _cdiv(a, b):
    return -(-a // b)


# ---- umma_conv_kernel ------------------------------------------------------------------------------------------------------
def pick_box(W):
    """(bw, bh, bf): the TMA box of one 128-row M tile (umma_conv.cu: pick_box)"""
    if W % 8 == 0 and W >= 56:
        return 8, 8, 2
    if W % 4 == 0:
        return 4, 4, 8
    if W % 2 == 0:
        return 2, 2, 32
    if W <= 8:
        return W, 1, BLOCK_M // W
    return 1, 1, 128


def conv_plan(W, H, frames, K, N, ntaps, split, sms, kchunks=None):
    """one umma_conv_kernel launch over a W x H x frames output (tiles enumerate output pixels; a stride-2 forward is planned
    at its output geometry); K reduction channels (kchunks: a fused data gradient's two padded sources), N output channels;
    split: EXACT_TC (four-plane stages)"""
    bw, bh, bf = pick_box(W)
    tw, th, tf = _cdiv(W, bw), _cdiv(H, bh), _cdiv(frames, bf)
    n_tiles = _cdiv(N, MAX_BLOCK_N)
    block_n = _cdiv(_cdiv(N, n_tiles), N_STEP) * N_STEP
    kchunks = _cdiv(K, BLOCK_K) if kchunks is None else kchunks
    stage_bytes = _cdiv((A_BYTES + block_n * BLOCK_K * 2) * (2 if split else 1), 1024) * 1024
    stages = min(PIPE_BYTES // stage_bytes, MAX_STAGES)
    total = tw * th * tf * n_tiles
    grid = min(total, sms)
    q, r = divmod(total, grid)
    per_cta = {t: n for t, n in ((q + 1, r), (q, grid - r)) if n}       # tiles per CTA -> number of CTAs
    return dict(box=(bw, bh, bf), tiles_w=tw, tiles_h=th, tiles_f=tf, n_tiles=n_tiles, block_n=block_n, kchunks=kchunks,
                ntaps=ntaps, ksteps=ntaps * kchunks, stages=stages, total=total, grid=grid, per_cta=per_cta,
                frames=frames, sms=sms)


def _odd_ge3(p):
    return any(t >= 3 and t % 2 for t in p["per_cta"])


CONV_REGIMES = {
    # fewer tiles than SMs: the grid is the tile count, every CTA one tile (consumer warpgroup 1 idle)
    "grid_below_sms": lambda p: p["total"] < p["sms"],
    # CTAs with 1 tile next to CTAs with 2: the order barrier runs in some CTAs only
    "one_and_two_tiles": lambda p: set(p["per_cta"]) == {1, 2},
    # an odd tile count >= 3: consumer 0 runs one tile more than consumer 1, the last arrive is skipped
    "odd_tiles_ge3": _odd_ge3,
    # CTAs with q and q + 1 tiles, q >= 2
    "uneven_tiles_ge2": lambda p: len(p["per_cta"]) == 2 and min(p["per_cta"]) >= 2,
    # the last frame box overhangs F: its rows past the last frame are clipped
    "partial_frame_box": lambda p: p["frames"] % p["box"][2] != 0,
    # ksteps < stages with >= 2 tiles in a CTA: the ring holds stages of both consumers' tiles at once
    "ring_holds_tiles": lambda p: p["ksteps"] < p["stages"] and max(p["per_cta"]) >= 2,
}


# ---- umma_wgrad_kernel -----------------------------------------------------------------------------------------------------
def wgrad_box(W):
    """(bw, bh, bf): the 64-pixel box of the weight gradient, chosen by the width of dz (umma_wgrad_bind_taps)"""
    if W % 8 == 0:
        return 8, 8, 1
    if W % 4 == 0:
        return 4, 4, 4
    if W % 2 == 0:
        return 2, 2, 16
    return 1, 1, 64


def wgrad_ctas(cin, cout, ntaps):
    """(m_tiles, n_tiles, block_n, taps_per_cta, tap_groups): the CTAs of one pixel split"""
    m_tiles = _cdiv(cout, BLOCK_M)
    chunks = _cdiv(cin, 64)
    n_tiles = _cdiv(chunks, 4)
    block_n = _cdiv(chunks, n_tiles) * 64
    tpc = min(max(1, 4 // (block_n // 64)), ntaps)
    groups = _cdiv(ntaps, tpc)
    tpc = _cdiv(ntaps, groups)                  # balanced: 9 taps as 3 + 3 + 3
    return m_tiles, n_tiles, block_n, tpc, groups


def wgrad_splits(ctas, ptiles, sms, waves=1):
    """split count before the bind's caps (umma_wgrad_splits): one wave of SMs / ctas splits, plus whole waves until no split
    sums more than MAX_PTILES pixel tiles"""
    per_wave = max(1, waves * sms // ctas)
    return max(1, _cdiv(_cdiv(ptiles, MAX_PTILES), per_wave)) * per_wave


def conv1_tsplits(in_channels, frames, sms):
    """the bound of conv1's split count (engine.cu: plan, conv1_tsplits): 128, or as many whole waves as keep a split at most
    MAX_PTILES pixel tiles long where 128 would not"""
    cs = _cdiv(4 * in_channels, 8) * 8
    wb = wgrad_box(112)
    ptiles = _cdiv(112, wb[0]) * _cdiv(112, wb[1]) * _cdiv(frames, wb[2])
    if _cdiv(ptiles, MAX_PTILES) <= 128:
        return 128
    m_tiles, n_tiles, _bn, _tpc, groups = wgrad_ctas(4 * cs, 64, 4)
    return wgrad_splits(m_tiles * n_tiles * groups, ptiles, sms)


def tsplits(frames, cin, cout, k, out_hw, sms):
    """the engine's bound on a layer's tensor-core split count (engine.cu: plan): the larger of the SIMT split heuristic and
    wgrad_splits (at most 128)"""
    M = frames * out_hw * out_hw
    taps = k * k
    flat = cin < 16
    tiles = _cdiv(cout, 64) * (_cdiv(taps * cin, 64) if flat else _cdiv(cin, 64) * taps)
    splits = min(_cdiv(592, tiles), 128)
    while splits > 1 and M // splits < 256:
        splits -= 1
    rows = _cdiv(_cdiv(M, splits), 16) * 16
    wsplits = _cdiv(M, rows)
    m_tiles, n_tiles, _bn, _tpc, groups = wgrad_ctas(cin, cout, taps)
    wb = wgrad_box(out_hw)
    ptiles = _cdiv(out_hw, wb[0]) * _cdiv(out_hw, wb[1]) * _cdiv(frames, wb[2])
    return max(wsplits, min(128, wgrad_splits(m_tiles * n_tiles * groups, ptiles, sms)))


def wgrad_plan(W, H, frames, cin, cout, ntaps, max_splits, sms, waves=1):
    """one umma_wgrad_kernel launch over a W x H x frames dz"""
    bw, bh, bf = wgrad_box(W)
    ptiles = _cdiv(W, bw) * _cdiv(H, bh) * _cdiv(frames, bf)
    m_tiles, n_tiles, block_n, tpc, groups = wgrad_ctas(cin, cout, ntaps)
    ctas = m_tiles * n_tiles * groups
    want = min(wgrad_splits(ctas, ptiles, sms, waves), max_splits)
    splits = max(1, min(want, ptiles))
    pps = _cdiv(ptiles, splits)
    n = _cdiv(ptiles, pps)
    return dict(box=(bw, bh, bf), ptiles=ptiles, m_tiles=m_tiles, n_tiles=n_tiles, block_n=block_n, taps_per_cta=tpc,
                tap_groups=groups, ntaps=ntaps, ctas=ctas, max_splits=max_splits, per_wave=max(1, waves * sms // ctas), wanted_splits=want, splits=n,
                ptiles_per_split=pps, last_split=ptiles - (n - 1) * pps, frames=frames, sms=sms)


WGRAD_REGIMES = {
    # the last split-K range is shorter than the others
    "short_last_split": lambda p: p["last_split"] < p["ptiles_per_split"],
    # one pixel tile per split
    "one_ptile_per_split": lambda p: p["ptiles_per_split"] == 1,
    # fewer pixel tiles than the splits SMs / ctas would give: the pixel count bounds the split count
    "splits_capped_by_ptiles": lambda p: p["ptiles"] < p["wanted_splits"],
    # rounding ptiles_per_split up leaves fewer splits than were asked for
    "splits_trimmed": lambda p: p["splits"] < min(p["wanted_splits"], p["ptiles"]),
    # more than one wave of splits: one wave would sum more than MAX_PTILES pixel tiles per split
    "extra_waves": lambda p: p["splits"] > p["per_wave"],
    # the box holds several frames and the last frame box overhangs F (zero-filled rows in the reduction)
    "partial_frame_box": lambda p: p["box"][2] > 1 and p["frames"] % p["box"][2] != 0,
}


# ---- the engine's launch schedule ------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _graph(in_channels):
    return S.Graph(in_channels)


def _fused_blocks(G):
    """the sibling 1x1 blocks (engine.cu: plan): (op1 or None, 3x3_reduce, double_3x3_reduce) conv ids per inception block"""
    ids = set(G.conv_ids)
    out = []
    for cid in G.conv_ids:
        if cid.endswith("_3x3_reduce") and "double" not in cid:
            pre = cid[:-len("3x3_reduce")]
            if pre + "double_3x3_reduce" in ids:
                out.append((pre + "1x1" if pre + "1x1" in ids else None, cid, pre + "double_3x3_reduce"))
    return out


def schedule(in_channels, frames, precision, sms=SMS_H100_SXM, training=True, waves=1):
    """[launch dict] of one forward (+ backward when training) of a tensor-core engine, in launch order: kernel, phase (0
    forward, 1 data gradient, 2 weight gradient), op (the launch log's op name: "a+b+c" for a fused sibling launch), plan"""
    if precision not in ("exact_tc", "fast"):
        raise ValueError("only the tensor-core precisions run the wgmma kernels")
    split = precision == "exact_tc"
    G = _graph(in_channels)
    conv = {o["id"]: o for o in G.ops if o["kind"] == "conv"}
    hw = lambda v: G.shape[v][2]
    cs = _cdiv(4 * in_channels, 8) * 8              # conv1 runs as a 4-tap convolution over the space-to-depth input
    fused = _fused_blocks(G)
    role = {}                                       # conv id -> ("leader" | "follower", block)
    for fb in fused:
        members = [c for c in fb if c is not None]
        for c in members:
            role[c] = ("leader" if c == members[0] else "follower", fb)
    launches = []

    def add(kernel, phase, op, plan):
        launches.append(dict(kernel=kernel, phase=phase, op=op, plan=plan))

    def fwd_plan(o):
        a = o["a"]
        W = hw(o["out"])
        if o["id"] == "conv1_7x7_s2":
            return conv_plan(W, W, frames, 4 * cs, a["cout"], 4, split, sms)
        return conv_plan(W, W, frames, a["cin"], a["cout"], a["k"] ** 2, split, sms)

    for o in G.ops:
        if o["kind"] != "conv" or role.get(o["id"], ("",))[0] == "follower":
            continue
        if o["id"] in role:
            op1, r3, rd = role[o["id"]][1]
            n = sum(conv[c]["a"]["cout"] for c in (op1, r3, rd) if c is not None)
            W = hw(o["inp"])
            add("umma_conv_kernel", 0, "+".join(c for c in (op1, r3, rd) if c is not None),
                conv_plan(W, W, frames, conv[r3]["a"]["cin"], n, 1, split, sms))
        else:
            add("umma_conv_kernel", 0, o["id"], fwd_plan(o))
    if not training:
        return launches
    for o in reversed(G.ops):
        if o["kind"] != "conv":
            continue
        a, cid = o["a"], o["id"]
        Wo = hw(o["out"])
        if cid == "conv1_7x7_s2":
            add("umma_wgrad_kernel", 2, cid, wgrad_plan(Wo, Wo, frames, 4 * cs, a["cout"], 4, conv1_tsplits(in_channels, frames, sms), sms,
                                                                 waves))
            continue                                # the network input has no gradient
        ts = tsplits(frames, a["cin"], a["cout"], a["k"], Wo, sms)
        add("umma_wgrad_kernel", 2, cid, wgrad_plan(Wo, Wo, frames, a["cin"], a["cout"], a["k"] ** 2, ts, sms, waves))
        Wi = hw(o["inp"])
        r = role.get(cid, ("",))[0]
        if r == "":                                 # stride 2: a stride-1 convolution of dz zero-upsampled to the input size
            add("umma_conv_kernel", 1, cid, conv_plan(Wi, Wi, frames, a["cout"], a["cin"], a["k"] ** 2, split, sms))
        elif r == "leader":
            op1, r3, rd = role[cid][1]
            nr = conv[r3]["a"]["cout"] + conv[rd]["a"]["cout"]
            if op1 is not None:
                k1 = conv[op1]["a"]["cout"]
                kc = _cdiv(k1, BLOCK_K) + _cdiv(nr, BLOCK_K)
                p = conv_plan(Wi, Wi, frames, k1 + nr, a["cin"], 1, split, sms, kchunks=kc)
            else:
                p = conv_plan(Wi, Wi, frames, nr, a["cin"], 1, split, sms)
            add("umma_conv_kernel", 1, "+".join(c for c in (op1, r3, rd) if c is not None), p)
    return launches


def log_key(launch):
    """what ssnb_timing_launches reports for the launch: (kernel, phase, op, a, b) with (a, b) = (tiles, block_n) for
    umma_conv_kernel and (ctas, splits) for umma_wgrad_kernel"""
    p = launch["plan"]
    ab = (p["total"], p["block_n"]) if launch["kernel"] == "umma_conv_kernel" else (p["ctas"], p["splits"])
    return (launch["kernel"], launch["phase"], launch["op"]) + ab


def parse_launch_log(text):
    """the umma_conv_kernel / umma_wgrad_kernel lines of ssnb_timing_launches as log_key tuples, in launch order"""
    out = []
    for line in text.splitlines():
        c = line.split("\t")
        if c[0] in ("umma_conv_kernel", "umma_wgrad_kernel"):
            out.append((c[0], int(c[1]), c[2], int(c[5]), int(c[6])))
    return out


PASS = {0: "fwd", 1: "dgrad", 2: "wgrad"}


def launch_id(launch):
    return "%s %s" % (PASS[launch["phase"]], launch["op"])


def regimes(launch):
    table = CONV_REGIMES if launch["kernel"] == "umma_conv_kernel" else WGRAD_REGIMES
    return {name for name, pred in table.items() if pred(launch["plan"])}


def reached(in_channels, frames, sms, precisions=("exact_tc", "fast")):
    """{(precision, launch id, regime)} of the training schedule at this frame count"""
    out = set()
    for prec in precisions:
        for l in schedule(in_channels, frames, prec, sms):
            out |= {(prec, launch_id(l), r) for r in regimes(l)}
    return out


def greedy_cover(in_channels, frame_range, sms, cost=lambda f: f):
    """greedy weighted set cover of every (precision, launch, regime) reached somewhere in frame_range: repeatedly the frame
    count with the most newly reached pairs per cost (ties: the smaller frame count).  Returns (chosen frame counts in the
    order picked, the union of reached pairs, {frame count: its pairs})"""
    per = {f: reached(in_channels, f, sms) for f in frame_range}
    universe = set().union(*per.values())
    left, chosen = set(universe), []
    while left:
        f = max(per, key=lambda f: (len(per[f] & left) / cost(f), -f))
        chosen.append(f)
        left -= per[f]
    return chosen, universe, per
