"""CPU side of the frame-count sweep: which tile-schedule regimes of the wgmma kernels each launch of the backbone's training
schedule reaches at which frame count (oracle/tile_plan.py), and that the frame counts tests/test_gpu_tile_regimes.py runs
(tile_plan.FRAME_SET) reach all of them.  Run with -s to see the chosen set and the coverage table."""
import collections

import pytest

from oracle import tile_plan as T

FRAMES = range(1, T.FRAME_RANGE + 1)
_PER = {}


def _per_frame(sms):
    if sms not in _PER:
        _PER[sms] = {f: T.reached(3, f, sms) for f in FRAMES}
    return _PER[sms]


def _table(universe, covered):
    """rows: regime, pairs reachable in the range, pairs the frame set reaches"""
    n_all = collections.Counter(r for _p, _l, r in universe)
    n_cov = collections.Counter(r for _p, _l, r in covered)
    return ["    %-24s %5d %5d" % (r, n_all[r], n_cov[r]) for r in sorted(n_all)]


def _launch_ids():
    return {(p, T.launch_id(l)) for p in ("exact_tc", "fast") for l in T.schedule(3, 1, p)}


def test_frame_set_reaches_every_regime():
    """every (precision, launch, regime) that some frame count in [1, 640] reaches at 132 SMs is reached by FRAME_SET"""
    per = _per_frame(T.SMS_H100_SXM)
    universe = set().union(*per.values())
    covered = set().union(*(per[f] for f in T.FRAME_SET))
    chosen, _u, _p = T.greedy_cover(3, FRAMES, T.SMS_H100_SXM, T.COVER_COST)
    print("\n132 SMs: frame set %s (greedy now picks %s), %d of %d (precision, launch, regime) pairs" % (
        list(T.FRAME_SET), chosen, len(covered), len(universe)))
    print("    %-24s %5s %5s" % ("regime", "reach", "set"), *_table(universe, covered), sep="\n")
    # the pairs no frame count in the range reaches, regime by regime
    regs = sorted(set(T.CONV_REGIMES) | set(T.WGRAD_REGIMES))
    kinds = {(p, T.launch_id(l)): l["kernel"] for p in ("exact_tc", "fast") for l in T.schedule(3, 1, p)}
    print("unreachable in [1, %d] at 132 SMs:" % T.FRAME_RANGE)
    for r in regs:
        table = T.CONV_REGIMES if r in T.CONV_REGIMES else T.WGRAD_REGIMES
        never = {lid for lid, k in kinds.items()
                 if r in table and (k == "umma_conv_kernel") == (table is T.CONV_REGIMES) and lid + (r,) not in universe}
        # a launch unreachable in both precisions is listed once, without the precision
        names = sorted({l if all((p, l) in never for p in ("exact_tc", "fast")) else "%s %s" % (p, l) for p, l in never})
        print("  %s (%d pairs): %s" % (r, len(never), ", ".join(names) if names else "-"))
    missing = sorted(universe - covered)
    assert not missing, "FRAME_SET misses %d pairs, e.g. %s" % (len(missing), missing[:10])
    # every regime is reached by some launch, by both kernels where it is named for both
    for table in (T.CONV_REGIMES, T.WGRAD_REGIMES):
        kernel = "umma_conv_kernel" if table is T.CONV_REGIMES else "umma_wgrad_kernel"
        reach = {r for (p, lid, r) in covered if kinds[(p, lid)] == kernel}
        assert reach == set(table), (kernel, set(table) - reach)
    assert len(T.FRAME_SET) == len(set(T.FRAME_SET)) and all(1 <= f <= T.FRAME_RANGE for f in T.FRAME_SET)


def test_coverage_at_114_sms():
    """the split depends on the SM count as well: FRAME_SET's coverage on an H100 PCIe (114 SMs), reported.  Only the
    regimes themselves are required to stay reachable; which pairs the set reaches there is printed."""
    per = _per_frame(T.SMS_H100_PCIE)
    universe = set().union(*per.values())
    covered = set().union(*(per[f] for f in T.FRAME_SET))
    chosen, _u, _p = T.greedy_cover(3, FRAMES, T.SMS_H100_PCIE, T.COVER_COST)
    print("\n114 SMs: frame set %s reaches %d of %d pairs (%.1f %%); a cover for 114 SMs would be %s" % (
        list(T.FRAME_SET), len(covered), len(universe), 100.0 * len(covered) / len(universe), chosen))
    print("    %-24s %5s %5s" % ("regime", "reach", "set"), *_table(universe, covered), sep="\n")
    assert {r for (_p, _l, r) in universe} == set(T.CONV_REGIMES) | set(T.WGRAD_REGIMES)


@pytest.mark.parametrize("sms", [T.SMS_H100_SXM, T.SMS_H100_PCIE])
@pytest.mark.parametrize("frames", sorted(T.FRAME_SET) + [288, 576])
def test_plan_invariants(frames, sms):
    """what the kernels rely on: grid <= SMs and <= the tile count, the per-CTA counts are the round robin's, the splits
    cover every pixel tile once with a non-empty last split and none sums more than MAX_PTILES tiles where the partials have
    room for more splits, and the launch list is the same for both precisions"""
    for prec in ("exact_tc", "fast"):
        ls = T.schedule(3, frames, prec, sms)
        for l in ls:
            p = l["plan"]
            if l["kernel"] == "umma_conv_kernel":
                assert 1 <= p["grid"] <= min(sms, p["total"])
                assert sum(t * n for t, n in p["per_cta"].items()) == p["total"]
                assert sum(p["per_cta"].values()) == p["grid"]
                assert [-(-(p["total"] - b) // p["grid"]) for b in (0, p["grid"] - 1)] == [max(p["per_cta"]), min(p["per_cta"])]
                assert p["block_n"] % 16 == 0 and p["block_n"] <= 128 and p["n_tiles"] * p["block_n"] >= 16
                assert 1 <= p["stages"] <= T.MAX_STAGES
            else:
                assert 1 <= p["splits"] <= min(p["ptiles"], p["max_splits"])
                # as many whole waves of splits as keep a split at most MAX_PTILES pixel tiles long, unless the planner's
                # bound of the layer's split count (at most 128 but for conv1) stops it
                assert p["ptiles_per_split"] <= T.MAX_PTILES or p["splits"] == p["max_splits"]
                assert (p["splits"] - 1) * p["ptiles_per_split"] + p["last_split"] == p["ptiles"]
                assert 1 <= p["last_split"] <= p["ptiles_per_split"]
                assert p["taps_per_cta"] * p["block_n"] // 64 <= 4 and p["tap_groups"] * p["taps_per_cta"] >= p["ntaps"]
        assert [(l["kernel"], l["phase"], l["op"]) for l in ls] == \
            [(l["kernel"], l["phase"], l["op"]) for l in T.schedule(3, frames, "fast", sms)]
    # 69 weight gradients; 51 forwards (the 28 sibling 1x1 convolutions of the 10 blocks run as one launch per block); a data
    # gradient for every forward but conv1's
    fwd = [l for l in ls if l["phase"] == 0]
    assert len([l for l in ls if l["phase"] == 2]) == 69 and len(fwd) == 69 - 28 + 10
    assert len([l for l in ls if l["phase"] == 1]) == len(fwd) - 1
    assert len(T.schedule(3, frames, "fast", sms, training=False)) == len(fwd)


def test_launch_ids_are_unique():
    ids = [(p, T.launch_id(l)) for p in ("exact_tc", "fast") for l in T.schedule(3, 1, p)]
    assert len(ids) == len(set(ids)) == len(_launch_ids())
