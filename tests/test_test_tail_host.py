"""The packed test-time tail (ssn_test.py:87-92 for many videos per call) without a GPU: the numpy oracle
(oracle/test_tail_oracle.py) against tests/golden/test_tail.npz, which holds what the reference's STPPReorgainzed and the
script's de-normalisation lines computed (oracle/gen_golden_test_tail.py); the argument checks of ops.ssn_ops.reorg_packed
and of ssnb_stpp_reorg_batch, which refuse before any launch; the header declarations."""
import ast
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import test_tail_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "test_tail.npz"))
SETS = sorted({k.split("_", 1)[0] for k in GOLD.files if k.endswith("_K")})
SSNB_EINVAL, SSNB_ENOSUPPORT = 1, 4


def golden_set(name):
    """-> dict(K, cfg, tick_offsets, offsets, scores, ticks, scaling, act64, comp64, reg64, reg_raw32, reg32)"""
    f = {k[len(name) + 1:]: GOLD[k] for k in GOLD.files if k.startswith(name + "_")}
    f["K"] = int(f["K"])
    f["cfg"] = ast.literal_eval(str(f["cfg"]))
    return f


def lens(K):
    return K + 1, K, 2 * K


def rel_err(got, ref):
    """max |got - ref| / max(1, max |ref|), NaN positions required to match (inf when they do not)"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if got.shape != ref.shape or not (np.isnan(got) == np.isnan(ref)).all():
        return float("inf")
    ok = ~np.isnan(ref)
    if not ok.any():
        return 0.0
    return float(np.abs(got[ok] - ref[ok]).max() / max(1.0, np.abs(ref[ok]).max()))


@pytest.mark.parametrize("name", SETS)
def test_oracle_pooling_equals_reference_float64(name):
    f = golden_set(name)
    got = TO.reorg_packed64(f["scores"], f["tick_offsets"], f["ticks"], f["scaling"], f["offsets"], *lens(f["K"]), f["cfg"])
    for q, g, r in zip(("act", "comp", "reg"), got, (f["act64"], f["comp64"], f["reg64"])):
        assert rel_err(g.numpy(), r) <= 1e-12, (name, q, rel_err(g.numpy(), r))


@pytest.mark.parametrize("name", SETS)
def test_oracle_denorm_bitwise_equals_reference(name):
    f = golden_set(name)
    got = TO.denorm32(f["reg_raw32"], GOLD["reg_stats"])
    assert got.dtype == np.float32 and got.tobytes() == f["reg32"].tobytes()
    # the two ops rounded on their own: a fused multiply-add differs somewhere
    x = f["reg_raw32"].reshape(len(got), -1, 2).astype(np.float64)
    st = GOLD["reg_stats"]
    fused = np.stack([(x[:, :, c] * np.float32(st[1, c]) + np.float32(st[0, c])).astype(np.float32) for c in (0, 1)], 2)
    assert fused.tobytes() != f["reg32"].tobytes()


def test_fixtures_cover_the_edges():
    Ks, cfgs, Ts, fallback, touch0, touchT, negative, empty_act = set(), set(), set(), 0, 0, 0, 0, 0
    for name in SETS:
        f = golden_set(name)
        Ks.add(f["K"])
        cfgs.add(f["cfg"])
        to, o = f["tick_offsets"], f["offsets"]
        for v in range(len(o) - 1):
            T, tk = int(to[v + 1] - to[v]), f["ticks"][o[v]:o[v + 1]]
            Ts.add(T)
            fallback += len(tk) == 1
            touch0 += bool((tk[:, 1] == 0).any())
            touchT += bool((tk[:, 2] == T).any())
            negative += bool((tk < 0).any())
        empty_act += int(np.isnan(f["act64"]).any(1).sum())
    assert {20, 200} <= Ks and {(1, (1, 2), 1), ((1, 3), (1, 2, 3, 5), (1, 6))} <= cfgs
    assert 1 in Ts and fallback >= 2 and touch0 and touchT and negative and empty_act
    assert 8 <= sum(len(golden_set(n)["offsets"]) - 1 for n in SETS) <= 12
    st = GOLD["reg_stats"]
    assert st.shape == (2, 2) and all(float(np.float32(x)) != x for x in st.reshape(-1))     # not representable in fp32


def test_oracle_skips_videos_without_rows():
    f = golden_set(SETS[0])
    to, o = list(f["tick_offsets"]), list(f["offsets"])
    to2, o2 = to[:2] + to[1:], o[:2] + o[1:]            # a video with T = 0 and N = 0 after the first
    a = TO.reorg_packed64(f["scores"], to, f["ticks"], f["scaling"], o, *lens(f["K"]), f["cfg"])
    b = TO.reorg_packed64(f["scores"], to2, f["ticks"], f["scaling"], o2, *lens(f["K"]), f["cfg"])
    for x, y in zip(a, b):
        assert rel_err(x.numpy(), y.numpy()) == 0.0


# ---- the wrapper's checks, before anything reaches the device ----------------------------------------------------------------
def _args(V=2, T=(3, 4), N=(2, 1), K=2, cfg=(1, (1, 2), 1)):
    D = K + 1 + 5 * 3 * K
    toff, off = np.concatenate([[0], np.cumsum(T)]).tolist(), np.concatenate([[0], np.cumsum(N)]).tolist()
    return dict(scores=torch.zeros(sum(T), D), tick_offsets=toff, ticks32=torch.zeros(sum(N), 4, dtype=torch.int32),
                scaling32=torch.zeros(sum(N), 2), offsets=off, stpp_cfg=cfg, act_len=K + 1, comp_len=K, reg_len=2 * K)


@pytest.mark.parametrize("change, message", [
    (dict(tick_offsets=[0, 3]), "describe"),
    (dict(offsets=[1, 2, 3]), "starting at 0"),
    (dict(offsets=[0, 2, 1]), "non-decreasing"),
    (dict(tick_offsets=[0, 4, 3]), "non-decreasing"),
    (dict(tick_offsets=[0, 3, 8]), "scores must be"),
    (dict(scores=torch.zeros(7)), "scores must be"),
    (dict(act_len=2), "does not match"),
    (dict(stpp_cfg=(1, (1, 2, 3), 1)), "does not match"),
    (dict(stpp_cfg=(1, 1)), "three stages"),
    (dict(ticks32=torch.zeros(2, 4, dtype=torch.int32)), "ticks32 must be"),
    (dict(scaling32=torch.zeros(3, 3)), "ticks32 must be"),
    (dict(reg_stats=np.zeros((2, 3))), "reg_stats"),
    (dict(reg_stats=np.zeros(4)), "reg_stats"),
])
def test_reorg_packed_argument_checks(change, message):
    from ops.ssn_ops import reorg_packed
    a = _args()
    a.update(change)
    with pytest.raises(ValueError, match=message):
        reorg_packed(**a)


def test_reorg_packed_needs_cuda_tensors():
    from ops.ssn_ops import reorg_packed
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        reorg_packed(**_args(), reg_stats=np.ones((2, 2)))


# ---- the library's refusals: returned before any launch, so they run without a device ---------------------------------------
def _call(toff=(0, 3, 7), off=(0, 2, 3), D=33, act=3, comp=2, reg=4, counts=(1, 2, 1), levels=(1, 1, 2, 1), stats=None, ws_bytes=None,
          null=()):
    from ssn_b200._lib import lib, int_array
    V = len(off) - 1
    ct, co = (C.c_int64 * len(toff))(*toff), (C.c_int64 * len(off))(*off)
    fake = 1 << 20                                     # never dereferenced: every call here is refused, or has no row to write

    def p(name):
        return None if name in null else fake
    if ws_bytes is None:
        ws_bytes = (toff[-1] + V) * D * 8
    st = None if stats is None else (C.c_double * 4)(*stats)
    return lib.ssnb_stpp_reorg_batch(p("scores"), D, ct, p("toff_dev"), p("ticks"), p("scaling"), co, p("off_dev"), V, act, comp, reg,
                                     int_array(counts), int_array(levels), st, p("act"), p("comp"), p("reg"), p("ws"), ws_bytes, None)


def test_batch_workspace_bytes():
    from ssn_b200._lib import lib
    assert lib.ssnb_stpp_reorg_batch_workspace_bytes((C.c_int64 * 4)(0, 3, 3, 10), 3, 1601) == (10 + 3) * 1601 * 8
    assert lib.ssnb_stpp_reorg_batch_workspace_bytes((C.c_int64 * 1)(0), 0, 1601) == 0
    for offs, V, D in (((0, 3, 2), 2, 5), ((1, 3), 1, 5), ((0, 3), 1, 0), ((0, 3), -1, 5), ((0, 3), 1, 65535 * 128 + 1)):
        assert lib.ssnb_stpp_reorg_batch_workspace_bytes((C.c_int64 * len(offs))(*offs), V, D) == 0


@pytest.mark.parametrize("kw, rc", [
    (dict(toff=(0, 3, 2)), SSNB_EINVAL),              # tick offsets not monotone
    (dict(off=(0, 2, 1)), SSNB_EINVAL),               # row offsets not monotone
    (dict(toff=(1, 3, 7)), SSNB_EINVAL),              # not starting at 0
    (dict(D=34), SSNB_EINVAL),                        # D does not match act + M * (comp + reg)
    (dict(counts=(0, 2, 1)), SSNB_EINVAL),            # a stage without levels
    (dict(counts=(1, 2, 1), levels=(1, 0, 3, 1)), SSNB_EINVAL),    # a level with no part
    (dict(reg=3, D=3 + 5 * 5), SSNB_EINVAL),          # odd reg_len with reg_stats
    (dict(ws_bytes=(7 + 2) * 33 * 8 - 1), SSNB_EINVAL),            # workspace too small
    (dict(null=("toff_dev",)), SSNB_EINVAL),
    (dict(null=("reg",)), SSNB_EINVAL),
    (dict(null=("ws",)), SSNB_EINVAL),
    (dict(act=-1, D=-1 + 5 * 6), SSNB_EINVAL),
    (dict(off=(0, 2, 2 ** 31 + 5)), SSNB_ENOSUPPORT),  # more rows than one grid holds
    (dict(toff=(0, 3, 2 ** 31 + 3)), SSNB_ENOSUPPORT),  # a video of more than INT_MAX ticks
])
def test_batch_refusals(kw, rc):
    from ssn_b200._lib import lib
    kw.setdefault("stats", (0.1, 0.2, 0.3, 0.4))
    assert _call(**kw) == rc
    assert lib.ssnb_last_error(None)


def test_batch_without_rows_launches_nothing():
    """V = 0 and videos without proposal rows return before any launch: no device is needed"""
    from ssn_b200._lib import lib
    n = lib.ssnb_global_launch_count()
    assert _call(toff=(0,), off=(0,), null=("scores", "ticks", "scaling", "act", "comp", "reg", "ws", "toff_dev", "off_dev")) == 0
    assert _call(toff=(0, 3, 7), off=(0, 0, 0), null=("ticks", "scaling", "act", "comp", "reg", "ws")) == 0
    assert lib.ssnb_global_launch_count() == n


def test_header_declares_the_batch_entries():
    from ssn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "ssnb.h")).read()
    for name in ("ssnb_stpp_reorg_batch_workspace_bytes", "ssnb_stpp_reorg_batch"):
        m = re.search(r"\b%s\s*\(([^;]*)\);" % name, hdr)
        assert m, name
        params = [x for x in m.group(1).split(",") if x.strip()]
        assert len(params) == len(_lib.SIGNATURES[name][1]), name
    block = hdr[hdr.index("ssn_test.py:87-92"):hdr.index("ssnb_stpp_reorg_batch_workspace_bytes(")]
    assert "STPPReorgainzed" in block and "ops/ssn_ops.py" in block and "reg_stats" in block
