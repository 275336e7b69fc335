"""Forward engines at any frame count up to the planned one, CPU side: the header, the refusals of
ssnb_backbone_fwd_frames / ssnb_iv3_forward_frames before any launch, and reserve_frames() keeping one engine per model."""
import ctypes as C
import os
import re

import pytest

from ssn_b200 import _lib
from ssn_b200._lib import lib
from ssn_b200.engine import BackboneEngine, PlannedEngine
from ssn_b200.inception_v3 import InceptionV3Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# 20 distinct frame counts of a ragged 10-crop test loop with 40-tick chunks, and the reserved count
COUNTS = (400, 10, 20, 37, 40, 90, 127, 128, 129, 130, 200, 255, 256, 257, 300, 310, 370, 380, 390, 399)
RESERVED = 400


def test_header_declares_both_entry_points():
    with open(os.path.join(ROOT, "include", "ssnb.h")) as f:
        h = f.read()
    assert re.search(r"int ssnb_backbone_fwd_frames\(ssnb_handle h, const float\* input_nchw, int frames, float\* feat, void\* stream\);", h)
    assert re.search(r"int ssnb_iv3_forward_frames\(ssnb_iv3_handle h, const float\* input_nchw, int frames, float\* feat, void\* stream\);", h)
    for name in ("ssnb_backbone_fwd_frames", "ssnb_iv3_forward_frames"):
        assert _lib.SIGNATURES[name] == (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p])


# any non-null address: every call below is refused before the pointers are read
_P = C.c_void_p(4096)


@pytest.mark.parametrize("precision", [_lib.EXACT_FP32, _lib.FAST_FP16, _lib.EXACT_TC])
def test_backbone_fwd_frames_refusals_launch_nothing(precision):
    fwd = BackboneEngine(3, 16, precision, False, 1.0, None)
    trn = BackboneEngine(3, 16, precision, True, 1.0, None)
    n0 = lib.ssnb_global_launch_count()
    for n in (0, -1, 17, 1 << 30):
        assert lib.ssnb_backbone_fwd_frames(fwd.h, _P, n, _P, None) == 1, n                       # SSNB_EINVAL
        assert b"frames must be in 1 .. 16" in lib.ssnb_last_error(fwd.h)
    assert lib.ssnb_backbone_fwd_frames(fwd.h, None, 8, _P, None) == 1
    assert lib.ssnb_backbone_fwd_frames(fwd.h, _P, 8, None, None) == 1
    assert lib.ssnb_backbone_fwd_frames(None, _P, 8, _P, None) == 1
    for n in (1, 8, 16):                                                                            # SSNB_ESTATE, even at n == F
        assert lib.ssnb_backbone_fwd_frames(trn.h, _P, n, _P, None) == 3, n
        assert b"forward-only" in lib.ssnb_last_error(trn.h)
    # planned without a workspace: a valid call is refused for the state, still before any launch
    assert lib.ssnb_backbone_fwd_frames(fwd.h, _P, 8, _P, None) == 3
    assert lib.ssnb_global_launch_count() == n0


def test_backbone_fwd_frames_refuses_bn1_train():
    e = BackboneEngine(3, 8, _lib.EXACT_FP32, False, 1.0, None, bn1_train=True)
    n0 = lib.ssnb_global_launch_count()
    assert lib.ssnb_backbone_fwd_frames(e.h, _P, 4, _P, None) == 4                                 # SSNB_ENOSUPPORT
    assert lib.ssnb_global_launch_count() == n0


@pytest.mark.parametrize("precision", [_lib.EXACT_FP32, _lib.FAST_FP16, _lib.EXACT_TC])
def test_iv3_forward_frames_refusals_launch_nothing(precision):
    e = InceptionV3Engine(10, 37, precision)
    n0 = lib.ssnb_global_launch_count()
    for n in (0, -5, 38, 400):
        assert lib.ssnb_iv3_forward_frames(e.h, _P, n, _P, None) == 1, n
        assert b"frames must be in 1 .. 37" in lib.ssnb_last_error(None)
    assert lib.ssnb_iv3_forward_frames(e.h, None, 3, _P, None) == 1
    assert lib.ssnb_iv3_forward_frames(e.h, _P, 3, None, None) == 1
    assert lib.ssnb_iv3_forward_frames(None, _P, 3, _P, None) == 1
    assert lib.ssnb_iv3_forward_frames(e.h, _P, 3, _P, None) == 3                                  # no workspace
    assert lib.ssnb_global_launch_count() == n0


@pytest.fixture
def planned(monkeypatch):
    """engines planned with device=None (no workspace, no GPU); records every engine made and every weight pack"""
    made, packs = [], []
    for cls in (BackboneEngine, InceptionV3Engine):
        init = cls.__init__

        def wrapped(self, *a, _init=init, **k):
            _init(self, *a, **k)
            made.append(self)
        monkeypatch.setattr(cls, "__init__", wrapped)
    monkeypatch.setattr(PlannedEngine, "pack", lambda self, *a: packs.append(self))
    return made, packs


def _model(arch):
    import model_zoo
    return getattr(model_zoo, arch)(in_channels=3)


def _engine(m, arch, n, training=False):
    return m.engine_for(n, None) if arch == "InceptionV3" else m.engine_for(n, training, None)


@pytest.mark.parametrize("arch", ["InceptionV3", "BNInception"])
def test_reserve_frames_keeps_one_engine(planned, arch):
    made, packs = planned
    m = _model(arch)
    del made[:]                                  # InceptionV3's constructor plans a 1-frame engine for its op table
    m.reserve_frames(RESERVED)
    assert len(set(COUNTS)) == 20
    engines = {id(_engine(m, arch, n)) for n in COUNTS}
    assert len(engines) == 1 and len(m._engines) == 1
    (eng,) = m._engines.values()
    assert eng.frames == RESERVED and eng.device is None and len(made) == 1 and len(packs) == 1
    # back to one engine per frame count; the reserved engine keeps serving its own count
    m.reserve_frames(None)
    assert _engine(m, arch, RESERVED) is eng
    assert _engine(m, arch, 37).frames == 37 and len(m._engines) == 2


def test_reserve_frames_drops_per_count_forward_engines_only(planned):
    m = _model("BNInception")
    for n in (8, 24):
        _engine(m, "BNInception", n)
        _engine(m, "BNInception", n, training=True)
    assert len(m._engines) == 4
    m.reserve_frames(32)
    assert sorted((k[0], k[1]) for k in m._engines) == [(8, True), (24, True)]
    # autograd / fused_step engines stay per frame count, above the reserved count as well
    assert _engine(m, "BNInception", 8, training=True).frames == 8
    assert _engine(m, "BNInception", 48, training=True).frames == 48
    assert _engine(m, "BNInception", 8).frames == 32
    # bn_mode='partial' (bn1_train) is not reserved
    assert m.engine_for(8, False, None, bn1_train=True).frames == 8


@pytest.mark.parametrize("arch", ["InceptionV3", "BNInception"])
def test_forward_above_reserved_raises_before_the_library(planned, arch):
    made, packs = planned
    m = _model(arch)
    del made[:]
    m.reserve_frames(RESERVED)
    n0 = lib.ssnb_global_launch_count()
    with pytest.raises(ValueError, match="exceeds the 400 frames reserved"):
        _engine(m, arch, RESERVED + 1)
    assert not made and not packs and not m._engines and lib.ssnb_global_launch_count() == n0
    with pytest.raises(ValueError):
        m.reserve_frames(0)
