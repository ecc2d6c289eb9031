"""Host side of dormant-neuron recycling: the ctypes signatures of b200sac_redo / b200sac_read_redo against the header,
SacCore.redo's keyword checks (redo_taus) and the learners' argument checks, every refusal raised before a handle is
built; none of it needs a GPU."""
import json
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "b200sac.h")).read()


def _params(fn):
    decl = re.search(r"\nint %s\((.*?)\);" % fn, HDR, re.S).group(1)
    return [" ".join(p.split()[:-1]) for p in decl.replace("\n", " ").split(",")]


def test_ctypes_signatures_match_header():
    from distributed_sac_b200 import _lib
    C = _lib.C
    ctype = {"b200sac_t*": _lib._VP, "int32_t": C.c_int32, "int32_t n": C.c_int32, "int64_t": C.c_int64,
             "double": C.c_double, "uint64_t": C.c_uint64, "void*": _lib._VP, "const float*": _lib._VP,
             "double*": _lib._VP, "uint8_t*": _lib._VP, "int64_t*": C.POINTER(C.c_int64)}
    for fn in ("b200sac_redo", "b200sac_read_redo"):
        res, args = _lib.SYMBOLS[fn]
        assert res is C.c_int
        assert args == [ctype[t] for t in _params(fn)], fn


def test_taus():
    from distributed_sac_b200.core import redo_taus
    assert redo_taus() == (-math.inf, -math.inf)
    assert redo_taus(actor=0.1) == (0.1, -math.inf)
    assert redo_taus(critic=0) == (-math.inf, 0.0)
    assert redo_taus(np.float32(0.5), -1) == (0.5, -1.0)
    assert redo_taus(math.inf, -math.inf) == (math.inf, -math.inf)


@pytest.mark.parametrize("kw", [dict(actor=math.nan), dict(critic=float("nan")), dict(actor=True), dict(critic="0.1"),
                                dict(actor=[0.1]), dict(critic=np.nan), dict(actor=np.bool_(True))])
def test_bad_taus_raise_value_error(kw):
    from distributed_sac_b200.core import redo_taus
    with pytest.raises(ValueError):
        redo_taus(**kw)


_LL = {"device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "lr_actor": 3e-4,
       "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 1000}


@pytest.mark.parametrize("kw", [dict(redo_interval=0), dict(redo_interval=2.5), dict(redo_interval=True),
                                dict(redo_interval="3"), dict(redo=dict(actor=0.1)),
                                dict(redo_interval=5, redo=dict(actor=math.nan)),
                                dict(redo_interval=5, redo=dict(q1=0.1)), dict(redo_interval=5, redo=0.1),
                                dict(redo_interval=5, redo=dict(critic="low"))])
def test_learner_refuses_bad_redo_arguments_before_building_a_handle(tmp_path, kw, monkeypatch):
    import redis_stub
    from distributed_sac_b200 import core, learner as L

    def no_handle(*a, **k):
        raise AssertionError("a handle was built before the arguments were checked")
    monkeypatch.setattr(L, "SacCore", no_handle)
    monkeypatch.setattr(core, "SacCore", no_handle)
    p = tmp_path / "ll.json"
    p.write_text(json.dumps(_LL))
    with pytest.raises(ValueError):
        L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)), **kw)
