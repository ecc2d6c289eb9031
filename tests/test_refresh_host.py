"""Host side of critic inference and the priority refresh: the ctypes signatures against the header, the argument checks
of SacCore.critic_values and Replay.refresh_priorities, the learners' refresh_after_reset checks (raised before a handle
is built), and with stand-in cores the refreshes a learner enqueues after its resets and recycles.  No GPU needed."""
import json
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "b200sac.h")).read()


def _params(fn):
    decl = re.search(r"\nint %s\((.*?)\);" % fn, HDR, re.S).group(1)
    return [" ".join(p.split()[:-1]) for p in decl.replace("\n", " ").split(",")]


def test_ctypes_signatures_match_header():
    from distributed_sac_b200 import _lib
    C = _lib.C
    ctype = {"b200sac_t*": _lib._VP, "b200sac_replay_t*": _lib._VP, "int32_t": C.c_int32, "int64_t": C.c_int64,
             "uint64_t": C.c_uint64, "void*": _lib._VP, "const float*": _lib._VP, "float*": _lib._VP,
             "const int64_t*": _lib._VP, "int64_t*": C.POINTER(C.c_int64)}
    for fn in ("b200sac_critic_values", "b200sac_critic_values_chunk", "b200sac_replay_refresh_priorities"):
        res, args = _lib.SYMBOLS[fn]
        assert res is C.c_int
        assert args == [ctype[t] for t in _params(fn)], fn


class _Lib:
    """Records library calls instead of making them."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return 0
        return call


def _core(replicas=2):
    from distributed_sac_b200.core import CoreConfig, SacCore
    core = object.__new__(SacCore)
    core.cfg = CoreConfig(state_dim=3, act_dim=2, actor_hidden=[8], critic_hidden=[8], batch=8, replicas=replicas)
    core.lib = _Lib()
    core._h = None
    return core


def _replay(core):
    from distributed_sac_b200.core import Replay
    rb = object.__new__(Replay)
    rb.core, rb.lib, rb._h = core, core.lib, None
    return rb


@pytest.mark.parametrize("obs,act,kw", [((0, 3), (0, 2), {}), ((4, 3), (3, 2), {}), ((4, 2), (4, 2), {}),
                                        ((4, 3), (4, 3), {}), ((4,), (4, 2), {}), ((4, 3), (4, 2), dict(target=1)),
                                        ((4, 3), (4, 2), dict(target="yes"))])
def test_critic_values_refuses_bad_arguments(obs, act, kw):
    core = _core()
    with pytest.raises(ValueError):
        core.critic_values(torch.zeros(obs), torch.zeros(act), **kw)
    assert core.lib.calls == []


@pytest.mark.parametrize("kw", [dict(idx=[0, 1]), dict(idx=[0], replica=None), dict(stochastic=1),
                                dict(stochastic="no")])
def test_refresh_priorities_refuses_bad_arguments(kw):
    core = _core()
    with pytest.raises(ValueError):
        _replay(core).refresh_priorities(7, **kw)
    assert core.lib.calls == []


def test_refresh_priorities_calls(monkeypatch):
    from distributed_sac_b200 import core as core_mod
    monkeypatch.setattr(core_mod, "_stream", lambda: None)
    core = _core(replicas=3)
    _replay(core).refresh_priorities(2 ** 64 + 5)
    _replay(core).refresh_priorities(9, idx=[4, 4, 1], replica=1, stochastic=False)
    _replay(core).refresh_priorities(9, idx=[], replica=2)               # nothing to refresh: no call
    calls = [c for c in core.lib.calls if c[0] == "b200sac_replay_refresh_priorities"]
    assert [(a[1], a[2], a[4].value, a[5]) for _, a in calls] == [(0, 0, 5, 1), (1, 0, 5, 1), (2, 0, 5, 1), (1, 3, 9, 0)]
    assert calls[0][1][3].value is None


_LL = {"device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "lr_actor": 3e-4,
       "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 1000}
_PER = dict(alpha=0.6, beta=0.4, eps=1e-6)


def _no_handle(monkeypatch):
    from distributed_sac_b200 import core, learner as L

    def no_handle(*a, **k):
        raise AssertionError("a handle was built before the arguments were checked")
    monkeypatch.setattr(L, "SacCore", no_handle)
    monkeypatch.setattr(core, "SacCore", no_handle)
    return L


@pytest.mark.parametrize("value", [1, "yes", None, 0.0])
def test_learner_refuses_a_bad_refresh_after_reset(tmp_path, monkeypatch, value):
    import redis_stub
    L = _no_handle(monkeypatch)
    p = tmp_path / "ll.json"
    p.write_text(json.dumps(_LL))
    with pytest.raises(ValueError):
        L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)), replay_where="device",
                             prioritized=dict(_PER, refresh_after_reset=value))


def test_care_learner_refuses_refresh_after_reset(tmp_path, monkeypatch):
    L = _no_handle(monkeypatch)
    monkeypatch.setattr(L.CARELearner, "_set_dims", lambda self: setattr(self, "num_tasks", 10))
    p = tmp_path / "care.json"
    p.write_text("{}")
    with pytest.raises(ValueError, match="CARE"):
        L.CARELearner([], [], str(p), write_mode=False, replay_where="device", prioritized=dict(_PER, refresh_after_reset=True))


class _Log:
    def __init__(self):
        self.events = []

    def reset(self, seed, **parts):
        self.events.append(("reset", seed))

    def redo(self, seed, s, a, **taus):
        self.events.append(("redo", seed))


class _Ring:
    def __init__(self, log):
        self.log = log

    def refresh_priorities(self, seed, idx=None, replica=None, stochastic=True):
        assert idx is None and replica is None and stochastic is True
        self.log.events.append(("refresh", seed))


class _Memory:
    def __init__(self, log):
        self.ring = _Ring(log)

    def sample(self):
        return torch.zeros(4, 8), torch.zeros(4, 2)


def _stub_learner(refresh, reset_interval=None, redo_interval=None, seed=10):
    from distributed_sac_b200 import learner as L
    ln = object.__new__(L.LunarLanderLearner)
    log = _Log()
    ln.core, ln.memory = log, _Memory(log)
    ln.refresh_after_reset, ln.prioritized = refresh, dict(_PER)
    ln.reset_interval, ln.redo_interval, ln.reset, ln.redo = reset_interval, redo_interval, {}, dict(actor=0.0, critic=0.0)
    ln.seed, ln._n_updates, ln._n_manual_resets, ln._n_manual_redos, ln._n_manual_refreshes = seed, 0, 0, 0, 0
    ln.critic_layer_norm = False
    return ln, log


def test_scheduled_resets_and_recycles_are_followed_by_refreshes():
    ln, log = _stub_learner(True, reset_interval=4, redo_interval=6)
    assert sum(ln._chunks(13)) == 13
    s = ln.seed
    assert log.events == [("reset", s + 2 ** 32), ("refresh", s + 2 ** 32),
                          ("redo", s + 2 ** 62 + 2 ** 32), ("refresh", s + 2 ** 62 + 2 ** 32),
                          ("reset", s + 2 * 2 ** 32), ("refresh", s + 2 * 2 ** 32),
                          ("reset", s + 3 * 2 ** 32), ("refresh", s + 3 * 2 ** 32),
                          ("redo", s + 2 ** 62 + 2 * 2 ** 32), ("refresh", s + 2 ** 62 + 2 * 2 ** 32)]


def test_explicit_resets_and_recycles_are_followed_by_refreshes():
    ln, log = _stub_learner(True)
    ln.reset_networks()
    ln.recycle_dormant(seed=77)
    ln.refresh_priorities()
    s = ln.seed
    assert log.events == [("reset", s + 2 ** 63 + 2 ** 32), ("refresh", s + 2 ** 63 + 2 ** 32), ("redo", 77), ("refresh", 77),
                          ("refresh", s + 2 ** 63 + 2 ** 61 + 2 ** 32)]


def test_without_the_key_nothing_is_refreshed():
    ln, log = _stub_learner(False, reset_interval=2, redo_interval=3)
    sum(ln._chunks(7))
    ln.reset_networks(seed=1)
    ln.recycle_dormant(seed=2)
    assert [e[0] for e in log.events] == ["reset", "redo", "reset", "reset", "redo", "reset", "redo"]
