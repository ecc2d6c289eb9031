"""Host side of prior-data rings: the ctypes signatures against the header, the argument checks of Replay.attach_prior /
set_prior_rows and of the learners' prior= (raised before a handle is built), the learners' split with stand-in rings, and
self-checks of oracle/mix_ref.py, the numpy restatement of the device draw.  No GPU needed."""
import json
import math
import os
import re

import numpy as np
import pytest

import mix_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "b200sac.h")).read()


def _params(fn):
    decl = re.search(r"\nint %s\((.*?)\);" % fn, HDR, re.S).group(1)
    return [" ".join(p.split()[:-1]) for p in decl.replace("\n", " ").split(",")]


def test_ctypes_signatures_match_header():
    from distributed_sac_b200 import _lib
    C = _lib.C
    ctype = {"b200sac_replay_t*": _lib._VP, "int32_t": C.c_int32, "void*": _lib._VP, "int32_t*": C.POINTER(C.c_int32)}
    for fn in ("b200sac_replay_attach_prior", "b200sac_replay_set_prior_rows", "b200sac_replay_get_prior_rows"):
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


def _replay(core, h=None):
    from distributed_sac_b200.core import Replay
    rb = object.__new__(Replay)
    rb.core, rb.lib, rb._h, rb._prior = core, core.lib, h, None
    return rb


@pytest.mark.parametrize("call", [lambda rb: rb.attach_prior("ring"), lambda rb: rb.attach_prior(3),
                                  lambda rb: rb.set_prior_rows(True), lambda rb: rb.set_prior_rows(1.5),
                                  lambda rb: rb.set_prior_rows(float("nan")), lambda rb: rb.set_prior_rows("2")])
def test_replay_refuses_bad_arguments(call):
    core = _core()
    with pytest.raises(ValueError):
        call(_replay(core))
    assert core.lib.calls == []


def test_replay_calls_and_keeps_the_prior(monkeypatch):
    from distributed_sac_b200 import core as core_mod
    monkeypatch.setattr(core_mod, "_stream", lambda: None)
    core = _core(replicas=3)
    rb, prior = _replay(core, "online"), _replay(core, "prior")
    rb.attach_prior(prior)
    assert rb._prior is prior
    rb.set_prior_rows(4)
    rb.set_prior_rows(2.0, replica=1)
    rb.attach_prior(None)
    assert rb._prior is None
    assert core.lib.calls[0] == ("b200sac_replay_attach_prior", ("online", "prior"))
    assert [(n, a[:3]) for n, a in core.lib.calls[1:5]] == [("b200sac_replay_set_prior_rows", ("online", r, m))
                                                          for r, m in ((0, 4), (1, 4), (2, 4), (1, 2))]
    assert core.lib.calls[5] == ("b200sac_replay_attach_prior", ("online", None))


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


@pytest.mark.parametrize("prior,kw", [
    (dict(capacity=1000, fraction=0.5), dict(replay_where="host")),
    (dict(capacity=1000, fraction=0.5), dict(replay_where="device", prioritized=_PER)),
    (dict(capacity=1000, fraction=0.5), dict(replay_where="device", n_step=3)),
    (dict(capacity=1000, fraction=-0.1), {}), (dict(capacity=1000, fraction=1.5), {}),
    (dict(capacity=1000, fraction=float("nan")), {}), (dict(capacity=1000, fraction=True), {}),
    (dict(capacity=1000, fraction="0.5"), {}), (dict(capacity=1000), {}),
    (dict(capacity=1000, fraction=0.5, seed=3), {}), (dict(capacity=0, fraction=0.5), {}),
    (dict(capacity=1e4, fraction=0.5), {}), ([1000, 0.5], {})])
def test_learner_refuses_a_bad_prior(tmp_path, monkeypatch, prior, kw):
    import redis_stub
    L = _no_handle(monkeypatch)
    p = tmp_path / "ll.json"
    p.write_text(json.dumps(_LL))
    kw = dict(dict(replay_where="device"), **kw)
    with pytest.raises(ValueError):
        L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)), prior=prior, **kw)


class _Ring:
    def __init__(self):
        self.m = []

    def set_prior_rows(self, m, replica=None):
        self.m.append(m)


class _Memory:
    def __init__(self):
        self.ring = _Ring()


@pytest.mark.parametrize("batch,tasks,f,m", [(256, 0, 0.5, 128), (256, 0, 0.0, 0), (256, 0, 1.0, 256), (100, 0, 0.333, 33),
                                             (130, 10, 0.5, 7), (130, 10, 0.25, 3), (120, 4, 0.1, 3)])
def test_learner_split(batch, tasks, f, m):
    from distributed_sac_b200 import learner as L
    ln = object.__new__(L.MTSACLearner)
    ln.memory, ln.prior, ln.batch_size, ln.num_tasks = _Memory(), dict(capacity=10, fraction=0.0), batch, tasks
    ln.set_prior_fraction(f)
    assert ln.memory.ring.m == [m] == [math.floor(f * (batch // max(tasks, 1)) + 0.5)]
    assert ln.prior["fraction"] == f
    with pytest.raises(ValueError):
        ln.set_prior_fraction(1.01)
    assert ln.memory.ring.m == [m]


def test_learner_without_prior_refuses_prior_calls():
    from distributed_sac_b200 import learner as L
    ln = object.__new__(L.LunarLanderLearner)
    ln.prior = None
    for call in (lambda: ln.set_prior_fraction(0.5), lambda: ln.push_prior([], [], [], [], [])):
        with pytest.raises(ValueError):
            call()


# ---------------------------------------------------------------------------------------------------------------------
# oracle/mix_ref.py
# ---------------------------------------------------------------------------------------------------------------------
# (batch, num_tasks, online fills, prior fills): per-task fills at the sampler's minimum (4 per-task batches) make
# collisions, and with them redraws, common
CASES = {
    "single": (64, 0, [256], [300]),
    "tight": (32, 0, [128], [128]),
    "mt4": (40, 4, [40, 55, 70, 43], [40, 40, 47, 90]),
    "mt10": (130, 10, [52 + 3 * t for t in range(10)], [60 - 2 * t for t in range(10)]),
}


def _rings(name, cap_on=500, cap_pr=700):
    B, T, fo, fp = CASES[name]
    return B, T, mix_ref.Ring(11, fo, cap_on), mix_ref.Ring(29, fp, cap_pr)


@pytest.mark.parametrize("name", list(CASES))
def test_mix_ref_layout_and_distinct_slots(name):
    B, T, on, pr = _rings(name)
    Teff, P = max(T, 1), B // max(T, 1)
    for step, m in [(0, 1), (1, P // 2), (7, P - 1), (2 ** 32 + 3, P // 3)]:
        for replica in (0, 2):
            idx = mix_ref.draw(step, replica, B, T, m, on, pr)
            is_p, k = mix_ref.decode(idx)
            j = np.arange(B) % P
            t = np.arange(B) // P
            assert (is_p == (j < m)).all()
            cap = np.where(is_p, pr.cap_per_task, on.cap_per_task)
            fill = np.where(is_p, np.asarray(pr.fill)[t], np.asarray(on.fill)[t])
            assert (k // cap == t).all() and (k % cap < fill).all()
            for tt in range(Teff):
                for part in (True, False):
                    sel = (t == tt) & (is_p == part)
                    assert len(set(k[sel].tolist())) == sel.sum()


def _first_draws(ring, replica, step, B, T):
    """Attempt-0 draws of every slot (no duplicate rule)."""
    P = B // max(T, 1)
    i = np.arange(B)
    return mix_ref._draws(ring, replica, step, i, np.zeros(B, np.int64), np.minimum(i // P, max(T, 1) - 1))


@pytest.mark.parametrize("name", list(CASES))
def test_mix_ref_reduces_to_the_plain_draw(name):
    B, T, on, pr = _rings(name)
    P = B // max(T, 1)
    collided = False
    for step in (0, 5, 2 ** 33 + 1):
        plain_on = mix_ref.draw(step, 1, B, T, 0, on)
        assert (mix_ref.draw(step, 1, B, T, 0, on, pr) == plain_on).all()
        plain_pr = mix_ref.draw(step, 1, B, T, 0, mix_ref.Ring(pr.seed, pr.fill, pr.cap_per_task))
        assert (mix_ref.draw(step, 1, B, T, P, on, pr) == -1 - plain_pr).all()
        first = _first_draws(on, 1, step, B, T)
        keep = np.ones(B, bool)                 # the lowest slot of each index keeps its first draw
        for i in range(B):
            keep[i] = first[i] not in first[:i]
        assert (plain_on[keep] == first[keep]).all()
        collided |= not keep.all()
    assert collided or name == "single"


def test_mix_ref_parts_do_not_compete():
    """Online and prior rings of the same seed and fills: an online slot keeps its first draw unless a lower online slot
    drew the same index, whatever the prior slots drew -- and with these fills some prior slot does draw it."""
    B, T, m = 32, 0, 16
    on, pr = mix_ref.Ring(5, [128], 128), mix_ref.Ring(5, [128], 128)
    shared = 0
    for step in range(6):
        mixed = mix_ref.draw(step, 0, B, T, m, on, pr)
        first = _first_draws(on, 0, step, B, T)
        for i in range(m, B):
            if first[i] not in first[m:i]:
                assert mixed[i] == first[i]
                shared += first[i] in first[:m]
        assert (-1 - mixed[:m] == mix_ref.draw(step, 0, m, T, 0, on)).all()
    assert shared > 0
