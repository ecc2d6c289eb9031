"""GPU: network resets and shrink-and-perturb (b200sac_reset, SacCore.reset, the learners' reset_interval): a fresh draw is
create's draw bit for bit, partial resets touch exactly their tensors and optimizers, the blend is the fp64 formula of
include/b200sac.h, the call is stream ordered, bad arguments change nothing, and the learners' schedule is the hand-driven
sequence."""
import ctypes as C
import dataclasses
import itertools
import json
import os

import numpy as np
import pytest
import torch

import redis_stub
from _harness import (ADAM_M, ADAM_V, CARE_PLANS, LL_CFG, PARAMS, SAC_PLANS, _bits, _config, _inputs, _plan, _stream_run,
                      cuda, export)

pytestmark = pytest.mark.gpu

PLANS = list(SAC_PLANS) + list(CARE_PLANS) + ["grad_clip", "pcgrad"]
SEED = 5


def _make(name, R=3, seed=SEED):
    """(core, spec, care) of a SAC_PLANS / CARE_PLANS id, or of "grad_clip" (the LL shape with gradient clipping) or "pcgrad"
    (MTSAC at T = 10 with gradient surgery)."""
    from distributed_sac_b200.core import SacCore
    extra = {"grad_clip": dict(grad_clip=True), "pcgrad": dict(pcgrad=True)}.get(name, {})
    spec, care, precision = _plan({"grad_clip": "chained", "pcgrad": "mtsac_t10"}.get(name, name))
    cfg = dataclasses.replace(_config(spec, care, precision, R), **extra)
    return SacCore(cfg, 0, seed=seed), spec, care


def _step(core, spec, care, i):
    b, e1, e2 = _inputs(spec, care, core.cfg.replicas, i)
    core.step(*b, e1, e2)


def _state(core, r):
    """(params, m, v) of replica r as uint32 bit patterns, and its step counters."""
    return ([_bits(export(core, r))] + [_bits(core.export_arena(w, r).numpy()) for w in (ADAM_M, ADAM_V)],
            core.get_steps(r))


def _assert_state_equal(a, b, what):
    (xa, sa), (xb, sb) = a, b
    for name, u, v in zip(("params", "Adam m", "Adam v"), xa, xb):
        bad = np.flatnonzero(u != v)
        assert bad.size == 0, f"{what}: {name} differs at {bad.size} floats, first [{bad[0]}]"
    assert sa == sb, f"{what}: step counters {sa} != {sb}"


def _spans(core, pred):
    """Float ranges [(name, lo, hi)] of the layout tensors whose name satisfies pred."""
    return [(n, d[0], d[0] + d[1] * d[5]) for n, d in core.table.items() if pred(n)]


@pytest.mark.parametrize("name", PLANS)
def test_full_reset_with_the_create_seed_is_a_fresh_handle(cuda, name):
    a, spec, care = _make(name)
    twin, _, _ = _make(name)
    for i in range(3):
        for c in (a, twin):
            _step(c, spec, care, i)
    a.reset(SEED, replica=1)
    fresh, _, _ = _make(name)
    _assert_state_equal(_state(a, 1), _state(fresh, 1), f"{name}: replica 1 after a full reset")
    for r in (0, 2):
        _assert_state_equal(_state(a, r), _state(twin, r), f"{name}: replica {r} (not reset)")
    if name == "pcgrad":       # the surgery's permutations follow the step index, which a reset keeps: plain task sums
        for c in (a, fresh):
            c.set_pcgrad(critic=False, actor=False)
    for i in range(10, 13):
        for c in (a, fresh):
            _step(c, spec, care, i)
    la, lf = a.read_losses(3)[:, 1].numpy(), fresh.read_losses(3)[:, 1].numpy()
    assert np.array_equal(_bits(la), _bits(lf)), f"{name}: losses after the reset {la} != fresh {lf}"
    (xa, _), (xf, _) = _state(a, 1), _state(fresh, 1)
    for u, v in zip(xa, xf):
        assert np.array_equal(u, v), f"{name}: arenas differ from the fresh handle's three steps later"


@pytest.mark.parametrize("name", PLANS)
def test_partial_depth_touches_its_tensors_and_optimizers_only(cuda, name):
    core, spec, care = _make(name, R=2)
    for i in range(2):
        _step(core, spec, care, i)
    before = [_state(core, r) for r in range(2)]
    core.reset(SEED, replica=0, actor=1, critic=2)
    fresh, _, _ = _make(name, R=2)
    La, Lc = len(core.cfg.actor_hidden), len(core.cfg.critic_hidden)
    heads = {f"actor.{La}."} | {f"q{k}{t}.{j}." for k in (1, 2) for t in ("", "_target") for j in (Lc, Lc - 1) if j >= 0}
    touched = lambda n: any(n.startswith(h) for h in heads)
    (p, m, v), steps = _state(core, 0)
    fp = _bits(export(fresh, 0))
    for n, lo, hi in _spans(core, touched):
        assert np.array_equal(p[lo:hi], fp[lo:hi]), f"{name}: {n} is not the fresh draw"
    for n, lo, hi in _spans(core, lambda n: not touched(n)):
        assert np.array_equal(p[lo:hi], before[0][0][0][lo:hi]), f"{name}: untouched {n} changed"
    slot_of_opt = {0: 0, 1: 1, 2: 2, 3: 4}
    for n, d in core.table.items():
        if not d[3]:
            continue
        lo, hi = d[0], d[0] + d[1] * d[5]
        reset = slot_of_opt[d[4]] in (0, 1)
        for name_mv, got, old in (("m", m, before[0][0][1]), ("v", v, before[0][0][2])):
            want = np.zeros(hi - lo, np.uint32) if reset else old[lo:hi]
            assert np.array_equal(got[lo:hi], want), f"{name}: Adam {name_mv} of {n} (optimizer {d[4]})"
    old = before[0][1]
    assert steps[:2] == (0, 0) and steps[2:] == old[2:], f"{name}: counters {steps} (before {old})"
    _assert_state_equal(_state(core, 1), before[1], f"{name}: replica 1")


@pytest.mark.parametrize("lam", [0.5, 0.8, 1.0])
@pytest.mark.parametrize("name", PLANS)
def test_shrink_and_perturb_is_the_fp64_blend(cuda, name, lam):
    core, spec, care = _make(name, R=2)
    for i in range(2):
        _step(core, spec, care, i)
    x = export(core, 1).astype(np.float64)
    core.reset(SEED, replica=1, shrink=lam)
    th0 = export(_make(name, R=2)[0], 1).astype(np.float64)     # a fresh handle's targets equal its locals
    want = (lam * x + (1.0 - lam) * th0).astype(np.float32)
    if care:
        lo, hi = _spans(core, lambda n: n == "embedding")[0][1:]
        want[lo:hi] = x[lo:hi]
    got = export(core, 1)
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert bad.size == 0, f"{name}, shrink {lam}: {bad.size} floats differ, first [{bad[0]}] {got[bad[0]]!r} != {want[bad[0]]!r}"
    assert not core.export_arena(ADAM_M, 1).any() and not core.export_arena(ADAM_V, 1).any()
    assert core.get_steps(1)[:3] == (0, 0, 0)


@pytest.mark.parametrize("name", ["chained", "care_o"])
def test_fresh_draw_recovers_a_non_finite_network(cuda, name):
    core, spec, care = _make(name, R=1)
    p = export(core, 0)
    for n, (off, rows, cols, _t, _o, pitch) in core.table.items():      # tensor elements only: pads and gaps stay zero
        if n != "embedding":
            x = p[off:off + rows * pitch].reshape(rows, pitch)[:, :cols].reshape(-1)
            x[::7], x[3::11] = np.nan, np.inf
            p[off:off + rows * pitch].reshape(rows, pitch)[:, :cols] = x.reshape(rows, cols)
    core.import_arena(torch.from_numpy(p), PARAMS, 0)
    core.reset(SEED, shrink=0.0)
    got = export(core, 0)
    fresh = export(_make(name, R=1)[0], 0)
    if care:           # the frozen embedding is not part of any reset
        lo, hi = _spans(core, lambda n: n == "embedding")[0][1:]
        got[lo:hi] = fresh[lo:hi]
    assert np.isfinite(got).all() and np.array_equal(_bits(got), _bits(fresh))


@pytest.mark.parametrize("mode", ["stream", "legacy", "host"])
def test_reset_is_stream_ordered(cuda, mode):
    change = lambda core: core.reset(31, replica=1, shrink={"critic": 0.5, "actor": 0.25, "alpha": 0.0})

    def result(core):
        return [x for r in range(2) for x in _state(core, r)[0]] + [core.read_losses(16).numpy()]
    fast = _stream_run(mode, change, False, result)
    synced = _stream_run(mode, change, True, result)
    plain = _stream_run(mode, None, False, result)
    for u, v in zip(fast, synced):
        assert np.array_equal(u.view(np.uint32), v.view(np.uint32)), f"{mode}: the unsynchronised reset differs"
    assert np.array_equal(fast[0], plain[0]) and not np.array_equal(fast[3], plain[3])   # replica 0 kept, replica 1 reset


def test_bad_arguments_change_nothing(cuda):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import _stream
    core, spec, care = _make("care_m", R=2)
    _step(core, spec, care, 0)
    before = [_state(core, r) for r in range(2)]

    def spec_with(part, layers=1, shrink=0.0):
        s = _lib.ResetSpec()
        s.part[part].layers, s.part[part].shrink = layers, shrink
        return s
    A, Cr, Al, E, X = range(5)
    bad = [(0, spec_with(A, -1)), (0, spec_with(Cr, -3)), (0, spec_with(Al, 2)), (0, spec_with(E, 2)),
           (0, spec_with(A, 1, float("nan"))), (0, spec_with(Cr, 1, 1.5)), (0, spec_with(Al, 1, -0.5)),
           (0, spec_with(X)), (2, spec_with(A)), (-1, spec_with(A)), (0, None)]
    for r, s in bad:
        rc = core.lib.b200sac_reset(core._h, r, None if s is None else C.byref(s), C.c_uint64(SEED), _stream())
        assert rc == -1, f"replica {r}: rc {rc}"
    plain, pspec, pcare = _make("chained", R=1)
    rc = plain.lib.b200sac_reset(plain._h, 0, C.byref(spec_with(E)), C.c_uint64(SEED), _stream())
    assert rc == -1
    torch.cuda.synchronize()
    for r in range(2):
        _assert_state_equal(_state(core, r), before[r], f"replica {r} after refused resets")


# ---- learners ---------------------------------------------------------------------------------------------------------
_SERVERS = itertools.count()


def _ll(tmp_path, **kw):
    from distributed_sac_b200.learner import Learner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(LL_CFG))
    os.chdir(tmp_path)
    lrn = Learner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=f"{tmp_path}/{next(_SERVERS)}"), seed=3,
                  replay_where="device", **kw)
    lrn.memory.ring.fill_synthetic(20000, seed=1)
    return lrn


def _hand(lrn, n, one):
    """n updates of a learner without a schedule, with the resets of reset_interval=5 enqueued by hand."""
    for i in range(n):
        if i and i % 5 == 0:
            lrn.core.reset(lrn.seed + (i // 5) * 2 ** 32)
        one()


def _same_learners(a, b, what):
    _assert_state_equal(_state(a.core, 0), _state(b.core, 0), what)


def test_learner_update_schedule(cuda, tmp_path):
    a, b = _ll(tmp_path, reset_interval=5), _ll(tmp_path)
    la = [a.update() for _ in range(12)]
    lb = []
    _hand(b, 12, lambda: lb.append(b.update()))
    assert la == lb
    _same_learners(a, b, "update() x 12")
    assert a.core.get_steps() == (2, 2, 2)
    path = a.save_checkpoint(12)
    c = _ll(tmp_path, checkpoint_path=path)
    _same_learners(a, c, "checkpoint saved after a reset, loaded")
    for x in (a, b, c):
        x.memory.stop()


def test_learner_update_many_and_update_sac_schedule(cuda, tmp_path):
    a, b = _ll(tmp_path, reset_interval=5), _ll(tmp_path)
    la = a.update_many(12)
    for n, k in ((5, 1), (5, 2), (2, None)):
        b.core.step_sampled(b.memory.ring, n)
        if k:
            b.core.reset(b.seed + k * 2 ** 32)
    lb = b.core.read_losses(12)[:, 0][:, [0, 1]]
    assert torch.equal(la, lb)
    _same_learners(a, b, "update_many(12)")
    batch = [a.memory.sample() for _ in range(12)]
    g = torch.Generator().manual_seed(0)
    eps = [(torch.randn(256, 2, generator=g).cuda(), torch.randn(256, 2, generator=g).cuda()) for _ in range(12)]
    la = [a.update_SAC(*batch[i], None, eps_next=eps[i][0], eps_cur=eps[i][1]) for i in range(12)]   # updates 13..24
    lb = []
    for i in range(12):
        if (12 + i) % 5 == 0:
            b.core.reset(b.seed + ((12 + i) // 5) * 2 ** 32)
        lb.append(b.update_SAC(*batch[i], None, eps_next=eps[i][0], eps_cur=eps[i][1]))
    assert la == lb
    _same_learners(a, b, "update_SAC after update_many")
    for x in (a, b):
        x.memory.stop()


def test_learner_run_schedule_and_published_actor(cuda, tmp_path):
    a, b = _ll(tmp_path, reset_interval=5), _ll(tmp_path)
    assert a.run(max_updates=12) == 12
    b.soft_update(None, None, 1.0)
    _hand(b, 12, b.update)
    _same_learners(a, b, "run(max_updates=12)")
    # get_parameters() after a reset carries the new actor: a reset with the learner's own seed restores the created actor
    created = _ll(tmp_path)
    a.reset_networks(seed=a.seed, actor="all")
    pub = a.get_parameters()["actor"]
    want = created._module_state_dict("actor")
    assert set(pub) == set(want) and all(torch.equal(pub[k], want[k]) for k in want)
    for x in (a, b, created):
        x.memory.stop()
