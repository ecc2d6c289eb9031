"""GPU: dormant-neuron recycling (b200sac_redo, SacCore.redo / read_redo, the learners' redo_interval): the record's scores
against fp64 numpy over the device's own activations and against the autograd oracle's forward, forced-dead neurons
recycled exactly as redo_ref restates it, the network's function kept, measure-only and recycle-all thresholds, stream
order, refused calls, and the learners' schedule against recycles driven by hand."""
import ctypes as C
import dataclasses
import itertools
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import care_port as cp
import redis_stub
import redo_ref as rr
import sac_port as sp
from _harness import (ADAM_M, ADAM_V, CARE_ROW_OUTPUTS, LL_CFG, PARAMS, ROW_OUTPUTS, SMALL, _bits, _config, _inputs, _plan,
                      _stream_run, _tasks, check_losses, check_port_state, check_rows, cuda, export, kink_checked_step)

pytestmark = pytest.mark.gpu

PLANS = ["chained", "vs400_fp32", "vs400_tc", "care_m", "care_o", "grad_clip", "pcgrad"]
SEED, RSEED = 5, 77
# the step's outputs that depend on the state before the step alone (qmin is min(Q1, Q2)(s, a~) of the critic after the
# step's own Adam update, whose moments the recycle zeroed)
FORWARD = ("q1", "q2", "y", "a_next", "a_cur", "logp_next", "logp_cur")


def _make(name, R, seed=SEED):
    """(core, spec, care, precision) of a SAC_PLANS / CARE_PLANS id, or of "grad_clip" (the LL shape with gradient
    clipping) or "pcgrad" (MTSAC at T = 10 with gradient surgery)."""
    from distributed_sac_b200.core import SacCore
    extra = {"grad_clip": dict(grad_clip=True), "pcgrad": dict(pcgrad=True)}.get(name, {})
    spec, care, precision = _plan({"grad_clip": "chained", "pcgrad": "mtsac_t10"}.get(name, name))
    cfg = dataclasses.replace(_config(spec, care, precision, R), **extra)
    return SacCore(cfg, 0, seed=seed), spec, care, precision


def _stepped(name, R, n_steps=2):
    core, spec, care, precision = _make(name, R)
    for i in range(n_steps):
        b, e1, e2 = _inputs(spec, care, R, i)
        core.step(*b, e1, e2)
    return core, spec, care, precision


def _rows(spec, care, n, seed=4242):
    s, a = (cp if care else sp).synthetic_batch(spec, seed=seed)[:2]
    return s[:n].contiguous(), a[:n].contiguous()


def _state(core, r):
    return [_bits(export(core, r))] + [_bits(core.export_arena(w, r).numpy()) for w in (ADAM_M, ADAM_V)], core.get_steps(r)


def _assert_state_equal(a, b, what):
    (xa, sa), (xb, sb) = a, b
    for name, u, v in zip(("params", "Adam m", "Adam v"), xa, xb):
        bad = np.flatnonzero(u != v)
        assert bad.size == 0, f"{what}: {name} differs at {bad.size} floats, first [{bad[0]}]"
    assert sa == sb, f"{what}: step counters {sa} != {sb}"


def _widths(core):
    return {"actor": list(core.cfg.actor_hidden), "q1": list(core.cfg.critic_hidden), "q2": list(core.cfg.critic_hidden)}


def _device_hidden(core, n, r):
    """{net: [rows [0, n) of each hidden layer]} as the call's forward left them in hA / hQ."""
    B, out = core.cfg.batch, {}
    out["actor"] = [core.debug(f"hA.{l}", r).reshape(2 * B, H)[:n].double().numpy()
                    for l, H in enumerate(core.cfg.actor_hidden)]
    for k, net in enumerate(("q1", "q2")):
        out[net] = [core.debug(f"hQ.{l}", r).reshape(2, B, H)[k, :n].double().numpy()
                    for l, H in enumerate(core.cfg.critic_hidden)]
    return out


def _oracle_hidden(core, spec, care, obs, act, r):
    """The autograd oracle's hidden activations in fp64 from replica r's exported parameters (CARE: the critic's state
    encoder on the task's context code first)."""
    p = {k: v.double() for k, v in core.get_named(PARAMS, r).items()}
    x = obs.double()
    if care:
        z = cp.context_encode(spec, p, torch.as_tensor(_tasks(spec, obs)))
        x = cp.state_encode(spec, p, "cse", z, x)
    xq = torch.cat([x, act.double()], 1)
    out = {}
    for net, h in (("actor", x), ("q1", xq), ("q2", xq)):
        out[net] = []
        for l in range(len(_widths(core)[net])):
            h = torch.relu(F.linear(h, p[f"{net}.{l}.weight"], p[f"{net}.{l}.bias"]))
            out[net].append(h.detach().numpy())
    return out


# ---- 1: the record -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("name", PLANS)
def test_scores_match_fp64_numpy_and_the_oracle_forward(cuda, name, R):
    core, spec, care, _ = _stepped(name, R)
    rec0 = core.read_redo(R - 1)
    assert all(np.isnan(s).all() for net in rec0.values() for s in net["score"])
    assert not any(d.any() for net in rec0.values() for d in net["dormant"])
    n = spec.batch - 3
    obs, act = _rows(spec, care, n)
    before = [_state(core, r) for r in range(R)]
    core.redo(RSEED, obs, act)                               # measure only
    for r in range(R):
        _assert_state_equal(_state(core, r), before[r], f"{name}: replica {r} after a measure-only call")
        rec, dev, ref = core.read_redo(r), _device_hidden(core, n, r), _oracle_hidden(core, spec, care, obs, act, r)
        for net in rr.NETS:
            for l in range(len(_widths(core)[net])):
                got = rec[net]["score"][l]
                assert not rec[net]["dormant"][l].any()
                np.testing.assert_allclose(got, rr.scores(dev[net][l]), rtol=1e-12, atol=1e-12,
                                           err_msg=f"{name} R={R} replica {r} {net}.{l}: record vs the device's activations")
                np.testing.assert_allclose(dev[net][l], ref[net][l], rtol=1e-5, atol=1e-5 * np.abs(ref[net][l]).max(),
                                           err_msg=f"{name} replica {r} {net}.{l}: activations vs the oracle forward")
                want = rr.scores(ref[net][l])
                np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * np.abs(want).max(),
                                           err_msg=f"{name} replica {r} {net}.{l}: record vs the oracle forward")


# ---- 2 and 3: forced-dead neurons, recycled; the function kept ----------------------------------------------------------
def _kill(core, r, rng):
    """Bias -1e3 on 3 + r random neurons of every hidden layer of replica r; returns {net: [bool masks]}."""
    p = export(core, r)
    masks = {}
    for net, widths in _widths(core).items():
        masks[net] = []
        for l, H in enumerate(widths):
            idx = rng.choice(H, size=min(H, 3 + r), replace=False)
            p[core.table[f"{net}.{l}.bias"][0] + idx] = -1e3
            m = np.zeros(H, bool)
            m[idx] = True
            masks[net].append(m)
    core.import_arena(torch.from_numpy(p), PARAMS, r)
    return masks


def _port_of(core, spec, care, r=0):
    named = core.get_named(PARAMS, r)
    st = {"m": core.get_named(ADAM_M, r), "v": core.get_named(ADAM_V, r), "step": core.get_steps(r)}
    return cp.CarePortLearner(spec, named, st) if care else sp.PortLearner(spec, named, st)


@pytest.mark.parametrize("R", [1, 3])
@pytest.mark.parametrize("name", PLANS)
def test_forced_dead_neurons_are_recycled_and_the_function_kept(cuda, name, R):
    from distributed_sac_b200.core import SacCore
    a, spec, care, precision = _stepped(name, R)
    twin, _, _, _ = _stepped(name, R)
    masks = {}
    for r in range(R):
        for c in (a, twin):
            masks[r] = _kill(c, r, np.random.default_rng(100 + r))
    obs, act = _rows(spec, care, spec.batch)
    theta0 = SacCore(a.cfg, 0, seed=RSEED)
    before = [_state(a, r) for r in range(R)]
    launches = a.launches_per_step
    a.redo(RSEED, obs, act, actor=0.0, critic=0.0)          # every replica, each under its own key
    extra = 0
    for r in range(R):
        rec, dev = a.read_redo(r), _device_hidden(a, spec.batch, r)
        for net in rr.NETS:
            for l, m in enumerate(masks[r][net]):
                got = rec[net]["dormant"][l]
                # the forced neurons, and any other neuron that is dead on every one of these rows by itself
                want = rr.dormant(rr.scores(dev[net][l]), 0.0)
                assert np.array_equal(got, want) and not (m & ~got).any(), \
                    f"{name} replica {r} {net}.{l}: flagged {np.flatnonzero(got)}, forced {np.flatnonzero(m)}"
                extra += int((got & ~m).sum())
                masks[r][net][l] = got
        (p, mm, vv), steps = before[r]
        want = rr.recycle(p.view(np.float32), mm.view(np.float32), vv.view(np.float32), a.table, masks[r], export(theta0, r))
        _assert_state_equal(_state(a, r), ([_bits(x) for x in want], steps), f"{name} replica {r}: the recycle")
    forced = sum(int(m.sum()) for r in range(R) for ms in masks[r].values() for m in ms) - extra
    assert extra < forced, f"{name}: {extra} neurons dead by themselves beside {forced} forced ones"
    n = C.c_int32(0)
    assert a.lib.b200sac_launches_per_step(a._h, C.byref(n)) == 0 and n.value == launches

    # one step from the recycled and from the unrecycled state: the same forward outputs.  The step reads the scored rows
    # as s, a and s' (a neuron that is dead on those rows by itself need not be dead on others)
    b, e1, e2 = _inputs(spec, care, R, 7)
    for j, x in ((0, obs), (1, act), (3, obs)):
        b[j][:] = x
    for c in (a, twin):
        c.step(*b, e1, e2)
    for r in range(R):
        for k in FORWARD:
            u, v = a.debug(k, r).numpy(), twin.debug(k, r).numpy()
            if precision == 0:
                assert np.array_equal(_bits(u), _bits(v)), f"{name} replica {r}: {k} changed by the recycle"
            else:
                np.testing.assert_allclose(u, v, rtol=1e-6, atol=1e-6 * np.abs(v).max(),
                                           err_msg=f"{name} replica {r}: {k} changed by the recycle")

    # the step after a recycle against the autograd oracle, started from the recycled arena
    if R == 1 and name != "pcgrad":
        core, _, _, _ = _stepped(name, 1)
        _kill(core, 0, np.random.default_rng(5))
        core.redo(RSEED, obs, act, actor=0.0, critic=0.0)
        port = _port_of(core, spec, care)
        b, e1, e2 = _inputs(spec, care, 1, 9)
        o, _ = kink_checked_step(core, port, spec, [x[0] for x in b], e1[0], e2[0], care=care, want_intermediates=True)
        check_losses(core, o, what=f"{name} after a recycle: ")
        check_port_state(core, port)
        check_rows(core, spec, o, what=f"{name} after a recycle: ", outputs=CARE_ROW_OUTPUTS if care else ROW_OUTPUTS)


# ---- 4: thresholds -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PLANS)
def test_negative_tau_changes_nothing_and_a_huge_tau_recycles_every_neuron(cuda, name):
    from distributed_sac_b200.core import SacCore
    core, spec, care, _ = _stepped(name, 2)
    obs, act = _rows(spec, care, spec.batch // 2)
    before = [_state(core, r) for r in range(2)]
    for ta, tc in ((-1e-9, -0.5), (-math.inf, -math.inf), (-1.0, None)):
        core.redo(RSEED, obs, act, actor=ta, critic=tc)
        for r in range(2):
            _assert_state_equal(_state(core, r), before[r], f"{name}: replica {r} at tau ({ta}, {tc})")
            rec = core.read_redo(r)
            assert all(np.isfinite(s).all() for net in rec.values() for s in net["score"])
            assert not any(d.any() for net in rec.values() for d in net["dormant"])
    core.redo(RSEED, obs, act, actor=1e300, critic=math.inf, replica=0)
    rec = core.read_redo(0)
    masks = {net: rec[net]["dormant"] for net in rr.NETS}
    assert all(m.all() for ms in masks.values() for m in ms)
    theta0 = SacCore(core.cfg, 0, seed=RSEED)
    (p, mm, vv), steps = before[0]
    want = rr.recycle(p.view(np.float32), mm.view(np.float32), vv.view(np.float32), core.table, masks, export(theta0, 0))
    _assert_state_equal(_state(core, 0), ([_bits(x) for x in want], steps), f"{name}: recycle of every hidden neuron")
    _assert_state_equal(_state(core, 1), before[1], f"{name}: replica 1")


# ---- 5: stream order, refusals -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["stream", "legacy", "host"])
def test_redo_is_stream_ordered(cuda, mode):
    obs, act = _rows(SMALL, False, SMALL.batch)
    change = lambda core: core.redo(31, obs, act, actor=0.8, critic=1e30, replica=1)

    def result(core):
        return [x for r in range(2) for x in _state(core, r)[0]] + [core.read_losses(16).numpy()]
    fast = _stream_run(mode, change, False, result)
    synced = _stream_run(mode, change, True, result)
    plain = _stream_run(mode, None, False, result)
    for u, v in zip(fast, synced):
        assert np.array_equal(u.view(np.uint32), v.view(np.uint32)), f"{mode}: the unsynchronised recycle differs"
    assert np.array_equal(fast[0], plain[0]) and not np.array_equal(fast[3], plain[3])   # replica 0 kept, replica 1 recycled


def test_refused_calls_change_nothing(cuda):
    from distributed_sac_b200.core import _ptr, _stream
    core, spec, care, _ = _stepped("care_m", 2)
    obs, act = _rows(spec, care, spec.batch)
    before = [_state(core, r) for r in range(2)]
    B = spec.batch
    bad = [(2, B, obs, act, 0.0, 0.0), (-1, B, obs, act, 0.0, 0.0), (0, 0, obs, act, 0.0, 0.0),
           (0, B + 1, torch.cat([obs, obs[:1]]), torch.cat([act, act[:1]]), 0.0, 0.0),
           (0, B, None, act, 0.0, 0.0), (0, B, obs, None, 0.0, 0.0), (0, B, obs, act, math.nan, 0.0),
           (0, B, obs, act, 0.0, math.nan)]
    for r, n, o, a, ta, tc in bad:
        rc = core.lib.b200sac_redo(core._h, r, n, _ptr(o), _ptr(a), ta, tc, C.c_uint64(RSEED), _stream())
        assert rc == -1, f"replica {r} n {n}: rc {rc}"
    with pytest.raises(RuntimeError):
        core.redo(RSEED, obs[:0], act[:0])
    with pytest.raises(ValueError):
        core.redo(RSEED, obs, act, actor=math.nan)
    torch.cuda.synchronize()
    for r in range(2):
        _assert_state_equal(_state(core, r), before[r], f"replica {r} after refused calls")
        assert all(np.isnan(s).all() for net in core.read_redo(r).values() for s in net["score"])


# ---- 6: learners -------------------------------------------------------------------------------------------------------
_SERVERS = itertools.count()
TAUS = dict(actor=0.6, critic=0.6)


def _ll(tmp_path, **kw):
    from distributed_sac_b200.learner import Learner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(LL_CFG))
    os.chdir(tmp_path)
    lrn = Learner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=f"{tmp_path}/{next(_SERVERS)}"), seed=3,
                  replay_where="device", **kw)
    lrn.memory.ring.fill_synthetic(20000, seed=1)
    return lrn


def _boundary(lrn, u, reset=True):
    """What a learner with reset_interval=5 (actor head) and redo_interval=5 enqueues right before update u + 1."""
    if u and u % 5 == 0:
        if reset:
            lrn.core.reset(lrn.seed + (u // 5) * 2 ** 32, actor=1)
        s, a = lrn.memory.sample()[:2]
        lrn.core.redo(lrn.seed + 2 ** 62 + (u // 5) * 2 ** 32, s, a, **TAUS)


def _same_learners(a, b, what):
    _assert_state_equal(_state(a.core, 0), _state(b.core, 0), what)


def _sched(tmp_path):
    return _ll(tmp_path, reset_interval=5, reset=dict(actor=1), redo_interval=5, redo=TAUS)


def test_learner_update_schedule(cuda, tmp_path):
    a, b = _sched(tmp_path), _ll(tmp_path)
    la = [a.update() for _ in range(12)]
    lb = []
    for u in range(12):
        _boundary(b, u)
        lb.append(b.update())
    assert la == lb
    _same_learners(a, b, "update() x 12")
    rec = a.core.read_redo()
    assert any(d.any() for net in rec.values() for d in net["dormant"]), "no neuron was recycled: the case is vacuous"
    c = _ll(tmp_path)                      # the other order on the boundary gives another state
    for u in range(12):
        if u and u % 5 == 0:
            s, x = c.memory.sample()[:2]
            c.core.redo(c.seed + 2 ** 62 + (u // 5) * 2 ** 32, s, x, **TAUS)
            c.core.reset(c.seed + (u // 5) * 2 ** 32, actor=1)
        c.update()
    assert not np.array_equal(_state(a.core, 0)[0][0], _state(c.core, 0)[0][0])
    for x in (a, b, c):
        x.memory.stop()


def test_learner_update_many_and_update_sac_schedule(cuda, tmp_path):
    a, b = _sched(tmp_path), _ll(tmp_path)
    la = a.update_many(12)
    for n, u in ((5, 5), (5, 10), (2, None)):
        b.core.step_sampled(b.memory.ring, n)
        if u:
            _boundary(b, u)
    lb = b.core.read_losses(12)[:, 0][:, [0, 1]]
    assert torch.equal(la, lb)
    _same_learners(a, b, "update_many(12)")
    batch = [a.memory.sample() for _ in range(12)]
    for _ in range(12):
        b.memory.sample()                  # the same ring draws as a's
    g = torch.Generator().manual_seed(0)
    eps = [(torch.randn(256, 2, generator=g).cuda(), torch.randn(256, 2, generator=g).cuda()) for _ in range(12)]
    la = [a.update_SAC(*batch[i], None, eps_next=eps[i][0], eps_cur=eps[i][1]) for i in range(12)]   # updates 13..24
    lb = []
    for i in range(12):
        _boundary(b, 12 + i)
        lb.append(b.update_SAC(*batch[i], None, eps_next=eps[i][0], eps_cur=eps[i][1]))
    assert la == lb
    _same_learners(a, b, "update_SAC after update_many")
    for x in (a, b):
        x.memory.stop()


def test_learner_run_schedule_and_manual_calls(cuda, tmp_path):
    a, b = _sched(tmp_path), _ll(tmp_path)
    assert a.run(max_updates=12) == 12
    b.soft_update(None, None, 1.0)
    for u in range(12):
        _boundary(b, u)
        b.update()
    _same_learners(a, b, "run(max_updates=12)")
    # by hand: recycle_dormant and a direct SacCore.redo with the seed it documents are one thing
    a.recycle_dormant(critic=1e30)
    s, x = b.memory.sample()[:2]
    b.core.redo(b.seed + 2 ** 63 + 2 ** 62 + 2 ** 32, s, x, critic=1e30)
    _same_learners(a, b, "recycle_dormant")
    before = _state(a.core, 0)
    frac = a.dormant_fraction(0.3)
    _assert_state_equal(_state(a.core, 0), before, "dormant_fraction changed the learner")
    rec = a.core.read_redo()
    assert not any(d.any() for net in rec.values() for d in net["dormant"])
    assert frac == {net: [float(np.mean(s <= 0.3)) for s in rec[net]["score"]] for net in rr.NETS}
    assert all(0.0 <= f <= 1.0 for fs in frac.values() for f in fs) and len(frac["actor"]) == len(a.core.cfg.actor_hidden)
    for x in (a, b):
        x.memory.stop()
