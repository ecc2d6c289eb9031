"""GPU: per-replica actor and target update intervals (b200sac_get/set_update_intervals).

With n the critic's Adam step count after a step, the step updates the actor and the temperature iff n % actor_every == 0
and the targets iff n % target_every == 0.  Checked here: every plan follows the restore-based oracle (a full reference
update, then the actor side and / or the targets put back) at the 1e-4 bar; what a skipped update leaves alone stays bit
for bit; replicas with different intervals equal uniform handles; every step path and a change between graph launches
follow the schedule in stream order; prioritized replay keeps rewriting priorities; bad values are rejected; the learner
surface reports NaN actor losses on critic-only steps and keeps the phase across a checkpoint."""
import json
import math
import os

import pytest
import torch

import care_port as cp
import redis_stub
import sac_port as sp
from _golden import REL, check_forced, check_port_state, core_config, cuda_relu_masks, rel_scalar, sync_core_to_port
from _harness import LL_CFG, SMALL, _config, _inputs, _plan, _stream_run, cuda

pytestmark = pytest.mark.gpu

PARAMS, ADAM_M, ADAM_V = 0, 1, 2
PLANS = ["chained", "per_layer", "mtsac_weighted", "care_m", "care_o"]


def _inputs_iv(spec, care, R, i):
    return _inputs(spec, care, R, i, noise_seed=2000, batch_seed=7)


def _is_actor(name):
    return name.startswith("actor.") or name == "log_alpha"


def _is_target(name):
    return "_target" in name or name.startswith("tse.")


def _state(core, r=0):
    return {w: core.get_named(w, r) for w in (PARAMS, ADAM_M, ADAM_V)}, core.get_steps(r)


def _kinds(n, ae, te):
    return n % ae == 0, n % te == 0


# ---- 1. oracle parity ------------------------------------------------------------------------------------------------
def _oracle_step(core, port, spec, care, b, e1, e2, actor, target):
    """One CUDA step and one restore-based oracle step with the CUDA ReLU masks forced; returns the oracle's losses."""
    sync_core_to_port(core, port)
    core.step(*[t.unsqueeze(0) for t in b], e1.unsqueeze(0), e2.unsqueeze(0))
    forced = cuda_relu_masks(core, spec, 0, care)
    if not actor:       # the actor pass did not run: its activations are stale, the oracle's own are restored away below
        forced = {k: v for k, v in forced.items() if ":pi" not in k}
    keep_p = {k: v.detach().clone() for k, v in port.p.items() if (not actor and _is_actor(k)) or (not target and _is_target(k))}
    # (per-parameter copies: a deepcopy of the state dict would also copy its keys, the parameters themselves)
    keep_opt = {o: {q: {k: v.clone() for k, v in st.items()} for q, st in o.state.items()} for o in (port.opt_actor, port.opt_alpha)}
    with sp.ReluTape(forced) as tape:
        out = (port.update if care else port.update_SAC)(*b, e1, e2)
    check_forced(tape, forced)
    with torch.no_grad():
        for k, v in keep_p.items():
            port.p[k].copy_(v)
    if not actor:
        for o, st in keep_opt.items():
            o.state.clear()
            o.state.update(st)
    return out


@pytest.mark.parametrize("plan", PLANS)
def test_intervals_match_restore_oracle(cuda, plan):
    """actor_every = 2, target_every = 3 over 6 steps from critic count 7: all four step kinds.  Each step matches the
    oracle (full update, then actor side / targets restored) at 1e-4; the critic loss matches and the actor-side losses
    are NaN exactly on critic-only steps."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(plan)
    mod = cp if care else sp
    port = (cp.CarePortLearner if care else sp.PortLearner)(spec, mod.init_params(spec, seed=3))
    st = port.adam_state()
    st["step"] = (7, 4, 4) + tuple(st["step"][3:])
    port.load_adam(st)
    core = SacCore(_config(spec, care, precision), 0, seed=0)
    core.set_update_intervals(2, 3)
    assert core.get_update_intervals() == (2, 3)
    gen = torch.Generator().manual_seed(5)
    seen = set()
    for i in range(6):
        n = 8 + i
        actor, target = _kinds(n, 2, 3)
        seen.add((actor, target))
        b = mod.synthetic_batch(spec, seed=60 + i)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen)
        o = _oracle_step(core, port, spec, care, b, e1, e2, actor, target)
        L = core.read_losses(1)[0, 0]
        assert rel_scalar(float(L[0]), o["critic_loss"]) <= REL, (i, float(L[0]), o["critic_loss"])
        if actor:
            assert rel_scalar(float(L[1]), o["actor_loss"]) <= REL, (i, float(L[1]), o["actor_loss"])
            assert not any(math.isnan(float(x)) for x in L)
        else:
            assert all(math.isnan(float(x)) for x in L[1:]), (i, L)
        check_port_state(core, port)
        assert core.get_steps()[:3] == port.adam_state()["step"][:3] == (n, 4 + n // 2 - 3, 4 + n // 2 - 3)
    assert len(seen) == 4
    core.close()


# ---- 2. exactness ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", PLANS)
def test_skipped_updates_leave_state_bit_identical(cuda, plan):
    """On critic-only steps the actor, log_alpha, their m / v and counters are torch.equal to before; on non-target steps
    the targets are; on actor / target steps they change.  The critics change on every step."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(plan)
    core = SacCore(_config(spec, care, precision), 0, seed=1)
    core.set_named((cp if care else sp).init_params(spec, seed=4))
    core.set_steps((7, 4, 4))
    core.set_update_intervals(2, 3)
    for i in range(6):
        before, sb = _state(core)
        b, e1, e2 = _inputs_iv(spec, care, 1, i)
        core.step(*b, e1, e2)
        after, sa = _state(core)
        actor, target = _kinds(sb[0] + 1, 2, 3)
        assert sa[0] == sb[0] + 1 and sa[1:3] == tuple(x + (1 if actor else 0) for x in sb[1:3])
        if len(sa) > 3:
            assert sa[3] == sb[3] + 1          # the CARE(O) context encoder steps with the critic loss
        for which, named in after.items():
            for k, v in named.items():
                old = before[which][k]
                if _is_actor(k):
                    assert torch.equal(v, old) != actor, (i, which, k, actor)
                elif _is_target(k) and which == PARAMS:
                    assert torch.equal(v, old) != target, (i, k, target)
        assert not torch.equal(after[PARAMS]["q1.0.weight"], before[PARAMS]["q1.0.weight"])
    core.close()


# ---- 3. mixed replicas -----------------------------------------------------------------------------------------------
ROWS = [(1, 1), (2, 1), (4, 3)]


@pytest.mark.parametrize("plan", PLANS)
def test_mixed_replicas_equal_uniform_handles(cuda, plan):
    """R = 3 with rows (1,1), (2,1), (4,3) == three uniform R = 3 handles, bit for bit: parameters, moments, losses,
    counters."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(plan)
    R = len(ROWS)
    params = (cp if care else sp).init_params(spec, seed=3)
    mixed = SacCore(_config(spec, care, precision, R), 0, seed=0)
    for r, (a, t) in enumerate(ROWS):
        mixed.set_update_intervals(a, t, replica=r)
    uniform = [SacCore(_config(spec, care, precision, R), 0, seed=0) for _ in ROWS]
    for u, (a, t) in zip(uniform, ROWS):
        u.set_update_intervals(a, t)
    for core in [mixed] + uniform:
        for r in range(R):
            core.set_named(params, replica=r)
    n = 6
    for i in range(n):
        b, e1, e2 = _inputs_iv(spec, care, R, i)
        for core in [mixed] + uniform:
            core.step(*b, e1, e2)
    Lm = mixed.read_losses(n)
    for r, uni in enumerate(uniform):
        for which in (PARAMS, ADAM_M, ADAM_V):
            assert torch.equal(mixed.export_arena(which, r), uni.export_arena(which, r)), (plan, r, which)
        assert torch.equal(Lm[:, r].nan_to_num(7.0), uni.read_losses(n)[:, r].nan_to_num(7.0)), (plan, r)
        assert mixed.get_steps(r) == uni.get_steps(r)
    assert [mixed.get_steps(r)[:3] for r in range(R)] == [(6, 6, 6), (6, 3, 3), (6, 1, 1)]
    assert [int(Lm[:, r, 1].isnan().sum()) for r in range(R)] == [0, 3, 5]
    for core in [mixed] + uniform:
        core.close()


# ---- 4. paths and stream order ---------------------------------------------------------------------------------------
def test_multi_step_graphs_equal_single_steps(cuda):
    """One step_sampled(ring, 13) call (8/4/2/1-step graphs) == 13 single calls, bit for bit."""
    from distributed_sac_b200.core import Replay, SacCore
    out = []
    for split in (False, True):
        core = SacCore(core_config(SMALL, replicas=2), 0, seed=5)
        core.set_update_intervals(2, 3, replica=0)
        core.set_update_intervals(3, 2, replica=1)
        rb = Replay(core, 4096, seed=6)
        rb.fill_synthetic(4096, seed=8)
        if split:
            for _ in range(13):
                core.step_sampled(rb, 1)
        else:
            core.step_sampled(rb, 13)
        out.append(([core.export_arena(w, r) for w in (PARAMS, ADAM_M, ADAM_V) for r in range(2)], core.read_losses(13),
                     [core.get_steps(r) for r in range(2)]))
        rb.close()
        core.close()
    (a0, l0, s0), (a1, l1, s1) = out
    assert all(torch.equal(x, y) for x, y in zip(a0, a1))
    assert torch.equal(l0.nan_to_num(7.0), l1.nan_to_num(7.0))
    assert s0 == s1 == [(13, 6, 6), (13, 4, 4)]


def test_step_entry_points_follow_the_schedule(cuda):
    """b200sac_step and b200sac_step_host compute the same thing; both and b200sac_update report NaN actor-side losses on
    exactly the critic-only steps."""
    from distributed_sac_b200.core import Replay, SacCore
    dev, host = (SacCore(core_config(SMALL), 0, seed=2) for _ in range(2))
    for c in (dev, host):
        c.set_update_intervals(2, 1)
    for i in range(4):
        b, e1, e2 = _inputs_iv(SMALL, False, 1, i)
        dev.step(*b, e1, e2)
        Lh = host.step_host(*b, e1, e2)
        Ld = dev.read_losses(1)[0]
        assert torch.equal(Ld.nan_to_num(7.0), Lh.nan_to_num(7.0))
        assert bool(Lh[0, 1].isnan()) == (i % 2 == 0) and not bool(Lh[0, 0].isnan())
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(dev.export_arena(w), host.export_arena(w))
    assert dev.get_steps() == host.get_steps() == (4, 2, 2)
    rb = Replay(dev, 4096, seed=3)
    rb.fill_synthetic(4096, seed=4)
    for i in range(4):
        cl, al, _alpha_loss, ent = dev.update_sampled(rb)
        assert cl == cl and (al != al) == (ent != ent) == (i % 2 == 0)
    rb.close()
    dev.close()
    host.close()


def _read(core):
    return core.read_losses(16).nan_to_num(7.0), core.export_arena(0, 0), core.export_arena(1, 1), core.get_steps(1)


def _set_iv(core):
    core.set_update_intervals(2, 3)


@pytest.mark.parametrize("mode", ["stream", "legacy", "host"])
def test_set_update_intervals_is_stream_ordered(cuda, mode):
    """A change enqueued right behind a graph launch (after prepare) lands exactly between the steps before and after it:
    the same as setting it on an idle device.  On a side stream, on the legacy default stream and with a pinned-host ring."""
    lx, ax, mx, sx = _stream_run(mode, _set_iv, False, _read)
    ly, ay, my, sy = _stream_run(mode, _set_iv, True, _read)
    lz, _, _, sz = _stream_run(mode, None, False, _read)
    assert torch.equal(lx, ly) and torch.equal(ax, ay) and torch.equal(mx, my) and sx == sy
    assert torch.equal(lx[:8], lz[:8])
    assert (lx[8:, :, 1] == 7.0).sum() == 2 * 4 and (lz[:, :, 1] == 7.0).sum() == 0
    assert sx == (16, 12, 12) and sz == (16, 16, 16)


# ---- 5. prioritized replay -------------------------------------------------------------------------------------------
def test_prioritized_ring_updates_priorities_on_critic_only_steps(cuda):
    """actor_every = 2 on a prioritized ring: the priorities of every step's minibatch are rewritten in the step, critic-only
    steps included, and the importance weights stay finite."""
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(SMALL), 0, seed=4)
    core.set_update_intervals(2, 1)
    rb = Replay(core, 4096, seed=1, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6))
    rb.fill_synthetic(4096, seed=2)
    for i in range(4):
        actor_before = core.get_named()["actor.0.weight"]
        core.step_sampled(rb, 1)
        idx, prio, w = core.debug("idx").long(), core.debug("prio"), core.debug("isw")
        assert torch.isfinite(w).all() and (w > 0).all()
        assert torch.isfinite(prio).all() and (prio > 0).all()
        uniq, cnt = torch.unique(idx, return_counts=True)
        once = torch.isin(idx, uniq[cnt == 1])                         # (a slot drawn twice keeps one of its two values)
        assert once.sum() > 0
        got = torch.from_numpy(rb.priorities(idx[once].numpy()))
        assert torch.equal(got, prio[once])
        assert torch.equal(core.get_named()["actor.0.weight"], actor_before) == (i % 2 == 0)
    rb.close()
    core.close()


# ---- 6. rejection and copy_replica -----------------------------------------------------------------------------------
def test_bad_intervals_are_rejected_and_copy_keeps_them(cuda):
    from distributed_sac_b200.core import SacCore
    core, fresh = SacCore(core_config(SMALL, replicas=2), 0, seed=1), SacCore(core_config(SMALL, replicas=2), 0, seed=1)
    core.set_update_intervals(3, 2, replica=1)
    for a, t in [(0, 1), (1, 0), (-1, 1), (1, -5), (2 ** 30 + 1, 1), (1, 2 ** 31 - 1)]:
        for replica in (0, None):
            with pytest.raises(RuntimeError):
                core.set_update_intervals(a, t, replica=replica)
    for replica in (2, -1):
        with pytest.raises(RuntimeError):
            core.set_update_intervals(1, 1, replica=replica)
        with pytest.raises(RuntimeError):
            core.get_update_intervals(replica)
    assert core.get_update_intervals(0) == (1, 1) and core.get_update_intervals(1) == (3, 2)
    core.set_update_intervals(2 ** 30, 2 ** 30, replica=1)                 # the largest accepted value
    core.set_update_intervals(3, 2, replica=1)
    b, e1, e2 = _inputs_iv(SMALL, False, 2, 0)
    fresh.set_update_intervals(3, 2, replica=1)
    for c in (core, fresh):
        c.step(*b, e1, e2)
    for w in (PARAMS, ADAM_M, ADAM_V):
        for r in range(2):
            assert torch.equal(core.export_arena(w, r), fresh.export_arena(w, r))
    # copy_replica: the counters (and with them the phase) are copied, the intervals are not
    core.set_steps((5, 1, 1), replica=1)
    core.copy_replica(1, 0)
    assert core.get_steps(0) == (5, 1, 1) and core.get_update_intervals(0) == (1, 1)
    core.set_update_intervals(3, 2, replica=0)
    b, e1, e2 = _inputs_iv(SMALL, False, 2, 1)
    for t in b + [e1, e2]:
        t[0] = t[1]
    core.step(*b, e1, e2)                                # n = 6: an actor step and a target step for both
    assert core.get_steps(0) == core.get_steps(1) == (6, 2, 2)
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(core.export_arena(w, 0), core.export_arena(w, 1))
    core.close()
    fresh.close()


# ---- 7. learner surface ----------------------------------------------------------------------------------------------

def test_learner_update_intervals_and_checkpoint(cuda, tmp_path):
    """LunarLanderLearner(actor_update_interval=3, target_update_interval=2): update() returns NaN actor loss on critic-only
    steps; a save / load round trip keeps the actor optimizer's step below the critic's, and the next actor step comes at
    the same critic count."""
    from distributed_sac_b200.learner import Learner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(LL_CFG))
    os.chdir(tmp_path)
    mk = lambda tag, ck=None: Learner(str(p), write_mode=False, checkpoint_path=ck, seed=3, actor_update_interval=3,
                                      target_update_interval=2, server=redis_stub.StrictRedis(host=str(tmp_path) + tag))
    lrn = mk("a")
    assert lrn.core.get_update_intervals() == (3, 2)
    lrn.memory.ring.fill_synthetic(20000, seed=1)
    for n in range(1, 5):
        cl, al = lrn.update()
        assert cl == cl and (al != al) == (n % 3 != 0), (n, al)
    assert lrn.core.get_steps() == (4, 1, 1)
    path = lrn.save_checkpoint(4)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert int(ck["critic_optimizer"]["state"][0]["step"]) == 4 and int(ck["actor_optimizer"]["state"][0]["step"]) == 1
    lrn.memory.stop()
    lrn2 = mk("b", path)
    assert lrn2.core.get_steps() == (4, 1, 1)
    lrn2.memory.ring.fill_synthetic(20000, seed=1)
    got = [lrn2.update()[1] for _ in range(3)]          # critic counts 5, 6, 7: the actor steps at 6
    assert [a != a for a in got] == [True, False, True]
    assert lrn2.core.get_steps() == (7, 2, 2)
    lrn2.memory.stop()
