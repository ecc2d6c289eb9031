"""GPU: per-replica hyperparameters (b200sac_get/set_hparams) and the on-device replica copy (b200sac_copy_replica).

A replica's hyperparameters live in a device table read by the step at the replica's index; set_hparams writes a row in
stream order.  Checked here: a handle whose replicas run different values computes, bit for bit, what uniform handles
created with each replica's values compute (every plan); the values mean what the reference means by them (the autograd
oracle given the same values); a change lands exactly between the steps enqueued before and after it, also between
graph launches and through the legacy-default-stream bridge; copy_replica copies the learner state and nothing else;
bad values are rejected without a change."""
import dataclasses
import math

import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import REL, check_port_state, core_config, kink_checked_step, rel_scalar
from _harness import ROWS, SMALL, _config, _inputs, _plan, _stream_run, cuda

pytestmark = pytest.mark.gpu

ARENAS = (0, 1, 2)     # _lib.PARAMS, ADAM_M, ADAM_V


@pytest.mark.parametrize("plan", ["chained", "per_layer", "care_m", "care_o"])
def test_mixed_replicas_equal_uniform_handles(cuda, plan):
    """R = 3 replicas with three different hyperparameter rows == three uniform R = 3 handles created with those rows,
    bit for bit (parameters, Adam moments, losses, step counters).  Same R on both sides: the plan depends on it."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(plan)
    R = len(ROWS)
    params = (cp if care else sp).init_params(spec, seed=3)
    mixed = SacCore(_config(spec, care, precision, R), 0, seed=0)
    for r, row in enumerate(ROWS):
        mixed.set_hparams(r, **row)
    for r, row in enumerate(ROWS):
        got = mixed.get_hparams(r)
        assert all(got[k] == v for k, v in row.items()), (r, got)
    uniform = [SacCore(_config(spec, care, precision, R, **row), 0, seed=0) for row in ROWS]
    for core in [mixed] + uniform:
        for r in range(R):
            core.set_named(params, replica=r)
    for i in range(3):
        b, e1, e2 = _inputs(spec, care, R, i)
        for core in [mixed] + uniform:
            core.step(*b, e1, e2)
    Lm = mixed.read_losses(3)
    for r, uni in enumerate(uniform):
        for which in ARENAS:
            assert torch.equal(mixed.export_arena(which, r), uni.export_arena(which, r)), (plan, r, which)
        assert torch.equal(Lm[:, r], uni.read_losses(3)[:, r]), (plan, r)
        assert mixed.get_steps(r) == uni.get_steps(r)
    # replica 0 saw the same inputs in every uniform handle: what differs between them is the hyperparameters alone
    assert not torch.equal(uniform[0].export_arena(0, 0), uniform[1].export_arena(0, 0))
    for core in [mixed] + uniform:
        core.close()


@pytest.mark.parametrize("plan", ["chained", "per_layer", "care_o"])
def test_replica_hyperparameters_match_oracle(cuda, plan):
    """Replica 1 runs non-default values (lr_alpha != lr_actor != lr_critic, tau != tau_se, gamma != 0.99,
    reward_scale != 1) next to a default replica 0; it must follow the autograd oracle given the same values at the
    1e-4 bar, ReLU kinks proven as in the parity tests.  A swapped table field fails here."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(plan)
    row = ROWS[0]
    skip = ("lr_alpha",) if care else ("lr_alpha", "tau_se", "lr_ctx")
    ref_spec = dataclasses.replace(spec, **{k: v for k, v in row.items() if k not in skip})
    mod = cp if care else sp
    port = (cp.CarePortLearner if care else sp.PortLearner)(ref_spec, mod.init_params(spec, seed=3))
    # the oracle builds the temperature Adam with lr_actor, as the reference does; torch reads a group's lr at every step
    port.opt_alpha.param_groups[0]["lr"] = row["lr_alpha"]
    core = SacCore(_config(spec, care, precision, 2), 0, seed=0)
    core.set_hparams(1, **row)
    gen = torch.Generator().manual_seed(9)
    rep2 = lambda t: t.unsqueeze(0).repeat(2, 1, 1).clone()
    for i in range(3):
        b = mod.synthetic_batch(spec, seed=40 + i)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen)
        o, _ = kink_checked_step(core, port, ref_spec, b, e1, e2, replica=1, care=care,
                                 step_cuda=lambda: core.step(*[rep2(t) for t in b], rep2(e1), rep2(e2)))
        L = core.read_losses(1)[0, 1]
        assert rel_scalar(float(L[0]), o["critic_loss"]) <= REL, (i, float(L[0]), o["critic_loss"])
        assert rel_scalar(float(L[1]), o["actor_loss"]) <= REL, (i, float(L[1]), o["actor_loss"])
        check_port_state(core, port, replica=1)
    core.close()


B_ROW = dict(gamma=0.9, reward_scale=3.0, tau=0.05, lr_critic=2e-3, lr_actor=1e-3, lr_alpha=4e-3)


def _read(core):
    return core.read_losses(16), core.export_arena(0, 0), core.export_arena(0, 1)


def _set_b(core):
    core.set_hparams(None, **B_ROW)


@pytest.mark.parametrize("mode", ["stream", "legacy", "host"])
def test_set_hparams_is_stream_ordered(cuda, mode):
    """set_hparams enqueued right behind a graph launch without a synchronisation affects exactly the steps enqueued
    after it: the same as setting it on an idle device.  On a torch side stream, on the legacy default stream (bridged
    onto the handle's own stream) and with a pinned-host ring."""
    lx, ax0, ax1 = _stream_run(mode, _set_b, False, _read)
    ly, ay0, ay1 = _stream_run(mode, _set_b, True, _read)
    lz, _, _ = _stream_run(mode, None, False, _read)
    assert torch.equal(lx, ly)
    assert torch.equal(ax0, ay0) and torch.equal(ax1, ay1)
    assert torch.equal(lx[:8], lz[:8])            # the steps before the change used the old values ...
    assert not torch.equal(lx[8:, :, 0], lz[8:, :, 0])   # ... and the ones after it the new values


def test_copy_replica(cuda):
    """copy_replica between steps: dst == src (parameters, Adam moments, step counters), and the two stay bit-identical
    given identical inputs; dst keeps its own hyperparameters, so different values make them diverge."""
    from distributed_sac_b200.core import Replay, SacCore
    spec = SMALL
    R = 3
    core = SacCore(core_config(spec, replicas=R), 0, seed=11)
    core.set_steps((50, 60, 70), replica=0)      # distinct counters (and bias-correction products) in the source
    rb = Replay(core, capacity=4096, where="device", seed=5)
    rb.fill_synthetic(4096, seed=2)

    def step_same(i):
        b, e1, e2 = _inputs(spec, False, R, i)
        for t in b + [e1, e2]:
            t[2] = t[0]                          # replicas 0 and 2 get the same minibatch and noise
        core.step(*b, e1, e2)

    core.step_sampled(rb, 4)                     # the replicas draw different minibatches
    core.copy_replica(0, 2)                      # enqueued between steps, no synchronisation
    for i in range(2):
        step_same(i)
    for which in ARENAS:
        assert torch.equal(core.export_arena(which, 0), core.export_arena(which, 2)), which
    assert core.get_steps(2) == core.get_steps(0) == (56, 66, 76)
    assert core.get_steps(1) == (6, 6, 6)
    L = core.read_losses(2)
    assert torch.equal(L[:, 0], L[:, 2])
    assert not torch.equal(core.export_arena(0, 0), core.export_arena(0, 1))
    # hyperparameters are not part of the copy
    core.set_hparams(2, **B_ROW)
    want = core.get_hparams(2)
    core.copy_replica(0, 2)
    assert core.get_hparams(2) == want and core.get_hparams(0) != want
    for which in ARENAS:
        assert torch.equal(core.export_arena(which, 0), core.export_arena(which, 2)), which
    step_same(2)
    assert not torch.equal(core.export_arena(0, 0), core.export_arena(0, 2))
    rb.close()
    core.close()


def test_bad_hyperparameters_are_rejected(cuda):
    """NaN / inf, tau outside [0, 1], a negative learning rate and an out-of-range replica raise; nothing changes, on
    the host mirror or on the device (a step still equals a fresh handle's)."""
    from distributed_sac_b200.core import SacCore
    spec = SMALL
    cfg = core_config(spec, replicas=2, gamma=0.98, lr_alpha=1e-3)
    core, fresh = SacCore(cfg, 0, seed=1), SacCore(cfg, 0, seed=1)
    before = [core.get_hparams(r) for r in range(2)]
    assert before[0] == before[1] == dict(gamma=0.98, reward_scale=1.0, tau=0.005, lr_critic=3e-4, lr_actor=3e-4,
                                          lr_alpha=1e-3, tau_se=0.0, lr_ctx=0.0)
    bad = [dict(gamma=math.nan), dict(reward_scale=math.inf), dict(lr_actor=-math.inf), dict(tau=1.5), dict(tau=-0.1),
           dict(tau_se=1.5), dict(lr_critic=-1e-4), dict(lr_alpha=-1e-4), dict(lr_ctx=math.nan)]
    for kw in bad:
        for replica in (0, None):
            with pytest.raises(RuntimeError):
                core.set_hparams(replica, **kw)
    for replica in (2, -1):
        with pytest.raises(RuntimeError):
            core.set_hparams(replica, gamma=0.9)
        with pytest.raises(RuntimeError):
            core.get_hparams(replica)
        with pytest.raises(RuntimeError):
            core.copy_replica(0, replica)
    with pytest.raises(TypeError):
        core.set_hparams(0, lr=1e-3)
    assert [core.get_hparams(r) for r in range(2)] == before
    b, e1, e2 = _inputs(spec, False, 2, 0)
    for c in (core, fresh):
        c.step(*b, e1, e2)
    assert torch.equal(core.export_arena(0, 0), fresh.export_arena(0, 0))
    assert torch.equal(core.export_arena(0, 1), fresh.export_arena(0, 1))
    core.close()
    fresh.close()
