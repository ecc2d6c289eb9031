"""GPU: the contract every per-replica setting keeps (hyperparameters, update intervals, gradient-clipping thresholds, PCGrad
switches, the PER beta and the n-step horizon), on a torch side stream and on the legacy default stream:
(a) a change enqueued right behind a prepared multi-step graph launch, without a synchronisation, gives the steps
    bit-identical to the same change made after one, and the steps after it differ from a run without it;
(b) the getter returns the new value at once;
(c) a refused value or an out-of-range replica leaves the getter's value as it was, and the next steps bit-identical to a
    handle that never saw the call;
(d) copy_replica leaves dst's row of a handle setting as it was."""
import contextlib
import dataclasses
import math

import numpy as np
import pytest
import torch

import sac_port as sp
from _golden import core_config
from _harness import PARAMS, SMALL, cuda  # noqa: F401

pytestmark = pytest.mark.gpu

R = 2
PCGRAD_SPEC = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[64, 48], critic_hidden=[48, 64], batch=96, num_tasks=2,
                         weighted_loss=True)


def _plain(core, rb):
    rb.fill_synthetic(4096, seed=9)


def _prioritized(core, rb):
    rb.fill_synthetic(4096, seed=9)
    for r in range(R):                             # non-uniform priorities: beta changes the importance weights
        rb.set_priorities(np.arange(4096), np.arange(4096) % 50 / 7.0, replica=r)


def _conflicting(core, rb):
    """Rewards of opposite sign for the two tasks, so that the critic's task gradients conflict."""
    spec = PCGRAD_SPEC
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=4, batch=2000)
    r = torch.where(s[:, spec.state_dim:spec.state_dim + 1] > 0, 5.0 + r.abs(), -5.0 - r.abs())
    for rep in range(R):
        rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy(), replica=rep)


def _raw(core, setter, *args):
    """b200sac_<setter>(handle, *args, current stream): values and replicas the Python methods would not pass on."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import _stream
    _lib.check(getattr(core.lib, "b200sac_" + setter)(core._h, *args, _stream()))


def _hparams_of(core, replica, **kw):
    import ctypes as C
    from distributed_sac_b200 import _lib
    return C.byref(_lib.Hparams(**dict(core.get_hparams(replica), **kw)))


@dataclasses.dataclass
class Setting:
    spec: sp.SacSpec
    cfg: dict                  # CoreConfig fields beyond the spec's
    ring: dict                 # Replay keywords beyond capacity and seed
    fill: object               # fill(core, rb)
    set: object                # set(core, rb, replica): the change
    get: object                # get(core, rb, replica), or None: no getter
    refused: tuple             # calls that must raise and change nothing
    handle: bool = True        # a handle setting (copy_replica concerns it)


SETTINGS = {
    "hparams": Setting(
        SMALL, {}, {}, _plain,
        lambda core, rb, r: core.set_hparams(r, lr_critic=3e-3, lr_actor=2e-3),
        lambda core, rb, r: core.get_hparams(r),
        (lambda core, rb: core.set_hparams(None, lr_critic=-1e-3), lambda core, rb: core.set_hparams(1, tau=math.nan),
         lambda core, rb: _raw(core, "set_hparams", R, _hparams_of(core, 0)),
         lambda core, rb: _raw(core, "set_hparams", -1, _hparams_of(core, 0)))),
    "intervals": Setting(
        SMALL, {}, {}, _plain,
        lambda core, rb, r: core.set_update_intervals(actor_every=2, target_every=2, replica=r),
        lambda core, rb, r: core.get_update_intervals(r),
        (lambda core, rb: core.set_update_intervals(actor_every=0), lambda core, rb: core.set_update_intervals(target_every=-2, replica=1),
         lambda core, rb: _raw(core, "set_update_intervals", R, 2, 2))),
    "grad_clip": Setting(
        SMALL, dict(grad_clip=True), {}, _plain,
        lambda core, rb, r: core.set_grad_clip(critic=1e-2, actor=1e-2, replica=r),
        lambda core, rb, r: core.get_grad_clip(r),
        (lambda core, rb: core.set_grad_clip(critic=0.0), lambda core, rb: core.set_grad_clip(actor=math.nan, replica=1),
         lambda core, rb: _raw(core, "set_grad_clip", R, 1e-2, 1e-2, 1e-2))),
    "pcgrad": Setting(
        PCGRAD_SPEC, dict(pcgrad=True, precision=1), {}, _conflicting,
        lambda core, rb, r: core.set_pcgrad(critic=False, actor=False, replica=r),
        lambda core, rb, r: core.get_pcgrad(r),
        (lambda core, rb: _raw(core, "set_pcgrad", 0, 2, 1), lambda core, rb: _raw(core, "set_pcgrad", 1, 0, -1),
         lambda core, rb: _raw(core, "set_pcgrad", R, 0, 0))),
    "beta": Setting(
        SMALL, {}, dict(prioritized=dict(alpha=0.6, beta=0.0, eps=1e-3)), _prioritized,
        lambda core, rb, r: rb.set_beta(1.0, replica=r),
        None,
        (lambda core, rb: rb.set_beta(1.5), lambda core, rb: rb.set_beta(math.nan, replica=1),
         lambda core, rb: rb.set_beta(1.0, replica=R)),
        handle=False),
    "nstep": Setting(
        SMALL, {}, dict(trajectories=True), _plain,
        lambda core, rb, r: rb.set_nstep(3, replica=r),
        lambda core, rb, r: rb.get_nstep(r),
        (lambda core, rb: rb.set_nstep(0), lambda core, rb: rb.set_nstep(17, replica=1), lambda core, rb: rb.set_nstep(3, replica=-1)),
        handle=False),
}
MODES = ["stream", "legacy"]


@contextlib.contextmanager
def _learner(name, mode):
    """A fresh R = 2 handle and its filled device ring, prepared, used on a torch side stream ("stream") or on the legacy
    default stream ("legacy": bridged onto the handle's own stream)."""
    from distributed_sac_b200.core import Replay, SacCore
    st = SETTINGS[name]
    core = SacCore(core_config(st.spec, replicas=R, **st.cfg), 0, seed=7)
    stream = torch.cuda.Stream() if mode == "stream" else None
    try:
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            rb = Replay(core, 4096, seed=3, **st.ring)
            try:
                st.fill(core, rb)
                core.prepare(rb)
                yield core, rb
            finally:
                rb.close()
    finally:
        core.close()


def _outcome(core):
    return core.read_losses(16).nan_to_num(7.0), [core.export_arena(PARAMS, r) for r in range(R)]   # (NaN: a skipped actor update)


def _equal(x, y):
    return torch.equal(x[0], y[0]) and all(torch.equal(a, b) for a, b in zip(x[1], y[1]))


def _run(name, mode, change, sync_before_change):
    """8 steps (one graph launch), change(core, rb) unless None, 8 more; returns (outcome, what change left the getters
    reading, read right after it)."""
    st = SETTINGS[name]
    with _learner(name, mode) as (core, rb):
        core.step_sampled(rb, 8)
        if sync_before_change:
            torch.cuda.synchronize()
        if change is not None:
            change(core, rb)
        got = None if st.get is None else [st.get(core, rb, r) for r in range(R)]
        core.step_sampled(rb, 8)
        return _outcome(core), got


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(SETTINGS))
def test_change_is_stream_ordered(cuda, name, mode):
    """(a) and (b)."""
    st = SETTINGS[name]
    change = lambda core, rb: st.set(core, rb, None)
    x, got_x = _run(name, mode, change, False)
    y, got_y = _run(name, mode, change, True)
    z, got_z = _run(name, mode, None, False)
    assert _equal(x, y)
    assert torch.equal(x[0][:8], z[0][:8])            # the steps before the change read the old value ...
    assert not torch.equal(x[0][8:], z[0][8:])        # ... and the ones after it the new one
    assert not _equal(x, z)
    if st.get is not None:
        assert got_x == got_y and got_x[0] == got_x[1] and got_x != got_z


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(SETTINGS))
def test_refusals_change_nothing(cuda, name, mode):
    """(c)."""
    st = SETTINGS[name]
    with _learner(name, mode) as (core, rb):
        before = None if st.get is None else [st.get(core, rb, r) for r in range(R)]
        for call in st.refused:
            with pytest.raises(RuntimeError):
                call(core, rb)
        if st.get is not None:
            assert [st.get(core, rb, r) for r in range(R)] == before
        core.step_sampled(rb, 8)
        core.step_sampled(rb, 8)
        seen = _outcome(core)
    with _learner(name, mode) as (core, rb):
        core.step_sampled(rb, 8)
        core.step_sampled(rb, 8)
        fresh = _outcome(core)
    assert _equal(seen, fresh)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", [n for n, st in SETTINGS.items() if st.handle])
def test_copy_replica_keeps_dst_row(cuda, name, mode):
    """(d): dst's row set before copy_replica == set after it (so the copy left it alone), and it still changes the steps."""
    st = SETTINGS[name]

    def set_then_copy(core, rb):
        st.set(core, rb, 1)
        core.copy_replica(0, 1)

    def copy_then_set(core, rb):
        core.copy_replica(0, 1)
        st.set(core, rb, 1)

    x, got_x = _run(name, mode, set_then_copy, False)
    y, got_y = _run(name, mode, copy_then_set, False)
    z, got_z = _run(name, mode, lambda core, rb: core.copy_replica(0, 1), False)
    assert _equal(x, y)
    assert got_x == got_y and got_x[0] == got_z[0] == got_z[1] and got_x[1] != got_z[1]
    assert not torch.equal(x[1][1], z[1][1])
