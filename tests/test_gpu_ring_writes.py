"""GPU: b200sac_replay_fill_synthetic is a writer of the ring like push -- it takes the ring's mutex and waits for every
gather already enqueued before it rewrites rows, fill, tree leaves or links.  Sampled steps enqueued on a side stream and
a refill issued right after them on the default stream must train exactly as when the two are separated by a device
synchronise."""
import pytest
import torch

import sac_port as sp
from _golden import core_config
from _harness import cuda

pytestmark = pytest.mark.gpu

_SPEC = sp.SacSpec(state_dim=39, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=256)
_KINDS = {"uniform": {}, "prioritized": dict(prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6)), "linked": dict(trajectories=True)}


def _run(kind, sync_before_refill):
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(_SPEC), 0, seed=5)
    ring = Replay(core, 16 * _SPEC.batch, "device", seed=6, **_KINDS[kind])
    ring.fill_synthetic(16 * _SPEC.batch, seed=7)
    if kind == "linked":
        ring.set_nstep(3)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for n in (8, 8, 5):
            core.step_sampled(ring, n)
    if sync_before_refill:
        torch.cuda.synchronize()
    ring.fill_synthetic(12 * _SPEC.batch, seed=8)        # default stream, right behind the enqueued steps
    with torch.cuda.stream(side):
        core.step_sampled(ring, 4)
    torch.cuda.synchronize()
    from distributed_sac_b200 import _lib
    out = dict(losses=core.read_losses(25), steps=core.get_steps(),
               **{w: core.export_arena(which) for w, which in (("params", _lib.PARAMS), ("adam_m", _lib.ADAM_M),
                                                               ("adam_v", _lib.ADAM_V))})
    ring.close()
    core.close()
    return out


@pytest.mark.parametrize("kind", list(_KINDS))
def test_refill_behind_side_stream_steps(cuda, kind):
    raced, ref = _run(kind, False), _run(kind, True)
    assert raced["steps"] == ref["steps"] == (25, 25, 25)
    for k in ("losses", "params", "adam_m", "adam_v"):
        assert torch.equal(raced[k], ref[k]), f"{kind}: {k} differs from the synchronised run"
