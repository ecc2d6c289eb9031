"""GPU: replay ring + sampled stepping (device-resident and pinned-host rings)."""
import numpy as np
import pytest
import torch

import sac_port as sp
from _golden import core_config
from _harness import cuda

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("where", ["device", "host"])
@pytest.mark.parametrize("T", [0, 4])
def test_push_sample_round_trip(cuda, where, T):
    from distributed_sac_b200.core import Replay, SacCore
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[32], critic_hidden=[32], batch=64, num_tasks=T)
    core = SacCore(core_config(spec), 0, seed=0)
    rb = Replay(core, capacity=4096, where=where, seed=1)
    n = 1500
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=3, batch=n)
    r = torch.arange(n, dtype=torch.float32).reshape(n, 1)     # reward == transition id
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    assert rb.size() == (n if T == 0 else min(int((s[:, 6:].argmax(1) == t).sum()) for t in range(T)))
    bs, ba, br, bs2, bd = rb.sample()
    ids = br[:, 0].long()
    assert len(set(ids.tolist())) == 64                     # without replacement
    assert torch.equal(bs, s[ids]) and torch.equal(ba, a[ids]) and torch.equal(bs2, s2[ids]) and torch.equal(bd, d[ids])
    if T:
        counts = np.bincount(bs[:, 6:].argmax(1).numpy(), minlength=T)
        assert (counts == 64 // T).all()                    # B/T per task (MS/replay_buffers.py:73-74)
    rb.close()
    core.close()


@pytest.mark.parametrize("where", ["device", "host"])
def test_sampled_steps_run_and_learn(cuda, where):
    """Critic loss on a fixed synthetic ring goes down over a few hundred sampled steps; ring
    wrap-around keeps the newest transitions."""
    from distributed_sac_b200.core import Replay, SacCore
    spec = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=128)
    core = SacCore(core_config(spec, replicas=2), 0, seed=5)
    rb = Replay(core, capacity=8192, where=where, seed=2)
    rb.fill_synthetic(8192, seed=9)
    assert rb.size(0) == 8192 and rb.size(1) == 8192
    core.step_sampled(rb, 300)
    L = core.read_losses(300)
    assert torch.isfinite(L).all()
    assert L[-20:, :, 0].mean() < L[:20, :, 0].mean()
    assert not torch.equal(L[:, 0], L[:, 1])                # replicas draw different minibatches
    rb.close()
    core.close()


def test_device_sampler_draws_unique_uniform_indices(cuda):
    """Device-side index sampling: no duplicates inside a minibatch; covers the ring."""
    _check_device_sampler(256)


def test_device_sampler_wide_batch(cuda):
    """The same at a batch above 256, which takes the 512-thread sampling launch (VSAC / MTSAC / CARE batches)."""
    _check_device_sampler(1024)


def _check_device_sampler(batch):
    from distributed_sac_b200.core import Replay, SacCore
    spec = sp.SacSpec(state_dim=4, act_dim=1, actor_hidden=[16], critic_hidden=[16], batch=batch)
    core = SacCore(core_config(spec), 0, seed=1)
    n = 4 * batch
    rb = Replay(core, capacity=n, where="device", seed=3)        # 4x batch: many collisions to resolve
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=4, batch=n)
    r = torch.arange(n, dtype=torch.float32).reshape(n, 1)
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    seen = np.zeros(n, np.int64)
    for _ in range(40):
        core.step_sampled(rb, 1)
        torch.cuda.synchronize()
        # the rewards of the ingested minibatch identify the sampled rows: y depends on r, read r via debug?
        # -> use the reference-shaped host sampler for distribution checks, the device sampler through 'y' is opaque,
        #    so check uniqueness through the ingest buffer exposed as debug tensor "r".
        ids = core.debug("r").long().numpy()
        assert len(set(ids.tolist())) == batch
        seen[ids] += 1
    assert (seen > 0).mean() > 0.99 and seen.max() <= 25
    rb.close()
    core.close()
