"""GPU: size-independent properties of the step at BASELINE.json's full sizes (no oracle needed)."""
import numpy as np
import pytest
import torch

import sac_port as sp
from _golden import core_config
from _harness import cuda

pytestmark = pytest.mark.gpu


def _inputs(spec, seed):
    b = sp.synthetic_batch(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    return b, torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)


@pytest.mark.parametrize("shape,precision", [("LL", 0), ("LL", 1), ("VS", 1), ("MS", 1)])
def test_zero_learning_rates_and_tau_leave_every_parameter_bit_identical(cuda, shape, precision):
    """lr = 0, tau = 0: Adam moments move, parameters and targets must not (exercises every write path)."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec = {"LL": sp.ll_spec, "VS": sp.vs_spec, "MS": sp.ms_spec}[shape](lr_actor=0.0, lr_critic=0.0, tau=0.0)
    core = SacCore(core_config(spec, precision=precision), 0, seed=3)
    before = core.export_arena()
    b, e1, e2 = _inputs(spec, 5)
    for _ in range(2):
        core.step(*b, e1, e2)
    L = core.read_losses(2)
    assert torch.equal(core.export_arena(), before)
    assert torch.isfinite(L).all() and torch.equal(L[0], L[1])          # same inputs, same weights -> same losses
    assert core.export_arena(_lib.ADAM_M).abs().sum() > 0
    core.close()


@pytest.mark.parametrize("shape,precision", [("LL", 0), ("VS", 1)])
def test_minibatch_row_order_does_not_matter(cuda, shape, precision):
    """The step is a sum over the minibatch: permuting the rows (with their noise) changes nothing beyond fp32
    summation order (MS/replay_buffers.py:83-84 shuffles rows for exactly that reason: it is irrelevant)."""
    from distributed_sac_b200.core import SacCore
    spec = {"LL": sp.ll_spec, "VS": sp.vs_spec}[shape]()
    p = sp.init_params(spec, seed=9)
    b, e1, e2 = _inputs(spec, 11)
    perm = torch.randperm(spec.batch, generator=torch.Generator().manual_seed(1))
    outs = []
    for order in (None, perm):
        core = SacCore(core_config(spec, precision=precision), 0, seed=0)
        core.set_named(p)
        bb = b if order is None else tuple(t[order] for t in b)
        ee = (e1, e2) if order is None else (e1[order], e2[order])
        core.step(*bb, *ee)
        outs.append((core.read_losses(1)[0, 0], core.export_arena()))
        core.close()
    (l0, a0), (l1, a1) = outs
    assert torch.allclose(l0, l1, rtol=2e-5, atol=1e-7)
    assert ((a0 - a1).norm() / a0.norm()).item() < 2e-5


def test_hard_target_copy_is_exact_and_idempotent(cuda):
    from distributed_sac_b200.core import SacCore
    spec = sp.vs_spec()
    core = SacCore(core_config(spec), 0, seed=1)
    p = sp.init_params(spec, seed=2)
    for k in list(p):
        if "_target" in k:
            p[k] = p[k] + 1.0
    core.set_named(p)
    core.soft_update(1.0)                                   # Learner.run(): soft_update(local, target, 1.0)
    n = core.get_named()
    for k in n:
        if "_target" in k:
            assert torch.equal(n[k], n[k.replace("_target", "")])
    a = core.export_arena()
    core.soft_update(1.0)
    assert torch.equal(core.export_arena(), a)
    core.soft_update(0.25)                                  # targets == locals: any tau is a fixed point
    assert torch.allclose(core.export_arena(), a, rtol=0, atol=1e-7)
    core.close()


def test_in_kernel_noise_path_is_reproducible_and_seed_dependent(cuda):
    """Device ring + Philox sampling and noise: same seeds -> bit-identical learners; other seed -> different."""
    from distributed_sac_b200.core import Replay, SacCore
    spec = sp.ll_spec()
    arenas = []
    for seed in (7, 7, 8):
        core = SacCore(core_config(spec), 0, seed=seed)
        ring = Replay(core, 1 << 16, "device", seed=seed)
        ring.fill_synthetic(1 << 16, seed=123)
        core.step_sampled(ring, 50)
        arenas.append(core.export_arena())
        assert torch.isfinite(core.read_losses(50)).all()
        ring.close()
        core.close()
    assert torch.equal(arenas[0], arenas[1]) and not torch.equal(arenas[0], arenas[2])


@pytest.mark.parametrize("where", ["device", "host"])
def test_ring_wraps_and_keeps_the_newest_transitions(cuda, where):
    from distributed_sac_b200.core import Replay, SacCore
    spec = sp.SacSpec(state_dim=5, act_dim=2, actor_hidden=[16], critic_hidden=[16], batch=32)
    core = SacCore(core_config(spec), 0, seed=0)
    cap, n = 256, 700
    rb = Replay(core, cap, where, seed=0)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=2, batch=n)
    r = torch.arange(n, dtype=torch.float32).reshape(n, 1)
    for lo in range(0, n, 100):                              # pushed in chunks like the Redis drain thread does
        sl = slice(lo, min(n, lo + 100))
        rb.push(s[sl].numpy(), a[sl].numpy(), r[sl].numpy(), s2[sl].numpy(), d[sl].numpy())
    assert rb.size() == cap
    seen = set()
    for _ in range(60):
        seen |= set(rb.sample()[2][:, 0].long().tolist())
    assert min(seen) >= n - cap and max(seen) == n - 1 and len(seen) > 0.95 * cap   # deque(maxlen) semantics
    rb.close()
    core.close()
