"""GPU: the CUDA step (through the C ABI) against the reference fixtures and the oracles."""
import math

import numpy as np
import pytest
import torch

import sac_manual as smn
import sac_port as sp
from _golden import (CASES, Case, REL, check_port_state, check_state, core_config, kink_checked_step, rel_l2, rel_scalar,
                     sync_core_to_port)
from _harness import cuda

pytestmark = pytest.mark.gpu


def _load(core, case, replica=0):
    from distributed_sac_b200 import _lib
    core.set_named(case.p_in, _lib.PARAMS, replica)
    core.set_named(case.m_in, _lib.ADAM_M, replica)
    core.set_named(case.v_in, _lib.ADAM_V, replica)
    core.set_steps(case.step_in, replica)


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("name", CASES)
def test_step_matches_reference_fixture(cuda, name, precision):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    c = Case(name)
    core = SacCore(core_config(c.spec, precision=precision), 0, seed=0)
    _load(core, c)
    for i in range(c.n_steps):
        core.step(*c.step_batch(i), c.eps_next[i], c.eps_cur[i])
        if i == 0:
            for k, ref in c.i0.items():
                got = core.debug(k).reshape(ref.shape)
                assert rel_l2(got, ref) <= REL, (k, rel_l2(got, ref))
        L = core.read_losses(1)[0, 0]
        assert rel_scalar(float(L[0]), c.losses[i, 0]) <= REL, ("critic_loss", i, float(L[0]), c.losses[i, 0])
        assert rel_scalar(float(L[1]), c.losses[i, 1]) <= REL, ("actor_loss", i, float(L[1]), c.losses[i, 1])
        if not math.isnan(c.losses[i, 2]):
            assert rel_scalar(float(L[3]), c.losses[i, 2]) <= REL, ("entropy", i)
    check_state(c, core.get_named(_lib.PARAMS), core.get_named(_lib.ADAM_M), core.get_named(_lib.ADAM_V),
                core.get_steps(), what="CUDA state")
    core.close()


DEEP_CRITIC = [56, 88, 24, 40, 64, 32]


@pytest.mark.parametrize("precision,critic_hidden", [
    pytest.param(0, [56, 88, 24], id="fp32"),
    pytest.param(1, [56, 88, 24], id="tc3xtf32"),
    pytest.param(0, DEEP_CRITIC, id="fp32-deep_critic"),      # the layer-chained plan past 4 critic layers
    pytest.param(1, DEEP_CRITIC, id="tc3xtf32-deep_critic"),
])
def test_backward_intermediates_match_manual_oracle(cuda, precision, critic_hidden):
    """d(action), d(mu|log_std) and every gradient tensor against oracle/sac_manual.py."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(state_dim=11, act_dim=3, actor_hidden=[72, 40], critic_hidden=critic_hidden, batch=200,
                      num_tasks=5, weighted_loss=False)
    p = sp.init_params(spec, seed=11)
    gen = torch.Generator().manual_seed(5)
    for k in p:
        p[k] = p[k] + 0.05 * torch.randn(p[k].shape, generator=gen)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=21)
    e1, e2 = torch.randn(200, 3, generator=gen), torch.randn(200, 3, generator=gen)
    man = smn.ManualLearner(spec, p, None, np.float32)
    I = man.update_SAC(s, a, r, s2, d, e1, e2)
    core = SacCore(core_config(spec, precision=precision), 0, seed=0)
    core.set_named(p)
    core.step(s, a, r, s2, d, e1, e2)
    assert rel_l2(core.debug("d_action").reshape(200, 3), I["d_action"]) <= REL
    assert rel_l2(core.debug("d_head").reshape(200, 6), I["d_head"]) <= REL
    assert rel_l2(core.debug("qmin").reshape(200, 1), I["qmin"]) <= REL
    g = core.get_named(_lib.GRADS)
    for k, ref in {**I["critic_grads"], **I["actor_grads"], "log_alpha": I["alpha_grad"]}.items():
        assert rel_l2(g[k].reshape(ref.shape), ref) <= REL, (k, rel_l2(g[k].reshape(ref.shape), ref))
    core.close()


def test_chained_plan_launch_count_does_not_grow_with_critic_depth(cuda):
    """The twin-critic passes of the layer-chained plan are one clustered launch each at every critic depth it accepts."""
    from distributed_sac_b200.core import SacCore
    counts = []
    for critic_hidden in ([64] * 3, [64] * 6):
        spec = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=critic_hidden, batch=256)
        core = SacCore(core_config(spec, precision=0), 0, seed=0)
        counts.append(core.launches_per_step)
        core.close()
    assert counts[0] == counts[1], counts


@pytest.mark.parametrize("state", ["fresh", "trained"])
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("shape", ["LL", "VS", "MS"])
def test_full_size_shapes_match_port(cuda, shape, precision, state):
    """BASELINE.json config shapes at full size vs the autograd oracle, three steps, everything at 1e-4.
    ReLU kinks are PROVEN, not budgeted (tests/_golden.py::kink_checked_step): the masks the CUDA step used are forced
    into the oracle, and every forced bit that differs from the oracle's own must sit on a numerically-zero pre-activation.
    state = "trained": the optimizers start deep into training -- step counts of the shipped checkpoints (3.3 M: bias
    corrections == 1), non-zero first and second moments, a non-zero temperature -- the regime the oracle itself is pinned
    to the reference in by tests/test_oracle_vs_reference.py (shipped MTSAC / CARE(M) checkpoints, container only)."""
    from distributed_sac_b200.core import SacCore
    spec = {"LL": sp.ll_spec, "VS": sp.vs_spec, "MS": sp.ms_spec}[shape]()
    p = sp.init_params(spec, seed=3)
    adam = None
    if state == "trained":
        g0 = torch.Generator().manual_seed(5)
        p = {k: (v * 1.5 if v.dim() == 2 else v + 0.05 * torch.randn(v.shape, generator=g0)) for k, v in p.items()}
        p["log_alpha"] = torch.full_like(p["log_alpha"], -1.2) + 0.3 * torch.randn(p["log_alpha"].shape, generator=g0)
        names = sp.param_names(spec, sp.TRAINABLE_NETS)
        m = {k: 1e-3 * torch.randn(p[k].shape, generator=g0) for k in names}
        v = {k: m[k] ** 2 * (1.0 + torch.rand(p[k].shape, generator=g0)) + 1e-10 for k in names}
        adam = {"m": m, "v": v, "step": (3300000, 3300000, 3300000)}
    port = sp.PortLearner(spec, p, adam_state=adam)
    core = SacCore(core_config(spec, precision=precision), 0, seed=0)
    gen = torch.Generator().manual_seed(77)
    total_flips = 0
    for i in range(3):
        b = sp.synthetic_batch(spec, seed=100 + i)
        e1 = torch.randn(spec.batch, spec.act_dim, generator=gen)
        e2 = torch.randn(spec.batch, spec.act_dim, generator=gen)
        o, flips = kink_checked_step(core, port, spec, b, e1, e2)
        total_flips += sum(flips.values())
        L = core.read_losses(1)[0, 0]
        assert rel_scalar(float(L[0]), o["critic_loss"]) <= REL, (i, float(L[0]), o["critic_loss"])
        assert rel_scalar(float(L[1]), o["actor_loss"]) <= REL, (i, float(L[1]), o["actor_loss"])
        assert rel_scalar(float(L[3]), o["entropy"]) <= REL
        check_port_state(core, port)
    print(f"[kinks] {shape} precision {precision}: {total_flips} mask bits differed, all at numerically-zero pre-activations")
    core.close()


def test_replicas_are_bit_identical_and_independent(cuda):
    """Same params + same minibatch in every replica slot => bit-identical results (no atomics, no
    cross-replica leakage); a different minibatch in one slot changes only that replica."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    c = Case("vs_small_s10")
    R = 3
    core = SacCore(core_config(c.spec, replicas=R, precision=1), 0, seed=0)
    for rep in range(R):
        _load(core, c, rep)
    for i in range(3):
        b = [t.unsqueeze(0).repeat(R, 1, 1).clone() for t in c.step_batch(i)]
        en = c.eps_next[i].unsqueeze(0).repeat(R, 1, 1).clone()
        ec = c.eps_cur[i].unsqueeze(0).repeat(R, 1, 1).clone()
        if i == 2:
            b[2][1] += 1.0            # perturb replica 1's rewards on the last step
        core.step(*b, en, ec)
    a0, a1, a2 = (core.export_arena(_lib.PARAMS, rep) for rep in range(R))
    assert torch.equal(a0, a2)
    assert not torch.equal(a0, a1)
    L = core.read_losses(3)
    assert torch.equal(L[:, 0], L[:, 2])
    core.close()


def test_host_step_equals_device_step(cuda):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    c = Case("ms_small_s5")
    a = SacCore(core_config(c.spec), 0, seed=0)
    b = SacCore(core_config(c.spec), 0, seed=0)
    _load(a, c)
    _load(b, c)
    for i in range(c.n_steps):
        a.step(*c.step_batch(i), c.eps_next[i], c.eps_cur[i])
        lb = b.step_host(*c.step_batch(i), c.eps_next[i], c.eps_cur[i])
        la = a.read_losses(1)[0]
        assert torch.equal(la, lb)
    assert torch.equal(a.export_arena(), b.export_arena())
    a.close()
    b.close()


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
def test_gradient_slices_with_replicas_match_port(cuda, precision):
    """Batch >= 512 switches on the gradient slices (split-K weight gradients, row-sliced head backward, slices summed in
    Adam).  Two replicas with the same inputs must stay bit-identical (parameters, Adam moments, exported slice-summed
    gradients) and follow the autograd port over three chained steps."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=640, num_tasks=0)
    p = sp.init_params(spec, seed=5)
    port = sp.PortLearner(spec, p)
    R = 2
    core = SacCore(core_config(spec, replicas=R, precision=precision), 0, seed=0)
    gen = torch.Generator().manual_seed(9)
    rep2 = lambda t: t.unsqueeze(0).repeat(R, 1, 1).clone()
    for i in range(3):
        b = sp.synthetic_batch(spec, seed=40 + i)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen)
        sync_core_to_port(core, port, 0)          # (kink_checked_step syncs replica 1; both replicas start from the oracle's state)
        o, _ = kink_checked_step(core, port, spec, b, e1, e2, replica=1,
                                 step_cuda=lambda: core.step(*[rep2(t) for t in b], rep2(e1), rep2(e2)))
        L = core.read_losses(1)[0]
        assert torch.equal(L[0], L[1])
        assert rel_scalar(float(L[0, 0]), o["critic_loss"]) <= REL and rel_scalar(float(L[0, 1]), o["actor_loss"]) <= REL
        check_port_state(core, port, replica=1)     # strict 1e-4 with the CUDA masks forced into the oracle
    assert torch.equal(core.export_arena(_lib.PARAMS, 0), core.export_arena(_lib.PARAMS, 1))
    assert torch.equal(core.export_arena(_lib.ADAM_V, 0), core.export_arena(_lib.ADAM_V, 1))
    g0, g1 = core.get_named(_lib.GRADS, 0), core.get_named(_lib.GRADS, 1)
    assert all(torch.equal(g0[k], g1[k]) for k in g0)
    core.close()
