"""CPU: the Gram-form PCGrad weights the device implements (pcgrad_ref.gram_solve) against the literal vector restatement
of PCGrad on flattened gradients, and the per-task oracle gradients against sac_port's ordinary step gradient."""
import numpy as np
import pytest
import torch

import pcgrad_ref as pr
import sac_port as sp


def _sets():
    rng = np.random.default_rng(7)
    for T in (2, 3, 10):
        for trial in range(6):
            g = rng.standard_normal((T, 257))
            if trial == 1:                        # a conflicting pair: task 1 points against task 0
                g[1] = -0.7 * g[0] + 0.1 * rng.standard_normal(257)
            if trial == 2:                        # a zero gradient never projects and is never projected onto
                g[T - 1] = 0.0
            if trial == 3:                        # every task shares a common direction, with strong conflicts on top
                g = 0.3 * rng.standard_normal(257)[None, :] + g * np.where(np.arange(T)[:, None] % 2 == 0, 1.0, -1.0)
            yield T, trial, g, pr.draw_perms(T, rng)


@pytest.mark.parametrize("T,trial,g,perms", list(_sets()), ids=lambda x: None)
def test_gram_form_matches_vector_pcgrad(T, trial, g, perms):
    c, w, taken = pr.gram_solve(pr.gram(g), perms)
    vec, vtaken = pr.pcgrad_vector(g, perms)
    gram_total = w @ g
    scale = np.abs(g).sum(0).max() + 1e-300
    assert np.max(np.abs(gram_total - vec)) <= 1e-12 * scale
    assert np.array_equal(taken, vtaken)
    if trial == 1:
        assert taken.any()
    if trial == 2:
        assert not taken[:, T - 1].any() and not taken[T - 1].any()


def test_self_projection_and_decisions():
    """j = i in the permutation projects once g_i^PC has turned against g_i; the vector form, told the Gram form's
    decisions, gives the same total."""
    g = np.array([[2.0, 2.0], [-2.0, -4.0], [-2.0, -1.0]])
    perms = np.array([[1, 2, 0], [0, 1, 2], [0, 1, 2]])
    c, w, taken = pr.gram_solve(pr.gram(g), perms)
    assert taken[0, 1] and taken[0, 2] and taken[0, 0]      # 0 onto 1 and 2, then 0 against itself
    vec, _ = pr.pcgrad_vector(g, perms, decisions=taken)
    assert np.allclose(w @ g, vec, rtol=0, atol=1e-12)


def test_switch_off_gives_unit_weights():
    g = np.random.default_rng(3).standard_normal((4, 33))
    _, w, taken = pr.gram_solve(pr.gram(g), pr.draw_perms(4, np.random.default_rng(0)), on=False)
    assert np.array_equal(w, np.ones(4)) and not taken.any()


@pytest.mark.parametrize("T", [2, 3, 10])
def test_task_grads_sum_to_step_gradient(T):
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[24, 20], critic_hidden=[20, 24], batch=30 * T if T != 10 else 60,
                      num_tasks=T, weighted_loss=True)
    params = sp.init_params(spec, seed=2)
    batch = pr.block_batch(spec, seed=11)
    g = torch.Generator().manual_seed(4)
    e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
    port = sp.PortLearner(spec, params)
    seen = {}

    def capture(which):       # the gradients each optimizer's step() sees; no update, so the actor pass reads `params`
        return lambda *a, **k: seen.update({which: {n: port.p[n].grad.clone() for n in pr.opt_names(spec, which)}})
    port.opt_critic.step, port.opt_actor.step = capture(0), capture(1)
    port.update_SAC(*batch, e1, e2)
    for which in (0, 1):
        per = pr.task_grads(spec, params, batch, e1, e2, which)
        for n in pr.opt_names(spec, which):
            tot = sum(t[n] for t in per)
            ref = seen[which][n]
            assert torch.allclose(tot, ref, rtol=1e-5, atol=1e-7 * ref.abs().max().item()), n


def test_pcgrad_update_switched_off_is_the_ordinary_step():
    """pcgrad_update with both switches off (w = 1) follows sac_port.update_SAC; on, it moves the parameters elsewhere."""
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[24, 20], critic_hidden=[20, 24], batch=60, num_tasks=3,
                      weighted_loss=True)
    params = sp.init_params(spec, seed=5)
    g = torch.Generator().manual_seed(6)
    ref, off, on = sp.PortLearner(spec, params), sp.PortLearner(spec, params), sp.PortLearner(spec, params)
    perms = np.stack([pr.draw_perms(3, np.random.default_rng(k)) for k in range(2)])
    for k in range(3):
        batch = pr.block_batch(spec, seed=20 + k)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
        ref.update_SAC(*batch, e1, e2)
        pr.pcgrad_update(off, *batch, e1, e2, perms, on=(False, False))
        pr.pcgrad_update(on, *batch, e1, e2, perms)
    a, b, c = ref.params(), off.params(), on.params()
    for n in a:
        assert torch.allclose(a[n], b[n], rtol=1e-5, atol=1e-6), n
    assert any(not torch.allclose(a[n], c[n], rtol=1e-5, atol=1e-6) for n in a)
