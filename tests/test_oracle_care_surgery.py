"""CPU: the CARE gradient-surgery oracle (oracle/care_surgery_ref.py) against care_port's ordinary step: the per-task
gradients of both losses sum to the gradients update() applies, PCGrad's Gram form equals its literal vector form on CARE
gradients, and the whole surgery step with every weight 1 is update() -- for CARE(M) and CARE(O)."""
import numpy as np
import pytest
import torch

import care_port as cp
import care_surgery_ref as cs
import pcgrad_ref as pr

VARIANTS = pytest.mark.parametrize("modified", [True, False], ids=["CARE(M)", "CARE(O)"])


def _spec(modified, T=3):
    return cp.CareSpec(state_dim=6, act_dim=2, num_tasks=T, actor_hidden=[24, 20], critic_hidden=[20, 24], batch=20 * T,
                       num_encoders=3, mix_hidden=[16, 12], mix_out=10, ctx_in=20, ctx_hidden=[12], ctx_out=10, emb_dim=10,
                       modified=modified, weighted_loss=modified)


def _batch(spec, seed):
    """care_port.synthetic_batch with the rows sorted into task blocks (row i of task i // (B / T))."""
    s, a, r, s2, d = cp.synthetic_batch(spec, seed=seed)
    order = torch.argsort(torch.argmax(s[:, -spec.num_tasks:], 1), stable=True)
    return s[order], a[order], r[order], s2[order], d[order]


def _eps(spec, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)


@VARIANTS
def test_task_grads_sum_to_step_gradient(modified):
    spec = _spec(modified)
    params = cp.init_params(spec, seed=2)
    batch, (e1, e2) = _batch(spec, 11), _eps(spec, 4)
    port = cp.CarePortLearner(spec, params)
    seen = {}

    def capture(which):       # the gradients each optimizer's step() sees; no update, so the actor pass reads `params`
        return lambda *a, **k: seen.update({which: {n: port.p[n].grad.clone() for n in cs.opt_names(port, which)}})
    port.opt_critic.step, port.opt_actor.step = capture(0), capture(1)
    if port.opt_ctx is not None:
        port.opt_ctx.step = capture(2)
    port.update(*batch, e1, e2)
    ref_port = cp.CarePortLearner(spec, params)
    for which in (0, 1):
        per = cs.task_grads(ref_port, batch, e1, e2, which)
        for opt in ((0, 2) if which == 0 and not modified else (which,)):
            for n in cs.opt_names(port, opt):
                tot = sum(t[n] for t in per)
                ref = seen[opt][n]
                assert torch.allclose(tot, ref, rtol=1e-5, atol=1e-7 * ref.abs().max().item()), n
    assert ("cenc.0.weight" in seen.get(2, {})) == (not modified)


@VARIANTS
def test_gram_form_matches_vector_pcgrad_on_care_gradients(modified):
    spec = _spec(modified, T=4)
    port = cp.CarePortLearner(spec, cp.init_params(spec, seed=3))
    batch, (e1, e2) = _batch(spec, 12), _eps(spec, 5)
    rng = np.random.default_rng(1)
    for which in (0, 1):
        names = cs.opt_names(port, which)
        g = pr.flat(cs.task_grads(port, batch, e1, e2, which), names)
        perms = pr.draw_perms(spec.num_tasks, rng)
        _, w, taken = pr.gram_solve(pr.gram(g), perms)
        vec, vtaken = pr.pcgrad_vector(g, perms)
        assert np.array_equal(taken, vtaken), which
        assert np.max(np.abs(w @ g - vec)) <= 1e-12 * (np.abs(g).sum(0).max() + 1e-300), which


def _conflict_batch(spec, seed):
    """Two tasks with the same states, actions and next states, and rewards of opposite sign."""
    s, a, r, s2, d = _batch(spec, seed)
    P = spec.batch // 2
    for x in (s, a, s2):
        x[P:] = x[:P]
    for x in (s, s2):                          # the one-hot stays the row's own task
        x[P:, spec.state_dim:] = x[:P, spec.state_dim:].flip(-1)
    r[:P] = 1000.0 + r[:P].abs()           # far above |Q| at the randn-initialised mixture encoders
    r[P:] = -r[:P]
    return s, a, r, s2, d


@VARIANTS
def test_surgery_update_with_unit_weights_is_the_ordinary_step(modified):
    """surgery_update with both PCGrad switches off, and with CAGrad c = 0, follows CarePortLearner.update over three
    steps on conflicting tasks; with PCGrad on the critic projects and the parameters move elsewhere."""
    spec = _spec(modified, T=2)
    params = cp.init_params(spec, seed=5)
    ref, off, c0, on = (cp.CarePortLearner(spec, params) for _ in range(4))
    perms = np.stack([pr.draw_perms(2, np.random.default_rng(k)) for k in range(2)])
    for k in range(3):
        batch, (e1, e2) = _conflict_batch(spec, 20 + k), _eps(spec, 30 + k)
        ref.update(*batch, e1, e2)
        cs.surgery_update(off, *batch, e1, e2, perms, on=(False, False))
        cs.surgery_update(c0, *batch, e1, e2, c=0.0)
        out = cs.surgery_update(on, *batch, e1, e2, perms)
        assert out[0][2].any(), k
    a = ref.params()
    for other in (off, c0):
        b = other.params()
        for n in a:
            assert torch.allclose(a[n], b[n], rtol=1e-5, atol=1e-6), n
        assert ref.adam_state()["step"] == other.adam_state()["step"]
    b = on.params()
    assert any(not torch.allclose(a[n], b[n], rtol=1e-5, atol=1e-6) for n in a)
