"""CPU: the clipping oracle of the grad_clip tests (_clip.clip_oracle: torch.nn.utils.clip_grad_norm_ right before each
optimizer's step(), the norms it returned kept) against the unclipped oracle and against scaling each optimizer's
gradients by hand; the layout call refuses an unknown grad_clip value."""
import dataclasses
import math

import pytest
import torch

import care_port as cp
import sac_port as sp
from _clip import clip_oracle
from _golden import CareCase

SPEC = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[32, 24], critic_hidden=[24, 32], batch=48)
CARE_O = dataclasses.replace(CareCase("care_o_small_s4").spec, num_tasks=4)
CASES = {"sac": (sp, SPEC), "care_o": (cp, CARE_O)}


def _run(mod, spec, n_steps, max_grad_norm=None):
    """n_steps updates of a fresh oracle learner clipped at max_grad_norm; returns (learner, [grad_norms of each step])."""
    port = (cp.CarePortLearner if mod is cp else sp.PortLearner)(spec, mod.init_params(spec, seed=3))
    clip_oracle(port, max_grad_norm)
    g = torch.Generator().manual_seed(5)
    norms = []
    for i in range(n_steps):
        b = mod.synthetic_batch(spec, seed=40 + i)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
        (port.update if mod is cp else port.update_SAC)(*b, e1, e2)
        norms.append(dict(port.grad_norms))
    return port, norms


def _state(port):
    st = port.adam_state()
    return [port.params(), st["m"], st["v"]]


def _equal(a, b):
    return all(torch.equal(x[k], y[k]) for x, y in zip(a, b) for k in x)


@pytest.mark.parametrize("case", CASES)
def test_infinite_max_grad_norm_is_no_clipping(case):
    mod, spec = CASES[case]
    clipped, norms = _run(mod, spec, 3, max_grad_norm=math.inf)
    free, _ = _run(mod, spec, 3)
    assert _equal(_state(clipped), _state(free))
    want = {"critic", "actor"} | ({"ctx"} if mod is cp else set())
    assert all(set(n) == want and all(v > 0 for v in n.values()) for n in norms)


@pytest.mark.parametrize("case", CASES)
def test_binding_max_grad_norm_scales_each_optimizer(case):
    """max_grad_norm = 0.3 x the smallest first-step norm == each optimizer's step() preceded by g *= min(1, max_norm /
    (||g|| + 1e-6)) over its own parameters (the temperature unscaled); the kept norms are the pre-scaling ones."""
    mod, spec = CASES[case]
    _, n0 = _run(mod, spec, 1, max_grad_norm=math.inf)
    thr = 0.3 * min(n0[0].values())
    clipped, norms = _run(mod, spec, 3, max_grad_norm=thr)

    by_hand = (cp.CarePortLearner if mod is cp else sp.PortLearner)(spec, mod.init_params(spec, seed=3))
    seen = []
    for opt in (by_hand.opt_critic, by_hand.opt_actor, getattr(by_hand, "opt_ctx", None)):
        if opt is None:
            continue

        def step(*a, _opt=opt, _orig=opt.step, **kw):
            gs = [t.grad for grp in _opt.param_groups for t in grp["params"] if t.grad is not None]
            norm = torch.linalg.vector_norm(torch.stack([torch.linalg.vector_norm(x) for x in gs]))
            coef = torch.clamp(thr / (norm + 1e-6), max=1.0)
            for x in gs:
                x.mul_(coef)
            seen.append(float(norm))
            return _orig(*a, **kw)
        opt.step = step
    g = torch.Generator().manual_seed(5)
    for i in range(3):
        b = mod.synthetic_batch(spec, seed=40 + i)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
        (by_hand.update if mod is cp else by_hand.update_SAC)(*b, e1, e2)
    assert _equal(_state(clipped), _state(by_hand))
    kept = [v for n in norms for v in n.values()]
    assert sorted(kept) == sorted(seen) and min(kept) > thr
    free, _ = _run(mod, spec, 3)
    assert not torch.equal(free.params()["actor.0.weight"], clipped.params()["actor.0.weight"])


def test_layout_rejects_unknown_grad_clip():
    import __graft_entry__ as ge
    ge.build()
    from distributed_sac_b200.core import CoreConfig, layout
    layout(CoreConfig(grad_clip=True))
    with pytest.raises(RuntimeError, match="b200sac error"):
        layout(CoreConfig(grad_clip=2))
