"""CPU: the hand-derived-gradient oracle (what the CUDA kernels implement) agrees with
the autograd port and with the reference fixtures."""
import math

import numpy as np
import pytest
import torch

import sac_manual as smn
import sac_port as sp
from _golden import CASES, Case, REL, check_state, rel_l2, rel_scalar


@pytest.mark.parametrize("name", CASES)
def test_manual_fp32_matches_reference_fixture(name):
    c = Case(name)
    lrn = smn.ManualLearner(c.spec, c.p_in, {"m": c.m_in, "v": c.v_in, "step": tuple(c.step_in)}, np.float32)
    for i in range(c.n_steps):
        out = lrn.update_SAC(*c.step_batch(i), c.eps_next[i], c.eps_cur[i])
        if i == 0:
            for k, ref in c.i0.items():
                assert rel_l2(out[k], ref) <= REL, (k, rel_l2(out[k], ref))
        assert rel_scalar(out["critic_loss"], c.losses[i, 0]) <= REL
        assert rel_scalar(out["actor_loss"], c.losses[i, 1]) <= REL
        if not math.isnan(c.losses[i, 2]):
            assert rel_scalar(out["entropy"], c.losses[i, 2]) <= REL
    tt = lambda d: {k: torch.from_numpy(np.asarray(v)) for k, v in d.items()}
    check_state(c, tt(lrn.p), tt(lrn.m), tt(lrn.v), lrn.step)


def test_manual_gradients_match_autograd_fp64():
    """Closed-form gradients vs autograd at fp64 on a ragged MT problem (tight tolerance)."""
    spec = sp.SacSpec(state_dim=5, act_dim=3, actor_hidden=[17, 9], critic_hidden=[11, 13, 7], batch=24,
                      num_tasks=4, weighted_loss=True)
    p = sp.init_params(spec, seed=5)
    for k in p:                       # non-zero biases, distinct targets, varied alpha
        p[k] = p[k] + 0.1 * torch.randn(p[k].shape, generator=torch.Generator().manual_seed(hash(k) % 1000))
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=9)
    g = torch.Generator().manual_seed(3)
    e1, e2 = torch.randn(24, 3, generator=g), torch.randn(24, 3, generator=g)
    torch.set_default_dtype(torch.float64)
    try:
        p64 = {k: v.double() for k, v in p.items()}
        port = sp.PortLearner.__new__(sp.PortLearner)
        port.spec = spec
        port.p = {k: torch.nn.Parameter(v.clone(), requires_grad="_target" not in k) for k, v in p64.items()}
        port.opt_actor = torch.optim.Adam([port.p[n] for n in sp.param_names(spec, ("actor",), False)], lr=spec.lr_actor)
        port.opt_critic = torch.optim.Adam([port.p[n] for n in sp.param_names(spec, ("q1", "q2"), False)], lr=spec.lr_critic)
        port.opt_alpha = torch.optim.Adam([port.p["log_alpha"]], lr=spec.lr_actor)
        man = smn.ManualLearner(spec, p64, None, np.float64)
        for _ in range(3):
            o1 = port.update_SAC(s.double(), a.double(), r.double(), s2.double(), d.double(), e1.double(), e2.double())
            o2 = man.update_SAC(s, a, r, s2, d, e1, e2)
            assert rel_scalar(o2["critic_loss"], o1["critic_loss"]) < 1e-10
            assert rel_scalar(o2["actor_loss"], o1["actor_loss"]) < 1e-10
        for k, v in port.p.items():
            assert rel_l2(man.p[k], v.detach()) < 1e-9, k
    finally:
        torch.set_default_dtype(torch.float32)


def test_port_backward_intermediates_match_manual():
    """The autograd port's d(action) (through the critics alone) and d(mu|log_std) -- the per-row references of the CUDA
    step's backward -- against the hand-derived ones, on a ragged MT problem with act_dim 1 and one hidden layer."""
    for spec in (sp.SacSpec(state_dim=7, act_dim=3, actor_hidden=[20, 12], critic_hidden=[16, 24, 8], batch=33,
                            num_tasks=4, weighted_loss=True),
                 sp.SacSpec(state_dim=5, act_dim=1, actor_hidden=[36], critic_hidden=[20], batch=37)):
        p = sp.init_params(spec, seed=2)
        g = torch.Generator().manual_seed(8)
        p = {k: v + 0.05 * torch.randn(v.shape, generator=g) for k, v in p.items()}
        b = sp.synthetic_batch(spec, seed=4)
        e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
        o = sp.PortLearner(spec, p).update_SAC(*b, e1, e2, want_intermediates=True)
        I = smn.ManualLearner(spec, p, None, np.float32).update_SAC(*b, e1, e2)
        for k in ("d_action", "d_head"):
            assert o[k].shape == I[k].shape, (k, tuple(o[k].shape), I[k].shape)
            assert rel_l2(o[k], I[k]) <= REL, (k, rel_l2(o[k], I[k]))
