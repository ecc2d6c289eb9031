"""The priority-refresh oracle (oracle/refresh_ref.py) against the autograd port: for the same rows and noise, the y, q1
and q2 that PortLearner.update_SAC(want_intermediates=True) computes give the priorities td_priorities gives, and the
slot-keyed noise is Philox + Box-Muller of the documented counter."""
import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import per_ref
import philox_ref
import refresh_ref as rr
import sac_port as sp


def _params(spec, seed, ln=False):
    p = (lnp if ln else sp).init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 7)
    for k in p:
        if k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
        elif "_target." in k and k.endswith(".weight"):
            p[k] = p[k] + 0.02 * torch.randn(p[k].shape, generator=g)
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


@pytest.mark.parametrize("shape,ln", [("LL", False), ("VS", False), ("MS", False), ("LL", True)])
def test_td_priorities_match_the_port_step(shape, ln):
    kw = dict(actor_hidden=[32, 32], critic_hidden=[32, 24], batch=48)
    spec = {"LL": sp.ll_spec, "VS": sp.vs_spec, "MS": sp.ms_spec}[shape](**kw)
    p = _params(spec, 3, ln)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=11)
    eps = torch.randn(spec.batch, spec.act_dim, generator=torch.Generator().manual_seed(5))
    port = (lnp.LnPortLearner if ln else sp.PortLearner)(spec, p)
    if ln:
        with lnp._layer_norm_mlp():
            o = port.update_SAC(s, a, r, s2, d, eps_next=eps, want_intermediates=True)
    else:
        o = port.update_SAC(s, a, r, s2, d, eps_next=eps, want_intermediates=True)
    want = per_ref.td_priority(o["y"].reshape(-1), o["q1"].reshape(-1), o["q2"].reshape(-1))
    rows = dict(s=s.numpy(), a=a.numpy(), R=r.reshape(-1).numpy(), s2=s2.numpy(), d=d.reshape(-1).numpy(),
                g=np.full(spec.batch, np.float32(spec.gamma)), task=sp.task_ids(spec, s).numpy())
    prio, y, q1, q2 = rr.td_priorities(spec, p, rows, eps.numpy())
    np.testing.assert_allclose(q1, o["q1"].reshape(-1).numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(q2, o["q2"].reshape(-1).numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(y, o["y"].reshape(-1).numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(prio, want, rtol=1e-4, atol=1e-5)


def test_critic_values_are_the_port_mlp():
    spec = sp.ll_spec(actor_hidden=[16], critic_hidden=[16, 8], batch=8)
    p = _params(spec, 1)
    s, a = sp.synthetic_batch(spec, seed=2)[:2]
    for target in (False, True):
        q1, q2 = rr.critic_values(p, s, a, target)
        x = torch.cat([s, a], -1)
        sfx = "_target" if target else ""
        np.testing.assert_array_equal(q1, sp.mlp(p, "q1" + sfx, x).detach().reshape(-1).numpy())
        np.testing.assert_array_equal(q2, sp.mlp(p, "q2" + sfx, x).detach().reshape(-1).numpy())


def test_refresh_eps_is_the_documented_draw():
    slots, tasks = np.array([0, 5, 2 ** 33 + 7]), np.array([0, 1, 3])
    e = rr.refresh_eps(123, 2, slots, tasks, 3)
    key = (123 ^ (0xC2B2AE3D27D4EB4F * 3)) & (2 ** 64 - 1)
    for n, (i, t) in enumerate(zip(slots, tasks)):
        for k in range(3):
            w = philox_ref.philox(key, int(i) & 0xFFFFFFFF, int(i) >> 32, int(t), 0x7E00 + k)
            u, v = (((int(w[q]) >> 8) + 1) / 2 ** 24 for q in (0, 1))
            assert abs(e[n, k] - np.sqrt(-2 * np.log(u)) * np.cos(2 * np.pi * v)) < 1e-6
    # the slot, the task and the replica each change the draw; the order of the slots does not
    assert not np.array_equal(e, rr.refresh_eps(123, 1, slots, tasks, 3))
    assert not np.array_equal(e[0], rr.refresh_eps(123, 2, [0], [1], 3)[0])
    np.testing.assert_array_equal(rr.refresh_eps(123, 2, slots[::-1], tasks[::-1], 3), e[::-1])


def test_slot_rows_fold_a_linked_ring():
    cap_t, n = 8, 3
    r = np.arange(16, dtype=np.float32)
    d = np.zeros(16, np.float32)
    d[3] = 1
    link = np.full(16, -1, np.int64)
    link[0], link[1], link[2], link[3] = 1, 2, 3, 4
    s = np.arange(16 * 2, dtype=np.float32).reshape(16, 2)
    ring = (s, s[:, :1], r, s + 100, d)
    rows = rr.slot_rows(ring, [0, 2, 9], cap_t, 0.5, link, n)
    np.testing.assert_array_equal(rows["s2"][0], s[2] + 100)          # two hops from slot 0
    np.testing.assert_array_equal(rows["s2"][1], s[3] + 100)          # slot 3 is terminal
    assert rows["R"][0] == np.float32(0 + 0.5 * 1 + 0.25 * 2) and rows["g"][0] == np.float32(0.125)
    assert rows["d"][1] == 1 and list(rows["task"]) == [0, 0, 1]
    plain = rr.slot_rows(ring, [0, 9], cap_t, 0.5)
    assert list(plain["R"]) == [0, 9] and list(plain["g"]) == [0.5, 0.5]
