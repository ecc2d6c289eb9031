"""CPU: the prioritized-replay references in oracle/per_ref.py -- the numpy sum-tree and the importance weighting of the
autograd oracle's critic update."""
import json

import numpy as np
import pytest
import torch

import per_ref
import sac_port as sp
from _golden import REL, rel_l2


def test_tree_sums_and_padding():
    rng = np.random.default_rng(0)
    leaves = rng.random(1000).astype(np.float32)
    tree = per_ref.build_tree(leaves)
    P = len(tree) // 2
    assert P == 1024 and (tree[P + 1000:] == 0).all()
    for n in (1, 2, 3, 17, 511):
        assert tree[n] == np.float32(tree[2 * n] + tree[2 * n + 1])
    assert abs(float(tree[1]) - float(leaves.astype(np.float64).sum())) <= 1e-5 * float(tree[1])


def test_leaf_values_and_weights():
    p = per_ref.leaf_values([0.0, 1.0, 3.0], alpha=0.5, eps=1.0)
    assert np.array_equal(p, np.float32(np.sqrt([1.0, 2.0, 4.0])))
    assert per_ref.leaf_values([0.0], 2.0, 1e-30)[0] == 0            # underflows to an empty-like leaf
    w = per_ref.is_weights(p, p.sum(), 3, 0.0)
    assert np.array_equal(w, np.ones(3, np.float32))
    w = per_ref.is_weights(p, p.sum(), 3, 1.0)
    assert w.max() == 1.0 and np.allclose(w, p.min() / p)
    y, q1, q2 = np.float32([1.0, -2.0]), np.float32([0.5, -2.0]), np.float32([2.0, -1.0])
    assert np.array_equal(per_ref.td_priority(y, q1, q2), [0.75, 0.5])


def test_descent_model_against_build_tree():
    """The numpy model of per_sample_kernel's descent: over a padded tree (cap 1000, P 1024, some empty slots) every draw
    lands on a filled slot of its stratum's prefix-sum interval, u = S (the rounding edge) stays off the empty tail, and
    with a zero root the descent ends on leaf P - 1 -- past a sub-ring of 1000 slots, i.e. in the next task's rows, which
    is why creation refuses an alpha, eps whose zero-priority leaf rounds to 0."""
    rng = np.random.default_rng(1)
    cap, fill, per = 1000, 950, 64
    leaves = np.zeros(cap, np.float32)
    leaves[:fill] = per_ref.leaf_values(rng.exponential(1.0, fill) ** 3, 0.6, 1e-6)
    tree = per_ref.build_tree(leaves)
    P = len(tree) // 2
    assert P == 1024
    cum = np.concatenate([[0.0], np.cumsum(tree[P:].astype(np.float64))])
    S = float(tree[1])
    lo, hi = per_ref.strata(tree, per)
    assert (np.diff(lo) >= 0).all() and (lo <= hi).all() and (hi[:-1] <= lo[1:]).all()
    for U in (np.zeros(per), np.full(per, per_ref.U_MAX), rng.random(per)):
        got = per_ref.stratified_draw(tree, per, U)
        assert (got < fill).all() and (tree[P + got] > 0).all() and (lo <= got).all() and (got <= hi).all()
        # the leaf's prefix-sum interval meets its stratum's (to fp32 rounding of the partial sums)
        j = np.arange(per)
        tol = 1e-6 * S
        assert (cum[got] <= (j + 1) * S / per + tol).all() and (cum[got + 1] >= j * S / per - tol).all()
    assert per_ref.descend(tree, S) == fill - 1 and per_ref.descend(tree, 2 * S) == fill - 1
    assert per_ref.descend(tree, 0.0) == 0
    # a zero root (every filled leaf 0): leaf P - 1, beyond the 1000 slots of the sub-ring
    zero = per_ref.build_tree(np.zeros(cap, np.float32))
    assert {int(x) for x in per_ref.stratified_draw(zero, per, rng.random(per))} == {P - 1} and P - 1 >= cap
    # which (alpha, eps) give such leaves: (0 + eps)^alpha rounding to 0 in fp32
    assert per_ref.leaf_values([0.0], 2.0, 1e-30)[0] == 0 and per_ref.leaf_values([0.0], 2.0, 1e-20)[0] > 0


def _problem(weighted_loss):
    spec = sp.SacSpec(state_dim=6, act_dim=3, actor_hidden=[32, 16], critic_hidden=[24, 40], batch=20,
                      num_tasks=4 if weighted_loss else 0, weighted_loss=weighted_loss)
    g = torch.Generator().manual_seed(6)
    e1, e2 = torch.randn(20, 3, generator=g), torch.randn(20, 3, generator=g)
    return spec, sp.init_params(spec, seed=4), sp.synthetic_batch(spec, seed=5), e1, e2, torch.rand(20, generator=g) * 0.9 + 0.1


@pytest.mark.parametrize("weighted_loss", [False, True])
def test_unit_weights_change_nothing(weighted_loss):
    """Weights of 1 give the unweighted oracle step bit for bit."""
    spec, params, batch, e1, e2, _w = _problem(weighted_loss)
    a, b = sp.PortLearner(spec, params), sp.PortLearner(spec, params)
    oa = a.update_SAC(*batch, e1, e2, want_intermediates=True)
    with per_ref.ImportanceWeights(np.ones(spec.batch)):
        ob = b.update_SAC(*batch, e1, e2, want_intermediates=True)
    assert oa["critic_loss"] == ob["critic_loss"] and oa["actor_loss"] == ob["actor_loss"]
    assert abs(per_ref.weighted_critic_loss(oa, np.ones(spec.batch), weighted_loss) - oa["critic_loss"]) <= 1e-6 * oa["critic_loss"]
    for k, v in a.params().items():
        assert torch.equal(v, b.params()[k]), k
    assert sp.mlp.__module__ == "sac_port"                     # the context restored the oracle


@pytest.mark.parametrize("weighted_loss", [False, True])
def test_weighted_critic_gradient(weighted_loss):
    """Inside ImportanceWeights the oracle's critic gradient is that of mean(w (y - Qk)^2) / div: with plain SGD (lr 1) on the
    critics, each parameter moves by minus the explicit weighted-loss gradient; the actor update is the unweighted one."""
    spec, params, batch, e1, e2, w = _problem(weighted_loss)
    s, a = batch[0], batch[1]
    port = sp.PortLearner(spec, params)
    critic = port.opt_critic.param_groups[0]["params"]
    port.opt_critic = torch.optim.SGD(critic, lr=1.0)
    before = port.params()
    with per_ref.ImportanceWeights(w):
        out = port.update_SAC(*batch, e1, e2, want_intermediates=True)
    after = port.params()
    div = float(spec.batch) if weighted_loss else 1.0
    x = torch.cat([s, a], -1)
    for q in ("q1", "q2"):
        pq = {k: v.clone().requires_grad_() for k, v in before.items() if k.startswith(q + ".")}
        loss = torch.mean(w.reshape(-1, 1) * (out["y"] - sp.mlp(pq, q, x)) ** 2) / div
        loss.backward()
        for k, v in pq.items():
            assert rel_l2(before[k] - after[k], v.grad) <= REL, (k, rel_l2(before[k] - after[k], v.grad))
    ref = sp.PortLearner(spec, params)
    ref.opt_critic = torch.optim.SGD(ref.opt_critic.param_groups[0]["params"], lr=1.0)
    unweighted = ref.update_SAC(*batch, e1, e2, want_intermediates=True)
    assert abs(per_ref.weighted_critic_loss(out, w, weighted_loss) - unweighted["critic_loss"]) > 1e-3 * unweighted["critic_loss"]
    assert not torch.equal(after["q1.0.weight"], ref.params()["q1.0.weight"])


def test_learner_rejects_prioritized_host_ring(tmp_path):
    from distributed_sac_b200.learner import Learner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps({"device": "cuda"}))
    with pytest.raises(ValueError, match="replay_where='device'"):
        Learner(str(p), write_mode=False, replay_where="host", prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6))
