"""GPU: prioritized experience replay on the device ring -- sum-tree sampling, importance-weighted critic loss and the
in-graph priority update (include/b200sac.h, per_kernels.cuh), against oracle/per_ref.py and the autograd oracle."""
import numpy as np
import pytest
import torch
from scipy import stats

import care_port as cp
import per_ref
import sac_port as sp
from _golden import REL, check_forced, check_port_state, cuda_relu_masks, rel_scalar, sync_core_to_port
from _harness import MTSAC_T4, PER_LAYER, VS400, _core, _tasks, care_t4, cuda

pytestmark = pytest.mark.gpu

PER = dict(alpha=0.6, beta=0.4, eps=1e-6)


def _spec(name):
    """(spec, care, precision): layer-chained fp32, per-layer wgmma, per-layer fp32 / wgmma at 400 wide, MTSAC weighted_loss,
    CARE(M) with T = 4."""
    if name == "chained":
        return sp.ll_spec(), False, 0
    if name == "per_layer":
        return sp.SacSpec(**PER_LAYER), False, 1
    if name in ("wide_p0", "wide_p1"):
        return sp.SacSpec(**VS400), False, int(name[-1])
    if name == "mtsac":
        return sp.SacSpec(**MTSAC_T4), False, 1
    return care_t4(), True, 1


def _filled_ring(core, spec, care, n, cap, seed=5, replica=0, prioritized=PER, ring_seed=1):
    """A prioritized ring holding n synthetic transitions; returns (ring, host table [ring index] -> the five row
    tensors).  The ring keeps each task's rows in push order in that task's sub-ring."""
    from distributed_sac_b200.core import Replay
    rb = Replay(core, cap, seed=ring_seed, prioritized=prioritized)
    s, a, r, s2, d = (cp if care else sp).synthetic_batch(spec, seed=seed, batch=n)
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy(), replica=replica)
    T = max(spec.num_tasks, 1)
    cap_t = cap // T
    tid = _tasks(spec, s)
    where = np.empty(n, np.int64)
    for t in range(T):
        rows = np.nonzero(tid == t)[0]
        where[rows] = t * cap_t + np.arange(len(rows))
    table = [torch.zeros(cap, x.shape[1]) for x in (s, a, r, s2, d)]
    for t, x in zip(table, (s, a, r, s2, d)):
        t[where] = x
    return rb, table


def _drawn(core, spec, table, replica=0):
    """The minibatch, noise and weights of the last sampled step."""
    B, A = spec.batch, spec.act_dim
    idx = core.debug("idx", replica).long()
    batch = [t[idx] for t in table]
    eps = core.debug("psave", replica).reshape(2 * B, A, 8)[:, :, 5]
    return batch, eps[:B].clone(), eps[B:].clone(), core.debug("isw", replica), idx


@pytest.mark.parametrize("name", ["chained", "wide_p0", "wide_p1", "care_m"])
def test_neutral_weights_bit_exact(cuda, name):
    """beta = 0: every weight is exactly 1 and ten PER steps equal b200sac_step on the same minibatches bit for bit
    (same seed, so the same Philox noise): parameters, targets, Adam moments, losses."""
    spec, care, precision = _spec(name)
    per_core, ref_core = _core(spec, care, precision), _core(spec, care, precision)
    rb, table = _filled_ring(per_core, spec, care, 4096, 4096, prioritized=dict(PER, beta=0.0))
    for _ in range(10):
        per_core.step_sampled(rb, 1)
        batch, _e1, _e2, w, _idx = _drawn(per_core, spec, table)
        assert torch.equal(w, torch.ones_like(w))
        ref_core.step(*[x.unsqueeze(0) for x in batch])
    for which in (0, 1, 2):
        assert torch.equal(per_core.export_arena(which), ref_core.export_arena(which)), (name, which)
    assert torch.equal(per_core.read_losses(10), ref_core.read_losses(10))
    rb.close()
    per_core.close()
    ref_core.close()


@pytest.mark.parametrize("name", ["chained", "per_layer", "mtsac", "care_m"])
def test_weighted_parity_with_oracle(cuda, name):
    """beta = 1 on skewed priorities: each PER step matches the autograd oracle given the step's importance weights
    (CUDA masks, tanh values and min routing forced, kinks proven) at the 1e-4 bar: losses, y, Q, actions, log-probs and
    every parameter, target and Adam moment."""
    spec, care, precision = _spec(name)
    core = _core(spec, care, precision)
    n = 4096
    rb, table = _filled_ring(core, spec, care, n, n, prioritized=dict(PER, beta=1.0))
    rng = np.random.default_rng(3)
    idx_all = np.arange(n)
    rb.set_priorities(idx_all, rng.exponential(1.0, n) ** 3)
    mod = cp if care else sp
    port = (cp.CarePortLearner if care else sp.PortLearner)(spec, mod.init_params(spec, seed=3))
    for step in range(3):
        sync_core_to_port(core, port)
        core.step_sampled(rb, 1)
        batch, e1, e2, w, _idx = _drawn(core, spec, table)
        assert float(w.max()) == 1.0 and float(w.min()) < 0.5, "the weights are not skewed"
        forced = cuda_relu_masks(core, spec, care=care)
        with per_ref.ImportanceWeights(w), sp.ReluTape(forced) as tape:
            out = (port.update if care else port.update_SAC)(*batch, e1, e2, want_intermediates=True)
        check_forced(tape, forced, f"{name} step {step}: ")
        L = core.read_losses(1)[0, 0]
        for j, want in enumerate((per_ref.weighted_critic_loss(out, w, spec.weighted_loss), out["actor_loss"])):
            assert rel_scalar(float(L[j]), want) <= REL, (name, step, j, float(L[j]), want)
        for key, got in (("y", core.debug("y")), ("q1", core.debug("q1")), ("q2", core.debug("q2")),
                         ("a_next", core.debug("a_next")), ("a_cur", core.debug("a_cur")),
                         ("logp_next", core.debug("logp_next")), ("logp_cur", core.debug("logp_cur"))):
            ref = out[key].reshape(-1)
            err = float((got - ref).abs().max())
            assert err <= REL * (float(ref.abs().max()) + 1.0), (name, step, key, err)
        check_port_state(core, port)
    rb.close()
    core.close()


def test_priority_update_duplicates_and_root(cuda):
    """After a step the sampled leaves hold ((|y-Q1| + |y-Q2|)/2 + eps)^alpha of that step exactly; a duplicated index
    keeps the highest slot's value; every root equals the oracle tree's root over all leaves."""
    spec, care, precision = _spec("chained")
    core = _core(spec, care, precision)
    cap = 4096
    rb, _table = _filled_ring(core, spec, care, 3000, cap, prioritized=dict(alpha=0.7, beta=0.5, eps=1e-3))
    core.step_sampled(rb, 1)
    idx = core.debug("idx").long().numpy()
    want = per_ref.leaf_values(per_ref.td_priority(core.debug("y"), core.debug("q1"), core.debug("q2")), 0.7, 1e-3)
    assert np.array_equal(core.debug("prio").numpy(), want)
    last = {}
    for slot, k in enumerate(idx):         # duplicates: the highest slot's value
        last[k] = want[slot]
    keys = np.array(sorted(last))
    assert np.array_equal(rb.priorities(keys), np.array([last[k] for k in keys], dtype=np.float32))
    # a constructed duplicate through set_priorities: the later entry wins
    rb.set_priorities([7, 9, 7], [5.0, 1.0, 2.0])
    assert np.array_equal(rb.priorities([7, 9]), per_ref.leaf_values([2.0, 1.0], 0.7, 1e-3))
    leaves = rb.priorities(np.arange(cap))
    assert (leaves[3000:] == 0).all() and (leaves[:3000] > 0).all()
    assert rb.priorities([-1])[0] == per_ref.root(leaves)
    rb.close()
    core.close()


@pytest.mark.parametrize("T", [0, 4, 16])
def test_sampling_distribution_on_partly_filled_rings(cuda, T):
    """2000 draws of a 4096-slot ring, each sub-ring 15/16 filled, with skewed priorities, some of them zero: counts fit
    p_i/S (chi-square), no empty slot is drawn, each task gets B/T rows, and the weights equal (N p / S)^-beta over their
    batch maximum.  (A zero priority's leaf is (0 + eps)^alpha > 0: creation refuses an alpha, eps that round it to 0.)"""
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[32], critic_hidden=[32], batch=256, num_tasks=T)
    core = _core(spec, False, 1)
    cap, beta, eps = 4096, 0.7, 1e-6
    Tn = max(T, 1)
    cap_t = cap // Tn
    n = Tn * (cap_t * 15 // 16)                      # the last 1/16 of every sub-ring stays empty
    rb, _ = _filled_ring(core, spec, False, n, cap, prioritized=dict(alpha=2.0, beta=beta, eps=eps))
    i = np.arange(cap)
    filled = i % cap_t < n // Tn
    prio = ((i * 37) % 101 / 25.0).astype(np.float32)
    prio[i % 13 == 0] = 0.0                          # (0 + eps)^2 = 1e-12: rare, but a filled slot's leaf is > 0
    rb.set_priorities(i[filled], prio[filled])
    leaves = rb.priorities(i)
    assert (leaves[~filled] == 0).all() and (leaves[filled] > 0).all()
    assert (leaves[filled & (prio == 0)] == per_ref.leaf_values([0.0], 2.0, eps)[0]).all()
    roots = rb.priorities(-1 - np.arange(Tn))
    counts = np.zeros(cap, np.int64)
    per = spec.batch // Tn
    for k in range(2000):
        *_rows, idx, w = rb.sample_prioritized()
        idx = idx.numpy()
        counts += np.bincount(idx, minlength=cap)
        assert (np.bincount(idx // cap_t, minlength=Tn) == per).all()
        if k < 20:
            t = idx // cap_t
            want = per_ref.is_weights(leaves[idx], roots[t], n // Tn, beta)
            np.testing.assert_allclose(w.numpy(), want, rtol=1e-6)
    assert counts[~filled].sum() == 0
    for t in range(Tn):
        sl = slice(t * cap_t, (t + 1) * cap_t)
        lt = leaves[sl]
        pos = lt > 0
        f_exp = per_ref.sample_probabilities(lt)[pos] * counts[sl].sum()
        obs = counts[sl][pos]
        big = f_exp >= 5                              # slots too rare for their own bin share one
        res = stats.chisquare(np.append(obs[big], obs[~big].sum()), np.append(f_exp[big], f_exp[~big].sum()))
        assert big.sum() > pos.sum() // 2 and res.pvalue > 1e-3, (T, t, int(big.sum()), res)
    rb.close()
    core.close()


def test_push_and_fill_get_max_p(cuda):
    """Rows written by push -- new ones and ones overwritten on wrap-around -- read back the running max p;
    fill_synthetic leaves every filled leaf at max p = 1 and the rest empty."""
    from distributed_sac_b200.core import Replay
    spec, care, precision = _spec("chained")
    core = _core(spec, care, precision)
    cap = 2048
    rb, _ = _filled_ring(core, spec, care, 1500, cap, prioritized=dict(alpha=1.0, beta=0.5, eps=1e-6))
    assert (rb.priorities(np.arange(1500)) == 1.0).all() and (rb.priorities(np.arange(1500, cap)) == 0).all()
    rb.set_priorities([3, 4], [6.5, 2.0])             # max p is now 6.5 + 1e-6 in fp32
    mp = per_ref.leaf_values([6.5], 1.0, 1e-6)[0]
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=8, batch=1000)
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())   # slots 1500..2047, then 0..451 (wrap)
    got = rb.priorities(np.arange(cap))
    assert (got[1500:] == mp).all() and (got[:452] == mp).all() and (got[452:1500] == 1.0).all()
    assert rb.priorities([-1])[0] == per_ref.root(got)
    rb2 = Replay(core, cap, prioritized=PER)
    rb2.fill_synthetic(1000)
    got = rb2.priorities(np.arange(cap))
    assert (got[:1000] == 1.0).all() and (got[1000:] == 0).all()
    rb.close()
    rb2.close()
    core.close()


def test_multi_step_graphs_equal_single_steps(cuda):
    """step_sampled(rb, 50) (8-step graphs, the next draw forked after each priority update) == 50 calls of
    step_sampled(rb, 1): parameters, Adam moments and every priority, bit for bit."""
    spec, care, precision = _spec("chained")
    cores = [_core(spec, care, precision) for _ in range(2)]
    rings = [_filled_ring(c, spec, care, 4096, 4096)[0] for c in cores]
    cores[0].step_sampled(rings[0], 50)
    for _ in range(50):
        cores[1].step_sampled(rings[1], 1)
    for which in (0, 1, 2):
        assert torch.equal(cores[0].export_arena(which), cores[1].export_arena(which))
    all_idx = np.arange(4096)
    p0, p1 = rings[0].priorities(all_idx), rings[1].priorities(all_idx)
    assert np.array_equal(p0, p1) and len(np.unique(p0)) > 100
    for c, rb in zip(cores, rings):
        rb.close()
        c.close()


def test_replicas_have_their_own_trees(cuda):
    """R = 3: priorities set on replica 1 change neither replica 0's tree nor its draws."""
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[32], critic_hidden=[32], batch=64)
    cores = [_core(spec, False, 0, replicas=3) for _ in range(2)]
    rings = []
    for c in cores:
        from distributed_sac_b200.core import Replay
        rb = Replay(c, 1024, seed=4, prioritized=PER)
        for r in range(3):
            s, a, rew, s2, d = sp.synthetic_batch(spec, seed=r, batch=1024)
            rb.push(s.numpy(), a.numpy(), rew.numpy(), s2.numpy(), d.numpy(), replica=r)
            rb.set_priorities(np.arange(1024), np.arange(1024) % 17 + r, replica=r)
        rings.append(rb)
    rings[0].set_priorities(np.arange(512), np.full(512, 40.0), replica=1)
    assert not np.array_equal(rings[0].priorities(np.arange(1024), 1), rings[1].priorities(np.arange(1024), 1))
    assert np.array_equal(rings[0].priorities(np.arange(1024), 0), rings[1].priorities(np.arange(1024), 0))
    for _ in range(3):
        a0, a1 = rings[0].sample_prioritized(0), rings[1].sample_prioritized(0)
        assert torch.equal(a0[5], a1[5]) and torch.equal(a0[6], a1[6])
    b0, b1 = rings[0].sample_prioritized(1), rings[1].sample_prioritized(1)
    assert not torch.equal(b0[5], b1[5])
    for c, rb in zip(cores, rings):
        rb.close()
        c.close()


def test_set_beta_between_steps(cuda):
    """set_beta between two step_sampled calls changes the importance weights from the next step on (same graph)."""
    spec, care, precision = _spec("chained")
    core = _core(spec, care, precision)
    rb, _ = _filled_ring(core, spec, care, 4096, 4096, prioritized=dict(PER, beta=0.0))
    rb.set_priorities(np.arange(4096), np.arange(4096) % 50 / 7.0)
    core.prepare(rb)
    core.step_sampled(rb, 2)
    assert (core.debug("isw") == 1).all()
    rb.set_beta(1.0)
    core.step_sampled(rb, 1)
    w = core.debug("isw")
    assert float(w.max()) == 1.0 and float(w.min()) < 0.9
    rb.close()
    core.close()


def test_rejections(cuda):
    from distributed_sac_b200.core import Replay
    spec, care, precision = _spec("chained")
    core = _core(spec, care, precision)
    with pytest.raises(ValueError, match="device"):
        Replay(core, 4096, where="host", prioritized=PER)
    # (the last two: (0 + eps)^alpha rounds to 0 in fp32, so a sub-ring of zero priorities would have a zero root)
    for bad in (dict(PER, alpha=-0.1), dict(PER, beta=1.5), dict(PER, beta=-0.1), dict(PER, eps=0.0), dict(PER, eps=-1e-6),
                dict(alpha=2.0, beta=0.5, eps=1e-30), dict(alpha=9.0, beta=0.5, eps=1e-6)):
        with pytest.raises(RuntimeError, match="alpha|beta|eps"):
            Replay(core, 4096, prioritized=bad)
    Replay(core, 4096, prioritized=dict(alpha=2.0, beta=0.5, eps=1e-20)).close()     # 1e-40: a denormal, still > 0
    rb, _ = _filled_ring(core, spec, care, 1024, 1024)
    with pytest.raises(RuntimeError, match="_prioritized"):
        rb.sample()
    with pytest.raises(RuntimeError, match="beta"):
        rb.set_beta(2.0)
    with pytest.raises(RuntimeError, match="empty slot|outside"):
        rb.set_priorities([5000], [1.0])
    rb.close()
    rb, _ = _filled_ring(core, spec, care, 1024, 1024, prioritized=dict(alpha=2.0, beta=0.5, eps=1e-6))
    rb.set_priorities([3], [1e19])                    # 1e38: the largest leaf fp32 holds
    with pytest.raises(RuntimeError, match="overflows"):
        rb.set_priorities([3, 4], [1.0, 1e20])        # 1e40 would be an inf leaf (NaN weights); nothing is written
    assert rb.priorities([3, 4]).tolist() == [per_ref.leaf_values(np.float32([1e19]), 2.0, 1e-6)[0], 1.0]
    rb.close()
    core.close()
