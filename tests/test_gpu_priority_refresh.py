"""GPU: the priority refresh (b200sac_replay_refresh_priorities; include/b200sac.h).

  1  leaves against per_ref.leaf_values(td_priorities(...)) of oracle/refresh_ref.py at the parity bar, stochastic 0 and
     1 (the oracle reproducing the slot-keyed noise), on a single-task ring, an MT ring (per-task alpha, sub-rings) and a
     linked ring at horizon 3 (the fold); internal nodes bit-equal to per_ref.build_tree of the leaves read back;
  2  an idx subset leaves every other leaf bit for bit; max p follows the full-refresh and subset rules;
  3  a full refresh equals slot lists refreshed piece by piece, and does not depend on the replica count;
  4  after a critic reset, the refresh gives the oracle's leaves on the reset parameters, and the sampler's importance
     weights follow the new tree;
  5  every refusal leaves the tree bit for bit;
  6  learners: refresh_after_reset=True equals a reset followed by a refresh by hand; without it, a reset alone;
  7  the step's launch count and plan labels do not change.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import per_ref
import redis_stub
import refresh_ref as rr
import sac_port as sp
from _golden import core_config
from _harness import LEARNER_CFGS, plan_labels

pytestmark = pytest.mark.gpu

PARAMS = 0
PER = dict(alpha=0.6, beta=0.4, eps=1e-3)
BAR = 1e-4
SPEC = dict(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 48], batch=64)


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_sac_b200 import _lib
    _lib.load()
    return torch.device("cuda", 0)


def _params(spec, seed):
    p = sp.init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in p:
        if k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
        elif "_target." in k:
            p[k] = p[k] + 0.02 * torch.randn(p[k].shape, generator=g)
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


class Setup:
    """A handle with R replicas holding `params` in each, and a prioritized ring whose replicas hold the same rows: per
    task t, n_t rows pushed in order, so ring slot t * cap_t + k holds task t's k-th row.  linked: one trajectory per task
    (stream t), a terminal every 11th row."""

    def __init__(self, spec, replicas=1, cap=8192, fill=1500, linked=False, seed=0):
        from distributed_sac_b200.core import Replay, SacCore
        self.spec = spec
        self.core = SacCore(core_config(spec, replicas=replicas, precision=0), 0, seed=seed)
        self.params = _params(spec, 3 + seed)
        for r in range(replicas):
            self.core.set_named(self.params, PARAMS, replica=r)
        self.ring = Replay(self.core, cap, "device", seed=5, prioritized=PER, trajectories=linked)
        T = max(spec.num_tasks, 1)
        self.cap_t = cap // T
        g = np.random.default_rng(seed + 11)
        obs = spec.obs_dim
        s = np.zeros((cap, obs), np.float32)
        a = np.zeros((cap, spec.act_dim), np.float32)
        r_, s2 = np.zeros(cap, np.float32), np.zeros((cap, obs), np.float32)
        d = np.zeros(cap, np.float32)
        self.slots = []
        for t in range(T):
            k = np.arange(fill)
            sl = t * self.cap_t + k
            s[sl, :spec.state_dim] = g.standard_normal((fill, spec.state_dim))
            s2[sl, :spec.state_dim] = g.standard_normal((fill, spec.state_dim))
            if spec.num_tasks:
                s[sl, spec.state_dim + t] = 1
                s2[sl, spec.state_dim + t] = 1
            a[sl] = g.uniform(-1, 1, (fill, spec.act_dim))
            r_[sl] = g.standard_normal(fill)
            d[sl] = (k % 11 == 10) if linked else (g.random(fill) < 0.05)
            for rep in range(replicas):
                if linked:
                    self.ring.push(s[sl], a[sl], r_[sl, None], s2[sl], d[sl, None], replica=rep, stream=t)
                else:
                    self.ring.push(s[sl], a[sl], r_[sl, None], s2[sl], d[sl, None], replica=rep)
            self.slots.append(sl)
        self.slots = np.concatenate(self.slots)
        self.data = (s, a, r_, s2, d)
        self.T = T

    def link_table(self, replica=0):
        return np.concatenate([self.ring.links(t, replica) for t in range(self.T)]).astype(np.int64)

    def leaves(self, replica=0):
        return self.ring.priorities(self.slots, replica)

    def trees(self, replica=0):
        return [self.ring.tree(t, replica) for t in range(self.T)]

    def expect(self, slots, stochastic, seed, replica=0, n=1, params=None):
        link = self.link_table(replica) if self.ring.trajectories else None
        rows = rr.slot_rows(self.data, slots, self.cap_t, self.spec.gamma, link, n)
        eps = (rr.refresh_eps(seed, replica, slots, rows["task"], self.spec.act_dim) if stochastic
               else np.zeros((len(slots), self.spec.act_dim), np.float32))
        prio = rr.td_priorities(self.spec, params or self.params, rows, eps)[0]
        return per_ref.leaf_values(prio, PER["alpha"], PER["eps"])


def _check(got, ref, what):
    err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= BAR, f"{what}: max error {err:.3g} over the parity bar"


def _check_trees(st, replica=0):
    for t, tree in enumerate(st.trees(replica)):
        P = len(tree) // 2
        np.testing.assert_array_equal(tree, per_ref.build_tree(tree[P:]), err_msg=f"task {t}")


@pytest.mark.parametrize("stochastic", [False, True])
@pytest.mark.parametrize("kind", ["single", "mt", "linked"])
def test_full_refresh_matches_the_oracle(cuda, kind, stochastic):
    spec = sp.SacSpec(**SPEC, num_tasks=4 if kind == "mt" else 0)
    st = Setup(spec, linked=kind == "linked")
    n = 1
    if kind == "linked":
        st.ring.set_nstep(3)
        n = 3
    st.ring.refresh_priorities(77, stochastic=stochastic)
    _check(st.leaves(), st.expect(st.slots, stochastic, 77, n=n), f"{kind} stochastic={stochastic}")
    _check_trees(st)
    # max p: the largest refreshed leaf of each task, which the next pushed row gets
    leaves = st.leaves()
    for t in range(st.T):
        top = leaves[st.slots // st.cap_t == t].max()
        spec_s = np.zeros((1, spec.obs_dim), np.float32)
        if spec.num_tasks:
            spec_s[0, spec.state_dim + t] = 1
        st.ring.push(spec_s, np.zeros((1, spec.act_dim), np.float32), np.zeros((1, 1), np.float32), spec_s,
                     np.zeros((1, 1), np.float32))
        fill = len(st.slots) // st.T
        assert st.ring.priorities([t * st.cap_t + fill])[0] == top


def test_subset_refresh(cuda):
    spec = sp.SacSpec(**SPEC, num_tasks=2)
    st = Setup(spec)
    rng = np.random.default_rng(3)
    st.ring.set_priorities(st.slots, rng.uniform(0, 0.01, len(st.slots)).astype(np.float32))   # low leaves, max p 1
    before = st.leaves()
    sub = rng.choice(st.slots, 300, replace=False)
    sub = np.concatenate([sub, sub[:20]])                # duplicates are harmless
    st.ring.refresh_priorities(5, idx=sub, replica=0)
    after = st.leaves()
    hit = np.isin(st.slots, sub)
    np.testing.assert_array_equal(after[~hit], before[~hit])
    pos = {k: i for i, k in enumerate(st.slots)}
    _check(after[[pos[k] for k in sub]], st.expect(sub, True, 5), "subset")
    _check_trees(st)
    # max p is only raised: it stays 1 unless a refreshed leaf is larger
    fill = len(st.slots) // st.T
    for t in range(st.T):
        s = np.zeros((1, spec.obs_dim), np.float32)
        s[0, spec.state_dim + t] = 1
        st.ring.push(s, np.zeros((1, spec.act_dim), np.float32), np.zeros((1, 1), np.float32), s, np.zeros((1, 1), np.float32))
        top = after[np.isin(st.slots, sub) & (st.slots // st.cap_t == t)].max()
        assert st.ring.priorities([t * st.cap_t + fill])[0] == max(np.float32(1.0), top)


def test_pieces_and_replica_count(cuda):
    spec = sp.SacSpec(**SPEC, num_tasks=2)
    one, three = Setup(spec), Setup(spec, replicas=3)
    one.ring.refresh_priorities(9)
    full = one.leaves()
    pieces = Setup(spec)
    perm = np.random.default_rng(0).permutation(pieces.slots)
    for part in np.array_split(perm, 5):
        pieces.ring.refresh_priorities(9, idx=part, replica=0)
    np.testing.assert_array_equal(pieces.leaves(), full)
    three.ring.refresh_priorities(9)
    np.testing.assert_array_equal(three.leaves(0), full)
    for a, b in zip(three.trees(0), one.trees(0)):
        np.testing.assert_array_equal(a, b)
    # replica 1's key differs; with the mean action it holds replica 0's values
    one.ring.refresh_priorities(9, stochastic=False)
    three.ring.refresh_priorities(9, stochastic=False)
    np.testing.assert_array_equal(three.leaves(1), one.leaves(0))


def test_refresh_after_a_critic_reset(cuda):
    spec = sp.SacSpec(**SPEC)
    st = Setup(spec)
    st.ring.refresh_priorities(1)
    st.core.reset(123, critic="all")
    st.ring.refresh_priorities(2)
    named = st.core.get_named()
    params = {k: v.reshape(st.params[k].shape) for k, v in named.items() if k in st.params}
    _check(st.leaves(), st.expect(st.slots, True, 2, params=params), "after reset")
    _check_trees(st)
    tree = st.trees()[0]
    P = len(tree) // 2
    s, a, r, s2, d, idx, w = st.ring.sample_prioritized()
    want = per_ref.is_weights(tree[P + idx.numpy()], tree[1], len(st.slots), PER["beta"])
    np.testing.assert_allclose(w.numpy(), want, rtol=1e-6)


def test_refusals_leave_the_tree(cuda):
    from distributed_sac_b200.core import Replay
    spec = sp.SacSpec(**SPEC)
    st = Setup(spec, fill=600)
    st.ring.refresh_priorities(1)
    before = st.trees()
    lib, h = st.core.lib, st.ring._h
    idx = np.array([0, 5, 3000], np.int64)
    good = np.array([1], np.int64)
    ptr = lambda x: C.c_void_p(x.ctypes.data)
    calls = [(5, 1, good, 1), (0, -1, good, 1), (0, 1, None, 1), (0, 3, idx, 1), (0, 1, good, 2)]
    for rep, n, ix, stoch in calls:
        rc = lib.b200sac_replay_refresh_priorities(h, rep, n, None if ix is None else ptr(ix), C.c_uint64(3), stoch, None)
        assert rc == -1, (rep, n, stoch)
        for x, y in zip(st.trees(), before):
            np.testing.assert_array_equal(x, y)
    plain = Replay(st.core, 1024, "device", seed=1)
    plain.fill_synthetic(512)
    assert lib.b200sac_replay_refresh_priorities(plain._h, 0, 0, None, C.c_uint64(3), 1, None) == -1


def _learner(tmp_path, tag, **kw):
    from distributed_sac_b200 import learner as L
    p = tmp_path / "ll.json"
    p.write_text(json.dumps(LEARNER_CFGS["LL"]))
    os.chdir(tmp_path)
    lrn = L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=f"{tmp_path}/{tag}"), seed=3,
                               replay_where="device", **kw)
    lrn.memory.ring.fill_synthetic(5000, seed=1)
    return lrn


def _tree(lrn):
    return lrn.memory.ring.tree(0)


def test_learners(cuda, tmp_path):
    a = _learner(tmp_path, "a", prioritized=dict(PER, refresh_after_reset=True), reset_interval=5)
    b = _learner(tmp_path, "b", prioritized=dict(PER))
    c = _learner(tmp_path, "c", prioritized=dict(PER), reset_interval=5)
    d = _learner(tmp_path, "d", prioritized=dict(PER))
    for x in (a, b, c, d):
        x.update_many(5)
    for x in (a, b, c, d):
        np.testing.assert_array_equal(_tree(x), _tree(a))
    a.update_many(1)                        # reset 1, its refresh, update 6
    c.update_many(1)
    seed = 3 + 2 ** 32
    for x, refresh in ((b, True), (d, False)):
        x.core.reset(seed)
        if refresh:
            x.memory.ring.refresh_priorities(seed)
        x.update_many(1)
    np.testing.assert_array_equal(_tree(a), _tree(b))
    np.testing.assert_array_equal(_tree(c), _tree(d))
    assert not np.array_equal(_tree(a), _tree(c))
    for w in (0, 1, 2):
        assert torch.equal(a.core.export_arena(w), b.core.export_arena(w))
    q1, q2 = a.q_values(torch.zeros(3, 8), torch.zeros(3, 2))
    assert q1.shape == (3, 1) and q2.shape == (3, 1)
    for x in (a, b, c, d):
        x.memory.stop()


def test_plan_unchanged(cuda):
    spec = sp.SacSpec(**SPEC)
    st, ref = Setup(spec), Setup(spec)
    n = st.core.launches_per_step
    st.ring.refresh_priorities(4)
    st.core.critic_values(torch.zeros(5, 8), torch.zeros(5, 2))
    got = C.c_int32(0)
    st.core.lib.b200sac_launches_per_step(st.core._h, C.byref(got))
    assert got.value == n
    assert plan_labels(st.core) == plan_labels(ref.core)
