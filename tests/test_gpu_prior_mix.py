"""GPU: prior-data rings (b200sac_replay_attach_prior, RLPD's symmetric sampling).  A ring with a prior attached draws rows
[tP, tP + m) of every task block from the prior and the rest from itself, inside the step's graph.

Every transition pushed here carries a reward of its own, so debug "r" names the rows a step trained on.  A host model of
each ring (per-task sub-rings at t * cap_t + k mod cap_t, the newest cap_t rows surviving a wrap) says which transition
each slot holds; oracle/mix_ref.py says which slots a step draws.  The in-kernel Philox noise is keyed by (seed, replica,
step counter), so a handle with the same seed running b200sac_step on the predicted rows must equal every mixed step bit
for bit.
"""
import dataclasses
import json
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mix_ref
import redis_stub
import sac_port as sp
from _golden import core_config
from _harness import VS400, _core, _tasks, care_t4, cuda

pytestmark = pytest.mark.gpu

_REWARDS = np.random.default_rng(2027).permutation(np.linspace(-3.0, 3.0, 1 << 21)).astype(np.float32)
_SMALL = dict(act_dim=3, actor_hidden=[64, 48], critic_hidden=[56, 64])
INVALID, STATE = -1, -4

# id -> (spec, care, precision, replicas)
SHAPES = {
    "ll_chained": (sp.ll_spec(), False, 0, 1),
    "vs_p0": (sp.SacSpec(**VS400), False, 0, 1),
    "vs_p1": (sp.SacSpec(**VS400), False, 1, 1),
    "ms_t10": (sp.SacSpec(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=130, num_tasks=10,
                          weighted_loss=True), False, 1, 1),
    "care_m": (care_t4(), True, 1, 1),
    "r3": (sp.SacSpec(state_dim=9, num_tasks=3, batch=99, **_SMALL), False, 0, 3),
}


def _per(spec):
    return spec.batch // max(spec.num_tasks, 1)


def _mixed_m(spec, R):
    """Prior rows per replica for the 0 < m < P cases: different on every replica."""
    P = _per(spec)
    return [P // 2] if R == 1 else [1, P // 2, P - 1][:R]


class Source:
    """Transitions with distinct rewards; d = 1 on about a third of them; the task of each row is given."""

    def __init__(self, spec, seed=0):
        self.spec, self.g = spec, torch.Generator().manual_seed(seed)

    k = 0                                  # shared by every Source: rewards stay distinct across rings

    def take(self, tasks):
        spec, g, n = self.spec, self.g, len(tasks)
        s = torch.randn(n, spec.state_dim, generator=g)
        a = torch.rand(n, spec.act_dim, generator=g) * 2 - 1
        s2 = torch.randn(n, spec.state_dim, generator=g)
        d = (torch.rand(n, 1, generator=g) < 1 / 3).float()
        r = torch.from_numpy(_REWARDS[Source.k:Source.k + n].copy()).reshape(n, 1)
        Source.k = (Source.k + n) % (len(_REWARDS) - (1 << 16))
        if spec.num_tasks > 0:
            oh = F.one_hot(torch.as_tensor(tasks, dtype=torch.long), spec.num_tasks).float()
            s, s2 = torch.cat([s, oh], 1), torch.cat([s2, oh], 1)
        return s, a, r, s2, d


def _tasks_of(counts, seed):
    return np.random.default_rng(seed).permutation(np.repeat(np.arange(len(counts)), counts))


class Ring:
    """Device rings of one or more handles, all pushed the same rows, and the host model of each (replica, slot)."""

    def __init__(self, cores, spec, cap, seed):
        from distributed_sac_b200.core import Replay
        self.rbs = [Replay(c, cap, "device", seed=seed) for c in cores]
        self.spec, self.seed, R = spec, seed, cores[0].cfg.replicas
        self.T = max(spec.num_tasks, 1)
        self.cap_t = cap // self.T
        self.head = np.zeros((R, self.T), np.int64)
        self.fill = np.zeros((R, self.T), np.int64)
        self.held = [dict() for _ in range(R)]      # ring slot -> row of `table`
        self.table = None

    def push(self, batch, replica=0):
        for rb in self.rbs:
            rb.push(*(x.numpy() for x in batch), replica=replica)
        base = 0 if self.table is None else self.table[0].shape[0]
        self.table = list(batch) if self.table is None else [torch.cat([t, x]) for t, x in zip(self.table, batch)]
        tid = _tasks(self.spec, batch[0])
        for t in range(self.T):
            for i in np.nonzero(tid == t)[0][-self.cap_t:]:
                self.held[replica][t * self.cap_t + int(self.head[replica, t])] = base + i
                self.head[replica, t] = (self.head[replica, t] + 1) % self.cap_t
                self.fill[replica, t] = min(self.fill[replica, t] + 1, self.cap_t)

    def fill_per_task(self, src, per_task, replica=0, seed=0):
        self.push(src.take(_tasks_of(per_task, seed)), replica)

    def spec_of(self, replica):
        return mix_ref.Ring(self.seed, self.fill[replica].tolist(), self.cap_t)

    def close(self):
        for rb in self.rbs:
            rb.close()


def predict(step, replica, B, T, m, online, prior):
    """(encoded indices, the 5 row tensors) of one step of one replica."""
    idx = mix_ref.draw(step, replica, B, T, m, online.spec_of(replica), None if prior is None else prior.spec_of(replica))
    is_p, k = mix_ref.decode(idx)
    src = [(prior if p else online, (prior if p else online).held[replica][int(x)]) for p, x in zip(is_p, k)]
    return idx, [torch.stack([ring.table[f][row] for ring, row in src]) for f in range(5)]


class Follower:
    """A same-seed handle that runs b200sac_step on the predicted rows of every step of the mixed handle."""

    def __init__(self, spec, care, precision, R, seed):
        self.core, self.spec, self.R, self.step = _core(spec, care, precision, R, seed=seed), spec, R, 0

    def run(self, online, prior, ms, n=1, core=None):
        """n steps with prior rows ms[r]; with `core`, the mixed handle's last step is checked slot by slot."""
        B, T = self.spec.batch, self.spec.num_tasks
        for j in range(n):
            per_rep = [predict(self.step, r, B, T, ms[r], online, prior) for r in range(self.R)]
            self.core.step(*[torch.stack([p[1][f] for p in per_rep]) for f in range(5)])
            self.step += 1
        if core is not None:
            for r, (idx, rows) in enumerate(per_rep):
                if prior is not None:
                    got = core.debug("idx", r).numpy()
                    assert np.array_equal(got, idx), f"replica {r}: the device draw is not mix_ref's"
                assert torch.equal(core.debug("r", r), rows[2][:, 0]), f"replica {r}: the step did not train on the drawn rows"
                assert torch.equal(core.debug("d", r), rows[4][:, 0])


def assert_identical(cores, n_steps, names):
    from distributed_sac_b200 import _lib
    ref = cores[0]
    for c, name in zip(cores[1:], names[1:]):
        for rep in range(ref.cfg.replicas):
            for which in (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V):
                assert torch.equal(c.export_arena(which, rep), ref.export_arena(which, rep)), (names[0], name, rep, which)
            assert c.get_steps(rep) == ref.get_steps(rep), (names[0], name, rep)
        assert torch.equal(c.read_losses(n_steps), ref.read_losses(n_steps)), (names[0], name)


def _rings(cores, spec, R, seed_on=1, seed_pr=2, pr_cores=None):
    """An online ring (capacity 8 P per task, filled 5-7 P per task) and a prior ring (6 P per task, filled 4-6 P)."""
    T, P = max(spec.num_tasks, 1), _per(spec)
    on = Ring(cores, spec, 8 * P * T, seed_on)
    pr = Ring(cores if pr_cores is None else pr_cores, spec, 6 * P * T, seed_pr)
    src = Source(spec, seed=seed_on * 31 + seed_pr)
    for r in range(R):
        on.fill_per_task(src, [P * (5 + (t + r) % 3) for t in range(T)], r, seed=10 + r)
        pr.fill_per_task(src, [P * (4 + (t + 2 * r) % 3) for t in range(T)], r, seed=20 + r)
    return on, pr, src


def _rc(call):
    try:
        call()
    except RuntimeError as e:
        return int(str(e).split("b200sac error ")[1].split(":")[0])
    return 0


# ---------------------------------------------------------------------------------------------------------------------
# 1, 2: m = 0 is the plain ring; m = P is a plain ring with the prior's seed and rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_zero_prior_rows_equal_a_never_attached_ring(cuda, name):
    """Attached with m = 0 (prepared graphs) against a never-attached twin (graphs built on use): 1-step calls and
    8/4/2/1-step graphs, bit for bit."""
    spec, care, precision, R = SHAPES[name]
    a, b = (_core(spec, care, precision, R, seed=3) for _ in range(2))
    on, pr, _ = _rings([a, b], spec, R)
    on.rbs[0].attach_prior(pr.rbs[0])
    a.prepare(on.rbs[0])
    n = 0
    for k in (1, 1, 15, 16, 3):
        a.step_sampled(on.rbs[0], k)
        b.step_sampled(on.rbs[1], k)
        n += k
        for r in range(R):
            assert torch.equal(a.debug("r", r), b.debug("r", r))
            assert (a.debug("idx", r) >= 0).all()
    assert_identical([b, a], n, ["never attached", "attached, m = 0"])
    on.close()
    pr.close()


@pytest.mark.parametrize("name", ["ll_chained", "ms_t10", "r3"])
def test_all_prior_rows_equal_a_plain_ring_of_the_prior(cuda, name):
    """m = P with a prior of seed 9 == a plain ring of seed 9 with the same pushes, bit for bit."""
    spec, care, precision, R = SHAPES[name]
    a, b = (_core(spec, care, precision, R, seed=3) for _ in range(2))
    on, pr, _ = _rings([a], spec, R, seed_on=1, seed_pr=9, pr_cores=[a, b])
    on.rbs[0].attach_prior(pr.rbs[0])
    on.rbs[0].set_prior_rows(_per(spec))
    n = 0
    for k in (1, 15, 3):
        a.step_sampled(on.rbs[0], k)
        b.step_sampled(pr.rbs[1], k)
        n += k
    for r in range(R):
        assert torch.equal(a.debug("r", r), b.debug("r", r))
        assert (a.debug("idx", r) < 0).all()
    assert_identical([b, a], n, ["plain ring of the prior", "m = P"])
    on.close()
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3, 4: 0 < m < P against mix_ref and b200sac_step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_mixed_steps_match_mix_ref_and_b200sac_step(cuda, name):
    spec, care, precision, R = SHAPES[name]
    a = _core(spec, care, precision, R, seed=3)
    f = Follower(spec, care, precision, R, seed=3)
    on, pr, _ = _rings([a], spec, R)
    on.rbs[0].attach_prior(pr.rbs[0])
    ms = _mixed_m(spec, R)
    for r, m in enumerate(ms):
        on.rbs[0].set_prior_rows(m, replica=r)
        assert on.rbs[0].get_prior_rows(r) == m
    B, T, P = spec.batch, max(spec.num_tasks, 1), _per(spec)
    for k in range(5):
        a.step_sampled(on.rbs[0], 1)
        f.run(on, pr, ms, 1, core=a)
        for r in range(R):                      # distinct within each part of each block; prior indices name filled slots
            is_p, idx = mix_ref.decode(a.debug("idx", r).numpy())
            t = np.arange(B) // P
            assert (is_p == (np.arange(B) % P < ms[r])).all()
            for tt in range(T):
                for part in (True, False):
                    sel = (t == tt) & (is_p == part)
                    assert len(set(idx[sel].tolist())) == sel.sum()
            assert all(int(x) in pr.held[r] for x in idx[is_p])
    for k in (8, 4, 2, 1, 15):
        a.step_sampled(on.rbs[0], k)
        f.run(on, pr, ms, k, core=a)
    assert_identical([f.core, a], f.step, ["b200sac_step on mix_ref's rows", "mixed sampled steps"])
    on.close()
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5, 6: stream order of set_prior_rows; a push into the prior after steps were enqueued
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["side", "legacy"])
def test_set_prior_rows_changes_only_later_steps(cuda, where):
    spec = sp.SacSpec(state_dim=8, batch=64, **_SMALL)
    R = 2
    a = _core(spec, False, 0, R, seed=5)
    f = Follower(spec, False, 0, R, seed=5)
    on, pr, _ = _rings([a], spec, R)
    rb = on.rbs[0]
    rb.attach_prior(pr.rbs[0])
    a.prepare(rb)
    st = torch.cuda.Stream() if where == "side" else torch.cuda.default_stream()
    schedule = [(None, 3), ([10, 40], 5), ([64, 40], 1), ([0, 0], 2), ([33, 1], 8)]
    ms = [0, 0]
    with torch.cuda.stream(st):
        for new, n in schedule:
            if new is not None:
                for r, m in enumerate(new):
                    rb.set_prior_rows(m, replica=r)
                ms = new
            a.step_sampled(rb, n)
            f.run(on, pr, ms, n)
    st.synchronize()
    assert [rb.get_prior_rows(r) for r in range(R)] == ms
    assert_identical([f.core, a], f.step, ["b200sac_step", f"set_prior_rows on the {where} stream"])
    on.close()
    pr.close()


def test_push_into_the_prior_waits_for_enqueued_steps(cuda):
    spec = sp.SacSpec(state_dim=8, num_tasks=2, batch=64, **_SMALL)
    a = _core(spec, False, 0, 1, seed=6)
    f = Follower(spec, False, 0, 1, seed=6)
    on, pr, src = _rings([a], spec, 1)
    on.rbs[0].attach_prior(pr.rbs[0])
    on.rbs[0].set_prior_rows(20)
    f.run(on, pr, [20], 8)                     # predicted from the prior as it is before the push
    a.step_sampled(on.rbs[0], 8)
    pr.fill_per_task(src, [pr.cap_t, pr.cap_t], 0, seed=99)      # overwrites every slot of the prior
    a.step_sampled(on.rbs[0], 4)
    f.run(on, pr, [20], 4, core=a)
    assert_identical([f.core, a], 12, ["b200sac_step", "steps around a push into the prior"])
    on.close()
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7: detach, explicit or by destroying either ring
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["explicit", "destroy_prior", "destroy_online"])
def test_detach(cuda, how):
    spec = sp.SacSpec(state_dim=8, num_tasks=3, batch=99, **_SMALL)
    a = _core(spec, False, 0, 1, seed=7)
    f = Follower(spec, False, 0, 1, seed=7)
    on, pr, _ = _rings([a], spec, 1)
    on.rbs[0].attach_prior(pr.rbs[0])
    on.rbs[0].set_prior_rows(12)
    a.prepare(on.rbs[0])
    a.step_sampled(on.rbs[0], 3)
    f.run(on, pr, [12], 3, core=a)
    if how == "destroy_online":                # the prior is an ordinary ring afterwards
        on.close()
        a.step_sampled(pr.rbs[0], 6)
        f.run(pr, None, [0], 6, core=a)
    else:
        if how == "explicit":
            on.rbs[0].attach_prior(None)
        else:
            pr.close()
        assert on.rbs[0].get_prior_rows(0) == 0
        assert _rc(lambda: on.rbs[0].set_prior_rows(1)) == STATE
        a.step_sampled(on.rbs[0], 1)
        a.step_sampled(on.rbs[0], 5)
        f.run(on, None, [0], 6, core=a)
        with pytest.raises(RuntimeError):      # "idx" of a plain uniform ring: as before, no such buffer
            a.debug("idx")
    assert_identical([f.core, a], 9, ["b200sac_step", f"detached ({how})"])
    on.close()
    pr.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8: refusals, with nothing enqueued
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals(cuda):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import Replay
    spec = sp.SacSpec(state_dim=8, num_tasks=2, batch=64, **_SMALL)
    R, P = 2, 32
    h, other = _core(spec, False, 0, R, seed=8), _core(spec, False, 0, R, seed=8)
    u1, u2, u3 = (Replay(h, 8 * 64, "device", seed=s) for s in (1, 2, 3))
    per = Replay(h, 8 * 64, "device", seed=4, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6))
    linked = Replay(h, 8 * 64, "device", seed=5, trajectories=True)
    host = Replay(h, 8 * 64, "host", seed=6)
    foreign = Replay(other, 8 * 64, "device", seed=7)
    lib = h.lib
    attach = lambda x, y: _lib.check(lib.b200sac_replay_attach_prior(x._h, None if y is None else y._h))
    for x, y in [(u1, per), (per, u1), (u1, linked), (linked, u1), (u1, host), (host, u1), (u1, foreign), (u1, u1)]:
        assert _rc(lambda: attach(x, y)) == INVALID
    assert _rc(lambda: u1.set_prior_rows(1)) == STATE          # no prior yet
    attach(u1, u2)
    assert _rc(lambda: attach(u1, u3)) == STATE                # u1 has a prior
    assert _rc(lambda: attach(u3, u2)) == STATE                # u2 is u1's prior
    assert _rc(lambda: attach(u3, u1)) == STATE                # u1 has a prior itself
    for x in (u1, u2):
        assert _rc(lambda: _lib.check(lib.b200sac_replay_enable_trajectories(x._h))) == STATE
    for m, r in [(-1, 0), (P + 1, 0), (1, R), (1, -1)]:
        assert _rc(lambda: u1.set_prior_rows(m, replica=r)) == INVALID
    assert [u1.get_prior_rows(r) for r in range(R)] == [0, 0]
    src = Source(spec, seed=3)
    for r in range(R):
        for rb in (u1, u2):
            rb.push(*(t.numpy() for t in src.take(_tasks_of([4 * P, 4 * P - (rb is u2) * (r == 1)], 5 + r))), replica=r)
    u1.set_prior_rows(1, replica=0)            # replica 0's prior sub-rings are ready
    a0 = [h.export_arena(_lib.PARAMS, r).clone() for r in range(R)]
    h.step_sampled(u1, 1)
    u1.set_prior_rows(5, replica=1)            # replica 1's prior task 1 holds 4P - 1 rows
    for call in (lambda: h.step_sampled(u1, 3), lambda: h.update_sampled(u1), lambda: h.prepare(u1) or h.step_sampled(u1, 1),
                 lambda: h.profile_step(u1, 1), lambda: h.graph_timeline(u1, 2)):
        assert _rc(call) == STATE
    torch.cuda.synchronize()
    assert [h.get_steps(r)[0] for r in range(R)] == [1, 1]
    u1.set_prior_rows(0, replica=1)
    h.step_sampled(u1, 2)
    assert [h.get_steps(r)[0] for r in range(R)] == [3, 3]
    assert not torch.equal(h.export_arena(_lib.PARAMS, 0), a0[0])
    for rb in (u1, u2, u3, per, linked, host, foreign):
        rb.close()
    h.close()
    other.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9: task blocks under pcgrad, launch count and labels
# ---------------------------------------------------------------------------------------------------------------------
def test_pcgrad_task_blocks_launches_and_labels(cuda):
    spec = sp.SacSpec(state_dim=12, act_dim=3, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=60, num_tasks=3)
    from distributed_sac_b200.core import SacCore
    core = SacCore(dataclasses.replace(core_config(spec, precision=1), pcgrad=True), 0, seed=1)
    n0 = core.launches_per_step
    on, pr, _ = _rings([core], spec, 1)
    plain = [n for n, _ in core.profile_step(on.rbs[0], 1)]
    tl_plain = len(core.graph_timeline(on.rbs[0], 2))
    on.rbs[0].attach_prior(pr.rbs[0])
    on.rbs[0].set_prior_rows(7)
    for n in (1, 8, 3):
        core.step_sampled(on.rbs[0], n)
        assert core.read_pcgrad(0)["task_mismatch"] == 0
    labels = [n for n, _ in core.profile_step(on.rbs[0], 2)]
    assert labels[0] == "sample_mixed+ingest_mixed" and plain[0] == "sample+ingest" and labels[1:] == plain[1:]
    assert core.launches_per_step == n0
    assert len(core.graph_timeline(on.rbs[0], 2)) == tl_plain
    assert (core.debug("idx") < 0).sum() == 3 * 7
    on.close()
    pr.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 10: learners
# ---------------------------------------------------------------------------------------------------------------------
_MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
           "log_alpha": 0, "start_memory_len": 100, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
           "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
           "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}
_LL_CFG = {"device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "lr_actor": 3e-4,
           "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 100}


@pytest.mark.parametrize("family", ["LL", "MS"])
def test_learner_prior(cuda, tmp_path, family):
    from distributed_sac_b200 import learner as L
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(_LL_CFG if family == "LL" else _MS_CFG))
    kw = dict(write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + family), replay_where="device",
              prior=dict(capacity=2048, fraction=0.5))
    lrn = L.LunarLanderLearner(str(p), **kw) if family == "LL" else L.MTSACLearner(None, ["t0", "t1", "t2"], str(p), **kw)
    try:
        T, B = max(lrn.num_tasks, 1), lrn.batch_size
        P = B // T
        assert lrn.memory.ring.get_prior_rows() == math.floor(0.5 * P + 0.5)
        spec = sp.SacSpec(state_dim=lrn.state_dim, act_dim=lrn.action_dim, num_tasks=lrn.num_tasks)
        src = Source(spec, seed=4)
        s, a, r, s2, d = src.take(_tasks_of([8 * P] * T, 1))
        lrn.memory.add_many(s.numpy(), a.numpy(), r.numpy()[:, 0], s2.numpy(), d.numpy()[:, 0])
        assert not lrn.memory.prior_ready()
        s, a, r, s2, d = src.take(_tasks_of([5 * P] * T, 2))
        lrn.push_prior(s.numpy(), a.numpy(), r.numpy()[:, 0], s2.numpy(), d.numpy()[:, 0])
        assert lrn.memory.prior_ready()
        out = lrn.update()
        assert all(math.isfinite(x) for x in out)
        assert (lrn.core.debug("idx") < 0).sum() == T * math.floor(0.5 * P + 0.5)
        L20 = lrn.update_many(20)
        assert L20.shape[0] == 20 and torch.isfinite(L20).all()
        lrn.set_prior_fraction(0.0)
        assert lrn.memory.ring.get_prior_rows() == 0
        lrn.update()
        assert (lrn.core.debug("idx") >= 0).all()
    finally:
        lrn.memory.stop()
        lrn.core.close()
