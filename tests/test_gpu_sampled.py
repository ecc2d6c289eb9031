"""GPU: the sampled step (b200sac_step_sampled / b200sac_update), the path Learner.update() and bench.py run, against
b200sac_step on the same minibatches and against the autograd oracle.

Every ring here is filled with `push` and every transition pushed in a test carries a reward of its own (a shuffled linspace),
so the rewards a step ingested (debug "r") name the exact ring rows it trained on.  A host model of the ring (per-task
sub-rings at t * cap_t + k mod cap_t, the newest cap_t rows surviving a wrap) says which transition each slot holds, and
about a third of the rows have d = 1, so that a lost or misplaced done flag changes the result.  The in-kernel Philox
noise is keyed by (seed, replica, step counter): a handle with the same seed that runs b200sac_step on the recovered rows
(no injected noise) draws the same noise, and every sampled step must equal it bit for bit.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import stats

import care_port as cp
import sac_port as sp
from _golden import REL, check_forced, check_port_state, cuda_relu_masks, rel_l2, rel_scalar, sync_core_to_port
from _harness import VS400, _core, _tasks, care_t4, check_active, cuda, plan_labels

pytestmark = pytest.mark.gpu

# distinct float32 rewards (the spacing 6 / 2^21 is 12 float32 ulps at |r| = 3)
_REWARDS = np.random.default_rng(2026).permutation(np.linspace(-3.0, 3.0, 1 << 21)).astype(np.float32)

_SMALL = dict(act_dim=3, actor_hidden=[64, 48], critic_hidden=[56, 64])


# id -> (spec, care, precision, replicas, plan)
SHAPES = {
    "ll_chained": (sp.ll_spec(), False, 0, 1, "chained"),
    "odd37_chained": (sp.SacSpec(state_dim=8, batch=37, **_SMALL), False, 0, 1, "chained"),
    "layer_p0": (sp.SacSpec(**VS400), False, 0, 1, "per_layer"),
    "layer_p1": (sp.SacSpec(**VS400), False, 1, 1, "wgmma"),
    "mtsac_t10": (sp.SacSpec(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=130, num_tasks=10,
                             weighted_loss=True), False, 1, 1, "wgmma"),
    "care_m": (care_t4(), True, 1, 1, "care"),       # batch 120 = 4 x 30
    "care_o": (care_t4(False), True, 0, 1, "care"),
    "r3_wrapped": (sp.SacSpec(state_dim=9, num_tasks=3, batch=99, **_SMALL), False, 0, 3, "chained"),
}


def check_plan(spec, care, precision, replicas, plan):
    """A throwaway handle of the same configuration runs the plan the case is meant to cover (labels of one eager step)."""
    core = _core(spec, care, precision, replicas)
    labels = plan_labels(core)
    core.close()
    chained = any(n.startswith("chain_fwd") for n in labels)
    wgmma = any("wgmma" in n for n in labels)
    want = dict(chained=chained and not wgmma, per_layer=not chained and not wgmma and "care_tables" not in labels,
                wgmma=not chained and wgmma and "care_tables" not in labels, care="care_tables" in labels)[plan]
    assert want, f"expected the {plan} plan, got {labels}"


def _shuffled_tasks(counts, seed):
    """Task ids holding counts[t] rows of task t, shuffled."""
    t = np.repeat(np.arange(len(counts)), counts)
    return np.random.default_rng(seed).permutation(t)


class Source:
    """Transitions with distinct rewards; d = 1 on about a third of them; the task of each row is given."""

    def __init__(self, spec, seed=0):
        self.spec, self.g, self.k = spec, torch.Generator().manual_seed(seed), 0

    def take(self, tasks):
        spec, g, n = self.spec, self.g, len(tasks)
        s = torch.randn(n, spec.state_dim, generator=g)
        a = torch.rand(n, spec.act_dim, generator=g) * 2 - 1
        s2 = torch.randn(n, spec.state_dim, generator=g)
        d = (torch.rand(n, 1, generator=g) < 1 / 3).float()
        r = torch.from_numpy(_REWARDS[self.k:self.k + n].copy()).reshape(n, 1)
        self.k += n
        if spec.num_tasks > 0:
            oh = F.one_hot(torch.as_tensor(tasks, dtype=torch.long), spec.num_tasks).float()
            s, s2 = torch.cat([s, oh], 1), torch.cat([s2, oh], 1)
        return s, a, r, s2, d


class Ring:
    """Replay rings of one or more twin handles, all pushed the same rows, and the host model of which transition each
    (replica, ring slot) holds."""

    def __init__(self, cores, spec, cap, where="device", seed=1):
        from distributed_sac_b200.core import Replay
        self.rbs = [Replay(c, cap, where, seed=seed) for c in cores]
        self.spec, R = spec, cores[0].cfg.replicas
        self.T = max(spec.num_tasks, 1)
        self.cap_t = cap // self.T
        self.head = np.zeros((R, self.T), np.int64)
        self.fill = np.zeros((R, self.T), np.int64)
        self.slot = [dict() for _ in range(R)]      # reward -> ring slot, for the rows a replica's ring holds now
        self.held = [dict() for _ in range(R)]      # ring slot -> reward
        self.index = {}                              # reward -> row of `table` (every transition ever pushed)
        self.table = None

    def push(self, batch, replica=0):
        for rb in self.rbs:
            rb.push(*(x.numpy() for x in batch), replica=replica)
        s, r = batch[0], batch[2][:, 0].tolist()
        base = 0 if self.table is None else self.table[0].shape[0]
        self.table = list(batch) if self.table is None else [torch.cat([t, x]) for t, x in zip(self.table, batch)]
        self.index.update({k: base + i for i, k in enumerate(r)})
        tid = _tasks(self.spec, s)
        for t in range(self.T):
            for i in np.nonzero(tid == t)[0][-self.cap_t:]:       # more than a full sub-ring: the newest cap_t survive
                k = t * self.cap_t + int(self.head[replica, t])
                old = self.held[replica].pop(k, None)
                if old is not None:
                    del self.slot[replica][old]
                self.held[replica][k], self.slot[replica][r[i]] = r[i], k
                self.head[replica, t] = (self.head[replica, t] + 1) % self.cap_t
                self.fill[replica, t] = min(self.fill[replica, t] + 1, self.cap_t)

    def keys(self, core, replica=0):
        """Rewards of the minibatch the last step of `core` ingested, with its d checked against the transitions'."""
        keys = core.debug("r", replica).tolist()
        missing = [k for k in keys if k not in self.index]
        assert not missing, f"replica {replica}: {len(missing)} ingested rewards belong to no pushed transition: {missing[:4]}"
        want_d = self.table[4][[self.index[k] for k in keys], 0]
        assert torch.equal(core.debug("d", replica), want_d), f"replica {replica}: d is not the d of the rows r names"
        return keys

    def slots(self, keys, replica=0):
        bad = [k for k in keys if k not in self.slot[replica]]
        assert not bad, f"replica {replica}: {len(bad)} rows are not in this replica's ring (outside its filled region)"
        return np.array([self.slot[replica][k] for k in keys])

    def rows(self, keys):
        i = torch.tensor([self.index[k] for k in keys])
        return [t[i] for t in self.table]

    def close(self):
        for rb in self.rbs:
            rb.close()


def check_draw(ring, keys, slots, B, what=""):
    """A device-sampler minibatch: unique rows, batch slot i from task i / (B/T)'s sub-ring, rows neither constant nor
    all of one done flag."""
    per = B // ring.T
    assert len(set(keys)) == B, f"{what}{B - len(set(keys))} repeated rows in one minibatch"
    assert (slots // ring.cap_t == np.minimum(np.arange(B) // per, ring.T - 1)).all(), f"{what}a slot drew from another task"
    d = ring.table[4][[ring.index[k] for k in keys], 0]
    assert 0 < float(d.mean()) < 1, f"{what}d is constant over the minibatch"


def stacked(rows_per_replica):
    return [torch.stack([rows[j] for rows in rows_per_replica]) for j in range(5)]


def assert_identical(cores, n_steps, names):
    from distributed_sac_b200 import _lib
    ref = cores[0]
    R = ref.cfg.replicas
    for c, name in zip(cores[1:], names[1:]):
        for rep in range(R):
            for which in (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V):
                assert torch.equal(c.export_arena(which, rep), ref.export_arena(which, rep)), (names[0], name, rep, which)
            assert c.get_steps(rep) == ref.get_steps(rep), (names[0], name, rep, c.get_steps(rep), ref.get_steps(rep))
        assert torch.equal(c.read_losses(n_steps), ref.read_losses(n_steps)), (names[0], name)
    for rep in range(R):
        assert ref.get_steps(rep) == (n_steps,) * len(ref.get_steps(rep)), ref.get_steps(rep)


def _fill(ring, src, spec, R):
    """Pushes for the A / C cases: unequal per-task fills of 5-7 x B/T; R = 3: three different fills, replica 2's task-2
    sub-ring wrapped by 90 rows over two pushes."""
    T, per = ring.T, spec.batch // ring.T
    if R == 1:
        ring.push(src.take(_shuffled_tasks([per * (5 + t % 3) for t in range(T)], seed=1)))
        return
    plans = [([140, 200, 170], [0, 0, 0]), ([200, 133, 150], [0, 0, 0]), ([100, 80, 150], [50, 80, 140])]
    for rep, chunks in enumerate(plans):
        for j, counts in enumerate(chunks):
            if sum(counts):
                ring.push(src.take(_shuffled_tasks(counts, seed=10 * rep + j)), replica=rep)
    assert (ring.fill[2] == [150, 160, 200]).all() and ring.head[2, 2] == 90


# ---------------------------------------------------------------------------------------------------------------------
# A: one-step calls == multi-step graphs == b200sac_step on the recovered rows, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_sampled_step_equals_split_step(cuda, name):
    spec, care, precision, R, plan = SHAPES[name]
    check_plan(spec, care, precision, R, plan)
    a, b, c = (_core(spec, care, precision, R, seed=3) for _ in range(3))
    T = max(spec.num_tasks, 1)
    ring = Ring([a, b], spec, (200 if R > 1 else 8 * spec.batch // T) * T)
    _fill(ring, Source(spec, seed=4), spec, R)
    calls = (15, 16, 3)                                       # 8+4+2+1, 8+8, 2+1
    step = 0
    for n in calls:
        for _ in range(n):
            a.step_sampled(ring.rbs[0], 1)
            drawn = []
            for rep in range(R):
                keys = ring.keys(a, rep)
                check_draw(ring, keys, ring.slots(keys, rep), spec.batch, f"{name} step {step} replica {rep}: ")
                if step == 0:
                    check_active(a, spec, rep, f"{name} replica {rep}: ", care=care)
                drawn.append(ring.rows(keys))
            c.step(*stacked(drawn))
            step += 1
        b.step_sampled(ring.rbs[1], n)
        for rep in range(R):                                  # the multi-step call's last step drew A's last minibatch
            assert torch.equal(b.debug("r", rep), a.debug("r", rep)), (name, n, rep)
    if R > 1:
        L = a.read_losses(1)[0]
        assert not torch.equal(L[0], L[1]) and not torch.equal(L[1], L[2])
    assert_identical([a, b, c], step, ["one-step calls", "multi-step calls", "b200sac_step"])
    ring.close()
    for x in (a, b, c):
        x.close()


# ---------------------------------------------------------------------------------------------------------------------
# B: the pinned-host ring (host draw, two staging slots, the next minibatch prefetched while a step runs)
# ---------------------------------------------------------------------------------------------------------------------
def test_host_ring_equals_split_step(cuda):
    """update_sampled, step_sampled(rb, n), step_host interleaved (two step_host calls in a row reuse the staging slot
    that holds the prefetched minibatch: acquire_slot voids it) and a push that wraps over rows already gathered into
    the prefetch slot.  A runs every sampled step as its own call, B the same program with multi-step calls, C
    b200sac_step on the rows A's steps ingested."""
    spec = sp.SacSpec(state_dim=8, num_tasks=4, batch=64, **_SMALL)
    R, per = 2, 16
    a, b, c = (_core(spec, False, 0, R, seed=5) for _ in range(3))
    ring = Ring([a, b], spec, 4 * 128, where="host", seed=7)
    src = Source(spec, seed=8)
    for rep in range(R):
        ring.push(src.take(_shuffled_tasks([128, 100, 90 + 20 * rep, 110], seed=rep)), replica=rep)
    program = [("update", 1), ("sampled", 3), ("host", 1), ("sampled", 2), ("host", 1), ("host", 1), ("update", 1),
               ("sampled", 1), ("push", 0), ("sampled", 4), ("update", 1), ("sampled", 2)]
    step, after_push, overwritten = 0, False, 0
    for op, n in program:
        if op == "push":                                     # overwrites 3/4 of every sub-ring of both replicas
            alive_before = [set(ring.slot[rep]) for rep in range(R)]
            for rep in range(R):
                ring.push(src.take(_shuffled_tasks([96] * 4, seed=20 + rep)), replica=rep)
            after_push = True
            continue
        if op == "host":
            x = [src.take(_shuffled_tasks([per] * 4, seed=30 + step + rep)) for rep in range(R)]
            for core in (a, b):
                core.step_host(*stacked(x), want_losses=False)
            c.step(*stacked(x))
            step += 1
            continue
        for i in range(n):
            if op == "update":
                got = a.update_sampled(ring.rbs[0])
                assert list(got) == a.read_losses(1)[0, 0].tolist()
            else:
                a.step_sampled(ring.rbs[0], 1)
            drawn = []
            for rep in range(R):
                keys = ring.keys(a, rep)
                assert len(set(keys)) == spec.batch
                if step == 0:
                    check_active(a, spec, rep, f"replica {rep}: ")
                if after_push:                               # the prefetched minibatch: gathered before the push
                    assert set(keys) <= alive_before[rep], f"step {step} replica {rep}: a row not in the ring at draw time"
                    overwritten += len(set(keys) - set(ring.slot[rep]))
                else:
                    ring.slots(keys, rep)
                drawn.append(ring.rows(keys))
            after_push = False
            c.step(*stacked(drawn))
            step += 1
        if op == "update":
            got = b.update_sampled(ring.rbs[1])
            assert list(got) == b.read_losses(1)[0, 0].tolist()
        else:
            b.step_sampled(ring.rbs[1], n)
    assert overwritten > 0, "the push overwrote none of the prefetched rows"
    assert_identical([a, b, c], step, ["one-step calls", "multi-step calls", "b200sac_step"])
    ring.close()
    for x in (a, b, c):
        x.close()


def test_push_then_step_on_a_side_stream(cuda):
    """push, then at once a sampled step on a non-blocking stream: the step gathers the rows and the fill of that push
    (b200sac_replay_push drains its copies before it returns) -- every row is in the ring as the model holds it after
    the push, and the steps equal b200sac_step on those rows bit for bit."""
    spec = sp.SacSpec(state_dim=8, batch=96, **_SMALL)
    a, c = _core(spec, False, 0, seed=2), _core(spec, False, 0, seed=2)
    ring = Ring([a], spec, 8 * 96)
    src = Source(spec, seed=9)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for k in range(6):
            ring.push(src.take(np.zeros(5 * 96 if k == 0 else 3 * 96, np.int64)))     # wraps from the third push on
            a.step_sampled(ring.rbs[0], 1)
            keys = ring.keys(a)
            slots = ring.slots(keys)
            check_draw(ring, keys, slots, spec.batch, f"step {k}: ")
            if k == 0:
                check_active(a, spec)
            c.step(*ring.rows(keys))
    torch.cuda.synchronize()
    assert ring.fill[0, 0] == 8 * 96 and ring.head[0, 0] == 4 * 96
    assert_identical([a, c], 6, ["sampled on a side stream", "b200sac_step"])
    ring.close()
    a.close()
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# C: each sampled step against the autograd oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ll_chained", "layer_p1", "mtsac_t10", "care_o"])
def test_sampled_step_matches_oracle(cuda, name):
    """From the oracle's state, one sampled step; the minibatch rebuilt from r, the noise read from psave; the CUDA
    masks, tanh values and min routing forced into the oracle (every flipped bit a kink): losses, y, Q, actions,
    log-probs and every parameter, target and Adam moment at 1e-4."""
    spec, care, precision, R, plan = SHAPES[name]
    from distributed_sac_b200 import _lib
    check_plan(spec, care, precision, R, plan)
    core = _core(spec, care, precision, seed=11)
    T = max(spec.num_tasks, 1)
    ring = Ring([core], spec, 8 * spec.batch // T * T)
    _fill(ring, Source(spec, seed=12), spec, 1)
    mod = cp if care else sp
    port = (cp.CarePortLearner if care else sp.PortLearner)(spec, mod.init_params(spec, seed=3))
    B, A = spec.batch, spec.act_dim
    worst = dict(loss=0.0, rows=0.0, state=0.0)
    for step in range(3):
        sync_core_to_port(core, port)
        core.step_sampled(ring.rbs[0], 1)
        keys = ring.keys(core)
        check_draw(ring, keys, ring.slots(keys), B, f"{name} step {step}: ")
        batch = ring.rows(keys)
        eps = core.debug("psave").reshape(2 * B, A, 8)[:, :, 5]
        check_active(core, spec, what=f"{name} step {step}: ", care=care)
        forced = cuda_relu_masks(core, spec, care=care)
        with sp.ReluTape(forced) as tape:
            out = (port.update if care else port.update_SAC)(*batch, eps[:B].clone(), eps[B:].clone(), want_intermediates=True)
        check_forced(tape, forced, f"{name} step {step}: ")
        L = core.read_losses(1)[0, 0]
        for j, k in ((0, "critic_loss"), (1, "actor_loss"), (3, "entropy")):
            e = rel_scalar(float(L[j]), out[k])
            assert e <= REL, (name, step, k, float(L[j]), out[k])
            worst["loss"] = max(worst["loss"], e)
        for key in ("y", "q1", "q2", "a_next", "a_cur", "logp_next", "logp_cur"):
            ref = out[key].reshape(-1)
            e = float((core.debug(key) - ref).abs().max()) / (float(ref.abs().max()) + 1.0)
            assert e <= REL, (name, step, key, e)
            worst["rows"] = max(worst["rows"], e)
        check_port_state(core, port)
        st, got = port.adam_state(), [core.get_named(w) for w in (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V)]
        for k, v in port.params().items():
            if k != "log_alpha":
                worst["state"] = max([worst["state"], rel_l2(got[0][k], v)] +
                                     ([rel_l2(got[1][k], st["m"][k]), rel_l2(got[2][k], st["v"][k])] if k in st["m"] else []))
    print(f"[oracle] {name}: largest deviation -- losses {worst['loss']:.2e}, per-row outputs {worst['rows']:.2e} "
          f"(of max|ref| + 1), state rel-L2 {worst['state']:.2e}")
    ring.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# D: the device sampler against its contract
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [0, 10])
@pytest.mark.parametrize("batch", [64, 256, 260, 2048])
def test_device_sampler_contract(cuda, T, batch):
    """Two replicas: replica 0 at larger, unequal per-task fills, replica 1 at the minimum 4 B/T.  Over 60 steps: slot i
    draws from task i / (B/T)'s sub-ring, rows are unique within a step and inside the replica's filled region, the
    replicas draw their own rows, consecutive minibatches differ, and per (replica, task) the slot counts fit uniform
    (chi-square; drawing without replacement within a step only under-disperses the counts).  B = 260 takes the
    512-thread launch; 2048 (check_cfg's maximum) fills half the 4096-slot hash.  With T = 10 the batch is the multiple
    of 10 below it."""
    B = batch // T * T if T else batch
    spec = sp.SacSpec(state_dim=4, act_dim=1, actor_hidden=[16], critic_hidden=[16], batch=B, num_tasks=T)
    Tn, per = max(T, 1), B // max(T, 1)
    fills = [[4 * per + per * ((7 * t + 3) % 10) // 3 + 5 * t + 1 for t in range(Tn)], [4 * per] * Tn]
    cap_t = max(fills[0])
    core = _core(spec, False, 0, replicas=2, seed=6)
    ring = Ring([core], spec, cap_t * Tn, seed=13)
    src = Source(spec, seed=14)
    for rep in range(2):
        ring.push(src.take(_shuffled_tasks(fills[rep], seed=rep)), replica=rep)
        assert (ring.fill[rep] == fills[rep]).all()
    counts = np.zeros((2, cap_t * Tn), np.int64)
    prev = [None, None]
    n_steps = 60
    for step in range(n_steps):
        core.step_sampled(ring.rbs[0], 1)
        slots = []
        for rep in range(2):
            keys = ring.keys(core, rep)
            sl = ring.slots(keys, rep)
            check_draw(ring, keys, sl, B, f"step {step} replica {rep}: ")
            assert (sl % cap_t < ring.fill[rep][sl // cap_t]).all()
            assert prev[rep] is None or set(sl.tolist()) != prev[rep], f"step {step} replica {rep}: the same minibatch again"
            prev[rep] = set(sl.tolist())
            counts[rep] += np.bincount(sl, minlength=cap_t * Tn)
            slots.append(sl)
        assert not np.array_equal(slots[0], slots[1]), f"step {step}: both replicas drew the same slots"
    for rep in range(2):
        for t in range(Tn):
            obs = counts[rep, t * cap_t:t * cap_t + fills[rep][t]]
            assert obs.sum() == n_steps * per
            p = stats.chisquare(obs).pvalue
            assert p > 1e-4, f"replica {rep} task {t}: slot counts are not uniform (p = {p:.2e}, min {obs.min()}, max {obs.max()})"
    ring.close()
    core.close()


def test_refuses_a_ring_below_four_per_task_batches(cuda):
    """One sub-ring one row short of 4 B/T: RuntimeError, and the handle is untouched; one more row and it steps."""
    from distributed_sac_b200 import _lib
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[32], critic_hidden=[32], batch=60, num_tasks=10)
    core = _core(spec, False, 0, seed=1)
    ring = Ring([core], spec, 10 * 40)
    src = Source(spec, seed=15)
    ring.push(src.take(_shuffled_tasks([24] * 9 + [23], seed=0)))
    before = [core.export_arena(w) for w in (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V)]
    with pytest.raises(RuntimeError, match="not ready"):
        core.step_sampled(ring.rbs[0], 1)
    with pytest.raises(RuntimeError, match="not ready"):
        core.update_sampled(ring.rbs[0])
    torch.cuda.synchronize()
    assert all(torch.equal(core.export_arena(w), x) for w, x in zip((_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V), before))
    assert core.get_steps() == (0, 0, 0)
    ring.push(src.take(np.full(1, 9)))
    core.step_sampled(ring.rbs[0], 1)
    assert core.get_steps() == (1, 1, 1)
    ring.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# E: prepare, profile_step and the loss ring's wrap
# ---------------------------------------------------------------------------------------------------------------------
def _twins(spec, n_rows, seed=0):
    cores = [_core(spec, False, 0, seed=seed) for _ in range(2)]
    ring = Ring(cores, spec, n_rows)
    ring.push(Source(spec, seed=seed + 1).take(np.zeros(n_rows, np.int64)))
    return cores, ring


def test_prepare_changes_nothing(cuda):
    spec = sp.SacSpec(state_dim=8, batch=64, **_SMALL)
    (a, b), ring = _twins(spec, 512)
    a.prepare(ring.rbs[0])
    a.step_sampled(ring.rbs[0], 11)
    b.step_sampled(ring.rbs[1], 11)
    assert_identical([a, b], 11, ["prepared", "not prepared"])
    ring.close()
    a.close()
    b.close()


def test_profile_step_runs_plain_sampled_steps(cuda):
    """profile_step's eager, unforked steps equal three one-step sampled calls, and read_losses(3) returns those steps."""
    spec = sp.SacSpec(state_dim=8, batch=64, **_SMALL)
    (a, b), ring = _twins(spec, 512, seed=4)
    a.profile_step(ring.rbs[0], iters=3)
    for _ in range(3):
        b.step_sampled(ring.rbs[1], 1)
    assert torch.equal(a.debug("r"), b.debug("r"))
    assert_identical([a, b], 3, ["profile_step", "step_sampled"])
    ring.close()
    a.close()
    b.close()


def test_loss_ring_wraps(cuda):
    """1030 steps in one call: read_losses(1024) equals the last 1024 losses a twin read after each of its one-step calls,
    and each of those is the critic loss of its own step (mean (y - Q1)^2 + mean (y - Q2)^2 from the step's y, q1, q2)."""
    spec = sp.SacSpec(state_dim=4, act_dim=1, actor_hidden=[16], critic_hidden=[16], batch=32)
    (a, b), ring = _twins(spec, 256, seed=7)
    a.step_sampled(ring.rbs[0], 1030)
    seen = []
    for _ in range(1030):
        b.step_sampled(ring.rbs[1], 1)
        L = b.read_losses(1)[0]
        y, q1, q2 = (b.debug(k).double() for k in ("y", "q1", "q2"))
        want = float(((y - q1) ** 2).mean() + ((y - q2) ** 2).mean())
        assert rel_scalar(float(L[0, 0]), want) <= REL, (len(seen), float(L[0, 0]), want)
        seen.append(L)
    seen = torch.stack(seen[-1024:])
    assert torch.equal(a.read_losses(1024), seen) and torch.equal(b.read_losses(1024), seen)
    with pytest.raises(RuntimeError, match="out of range"):
        a.read_losses(1025)
    ring.close()
    a.close()
    b.close()
