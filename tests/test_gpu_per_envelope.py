"""GPU: prioritized experience replay (per_kernels.cuh, the b200sac_replay_*_prioritized entry points, the weighted critic
loss in chain2_kernel and critic_heads_kernel) over its whole envelope, against the numpy sum-tree model and the autograd
oracle.

per_sample_kernel keeps the top Lc levels of every task's tree in 16 KB of shared memory (Lc = 12, lowered while T << Lc >
4096, capped at levels + 1) and gives a thread several rows above a batch of 512; per_update_kernel holds up to 8 batch
slots per thread (the 8th above a batch of 1792); set_priorities works in chunks of 2048; per_fill_kernel rebuilds the
ancestors of a leaf range level by level with 1024 threads.  The sampler cases reach a fully cached tree, a partly cached
one whose leaves come from L2 (a 2^20-slot ring), Lc cut down by T (T = 3 and T = 64), one row per task, batches of 2048,
padding leaves (cap_per_task not a power of two), pushes that wrap a sub-ring at T > 0 and fill_synthetic at R > 1; a
CPU-only test mirrors the geometry and names any branch the cases stop reaching.  Every tree is compared bit for bit with
oracle/per_ref.build_tree, every draw with the descent model's strata, every weight with per_ref.is_weights.
"""
import numpy as np
import pytest
import torch
from scipy import stats

import care_port as cp
import per_ref
import sac_port as sp
from _golden import REL, check_forced, check_port_state, cuda_relu_masks, rel_l2, rel_scalar, sync_core_to_port
from _harness import _core, _sms, _tasks, care_t4, cuda, plan_rows

gpu = pytest.mark.gpu

kPerTopNodes, kPerMaxB, kMaxPer = 4096, 2048, 8

# id -> (T, cap_per_task, batch, replicas, how the sub-rings are filled, rows per sub-ring)
#   cached_pad  P = 1024 for 1000 slots (24 padding leaves, 50 empty ones): Lc = levels + 1, the whole tree in shared memory
#   l2_2p20     one 2^20-slot ring, 20 levels: Lc = 12, the lower 8 levels read from L2; 2 rows per sampler thread;
#               fill_synthetic rebuilds ranges of 2^19 nodes
#   t3_r2       T = 3: Lc cut to 10 by the task count (12 levels); R = 2 filled by fill_synthetic
#   t64_per1    T = 64, one row per task, Lc = 6 < 8; cap 65 = 2^6 + 1 (63 padding leaves); pushes that wrap every sub-ring
#   b2048_t0    batch 2048, T = 0: 4 rows per sampler thread; cap 8193 = 2^13 + 1
#   b2048_t16   batch 2048, T = 16 (Lc = 8 of 11 levels), 128 rows per task
SAMPLER = {
    "cached_pad": (0, 1000, 200, 1, "push", 950),
    "l2_2p20": (0, 1 << 20, 1024, 1, "synthetic", 1 << 20),
    "t3_r2": (3, 3000, 768, 2, "synthetic", 2700),
    "t64_per1": (64, 65, 64, 1, "push_wrap", 65),
    "b2048_t0": (0, 8193, 2048, 1, "synthetic", 8193),
    "b2048_t16": (16, 600, 2048, 1, "synthetic", 560),
}
UPDATE_B = 2048                 # the in-graph update case (test_in_graph_update_b2048_r3)
SET_N = 5000                    # set_priorities with duplicates across chunk boundaries

PER = dict(alpha=0.6, beta=0.8, eps=1e-6)


def geometry(T, cap_t, B):
    """Mirror of per_kernels.cuh: tree size, cached levels Lc, rows per task and per thread of both kernels."""
    Tn = max(T, 1)
    P, levels = 1, 0
    while P < cap_t:
        P, levels = 2 * P, levels + 1
    Lc = 12
    while (Tn << Lc) > kPerTopNodes:
        Lc -= 1
    Lc = min(Lc, levels + 1)
    threads = 512 if B > 256 else 256                     # per_sample_kernel's block
    return dict(P=P, levels=levels, Lc=Lc, per=B // Tn, sample_rows=-(-B // threads), update_slots=-(-B // 256))


def reached_branches():
    """The branches of the PER kernels that the cases of this file reach."""
    have = set()
    for T, cap_t, B, _R, how, fill in SAMPLER.values():
        g = geometry(T, cap_t, B)
        if g["Lc"] == g["levels"] + 1:
            have.add("fully cached")
        if g["Lc"] < g["levels"] + 1:
            have.add("partly cached")
        if g["Lc"] < 12 and g["Lc"] < g["levels"] + 1:
            have.add("Lc limited by T")
        if g["per"] == 1:
            have.add("per = 1")
        if g["sample_rows"] > 1:
            have.add("several rows per sampler thread")
        if g["P"] > cap_t:
            have.add("padding leaves")
        if how == "synthetic" and g["P"] // 2 > 1024:
            have.add("per_fill range over 1024 nodes")
        if how == "push_wrap" and T > 0:
            have.add("push wraps a sub-ring at T > 0")
    if geometry(0, 8192, UPDATE_B)["update_slots"] == kMaxPer:
        have.add("kMaxPer slot 8")
    if SET_N > 2 * kPerMaxB:
        have.add("set_priorities chunks")
    return have


BRANCHES = {"fully cached", "partly cached", "Lc limited by T", "per = 1", "several rows per sampler thread",
            "padding leaves", "per_fill range over 1024 nodes", "push wraps a sub-ring at T > 0", "kMaxPer slot 8",
            "set_priorities chunks"}


def test_cases_reach_every_branch():
    """(CPU) the sweep is not vacuous: each size-dependent branch of the PER kernels is reached by some case."""
    missing = BRANCHES - reached_branches()
    assert not missing, f"no case reaches: {sorted(missing)}"
    assert geometry(3, 3000, 768)["Lc"] == 10 and geometry(64, 65, 64)["Lc"] == 6 and geometry(0, 1 << 20, 1024)["Lc"] == 12


def _tiny(T, B):
    return sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[32], critic_hidden=[32], batch=B, num_tasks=T)


def _push(rb, spec, care, n, seed, replica):
    """Push n synthetic transitions (tasks i mod T, balanced) to one replica; returns them."""
    s, a, r, s2, d = (cp if care else sp).synthetic_batch(spec, seed=seed, batch=n)
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy(), replica=replica)
    return s, a, r, s2, d


def _leaf_table(rb, T, cap_t, replica):
    """[T][cap_t] leaves and [T] roots of one replica, read as whole trees."""
    trees = [rb.tree(t, replica) for t in range(max(T, 1))]
    P = len(trees[0]) // 2
    return trees, np.stack([tr[P:P + cap_t] for tr in trees])


def _assert_tree(got, leaves, what):
    want = per_ref.build_tree(leaves, len(got) // 2)
    bad = np.nonzero(got[1:].view(np.int32) != want[1:].view(np.int32))[0] + 1
    assert bad.size == 0, f"{what}: {bad.size} nodes differ from the rebuilt tree, first node {bad[0]} got {got[bad[0]]} want {want[bad[0]]}"


def _ulps(a, b):
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32).astype(np.int64))


# ---------------------------------------------------------------------------------------------------------------------
# 1: trees and the sampler at every size-dependent branch
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", list(SAMPLER))
def test_sampler_and_trees(cuda, name):
    from distributed_sac_b200.core import Replay
    T, cap_t, B, R, how, fill = SAMPLER[name]
    Tn = max(T, 1)
    spec = _tiny(T, B)
    g = geometry(T, cap_t, B)
    core = _core(spec, replicas=R)
    rb = Replay(core, Tn * cap_t, seed=9, prioritized=PER)
    if how == "synthetic":
        rb.fill_synthetic(Tn * fill)
    elif how == "push":
        _push(rb, spec, False, Tn * fill, 5, 0)
    else:                                                 # two pushes of 40 rows per task: the second wraps every sub-ring
        _push(rb, spec, False, Tn * 40, 5, 0)
        rb.set_priorities(np.arange(Tn) * cap_t, np.full(Tn, 3.0))        # max p 3^0.6 for the wrapped rows
        _push(rb, spec, False, Tn * 40, 6, 0)
    # after the fill: filled leaves hold max p, the rest 0, every internal node the rebuilt sum
    mp = per_ref.leaf_values([3.0], PER["alpha"], PER["eps"])[0] if how == "push_wrap" else np.float32(1.0)
    for r in range(R):
        trees, leaves = _leaf_table(rb, T, cap_t, r)
        for t in range(Tn):
            want = np.zeros(cap_t, np.float32)
            want[:fill] = 1.0
            if how == "push_wrap":
                want[0] = mp                                # set before the wrap; then slots 40..64 and 0..14 get max p
                want[40:] = mp
                want[:15] = mp
            _assert_tree(trees[t], want, f"{name} replica {r} task {t} after the fill")
    # distinct, skewed priorities on every filled slot, in one call per replica (chunked above 2048 entries)
    rng = np.random.default_rng(11)
    slots = (np.arange(Tn)[:, None] * cap_t + np.arange(fill)[None, :]).reshape(-1)
    prio = {}
    for r in range(R):
        prio[r] = (rng.exponential(1.0, slots.size) ** 3).astype(np.float32)
        rb.set_priorities(slots, prio[r], replica=r)
    for r in range(R):
        trees, leaves = _leaf_table(rb, T, cap_t, r)
        want = np.zeros((Tn, cap_t), np.float32)
        want[:, :fill] = per_ref.leaf_values(prio[r], PER["alpha"], PER["eps"]).reshape(Tn, fill)
        for t in range(Tn):
            _assert_tree(trees[t], want[t], f"{name} replica {r} task {t} after set_priorities")
        bounds = [per_ref.strata(trees[t], g["per"]) for t in range(Tn)]
        roots = np.array([trees[t][1] for t in range(Tn)])
        i = np.arange(B)
        t_of, j_of = i // g["per"], i % g["per"]
        lo = np.array([bounds[t][0][j] for t, j in zip(t_of, j_of)])
        hi = np.array([bounds[t][1][j] for t, j in zip(t_of, j_of)])
        counts = np.zeros(Tn * cap_t, np.int64)
        n_draws = 100 if name == "l2_2p20" else 8
        for k in range(n_draws):
            *_rows, idx, w = rb.sample_prioritized(r)
            idx = idx.numpy()
            task, slot = idx // cap_t, idx % cap_t
            assert (task == t_of).all(), f"{name}: a row drawn from another task's sub-ring"
            assert (slot < fill).all() and (want[task, slot] > 0).all(), f"{name}: an empty slot was drawn"
            out = np.nonzero((slot < lo) | (slot > hi))[0]
            assert out.size == 0, (f"{name} replica {r} draw {k}: {out.size} rows outside their stratum, first batch slot "
                                   f"{out[0]}: leaf {slot[out[0]]} not in [{lo[out[0]]}, {hi[out[0]]}]")
            ww = per_ref.is_weights(want[task, slot], roots[task], fill, PER["beta"])
            assert _ulps(w.numpy(), ww).max() <= 1, f"{name}: weights differ from (N p / S)^-beta by {_ulps(w.numpy(), ww).max()} ulp"
            counts += np.bincount(idx, minlength=Tn * cap_t)
        if name == "l2_2p20":                            # counts over 256 groups of 4096 slots fit the groups' p / S
            grp = counts.reshape(256, -1).sum(1)
            expect = want[0].astype(np.float64).reshape(256, -1).sum(1)
            res = stats.chisquare(grp, expect / expect.sum() * grp.sum())
            assert res.pvalue > 1e-3, res
    print(f"[per] {name}: P {g['P']}, levels {g['levels']}, Lc {g['Lc']}, per {g['per']}, rows per sampler thread "
          f"{g['sample_rows']}, R {R}")
    rb.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: the in-graph priority update at B = 2048, R = 3, and set_priorities across its chunks
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_in_graph_update_b2048_r3(cuda):
    """A step's update writes leaf_values(td_priority(y, q1, q2)) at every drawn slot (the highest batch slot wins an
    index drawn several times: a few hundred hot slots make long duplicate chains), every ancestor is the rebuilt sum, and
    max p per (replica, task) is raised -- in all three replicas, each from its own y and Q."""
    from distributed_sac_b200.core import Replay
    spec = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=UPDATE_B)
    R, cap = 3, 8192
    core = _core(spec, precision=1, replicas=R)
    rb = Replay(core, cap, seed=2, prioritized=PER)
    rng = np.random.default_rng(4)
    leaves = {}
    for r in range(R):
        _push(rb, spec, False, cap, 40 + r, r)
        prio = np.zeros(cap, np.float32)
        prio[rng.choice(cap, 300, replace=False)] = 0.2               # hot: 0.38 against 2.5e-4 for the rest
        rb.set_priorities(np.arange(cap), prio, replica=r)
        leaves[r] = per_ref.leaf_values(prio, PER["alpha"], PER["eps"])
    core.step_sampled(rb, 1)
    for r in range(R):
        idx = core.debug("idx", r).long().numpy()
        assert len(np.unique(idx)) < 400 and np.bincount(idx).max() >= 4, "the batch has no long duplicate chains"
        new = per_ref.leaf_values(per_ref.td_priority(core.debug("y", r), core.debug("q1", r), core.debug("q2", r)),
                                  PER["alpha"], PER["eps"])
        assert np.array_equal(core.debug("prio", r).numpy(), new), f"replica {r}: leaf values of the step"
        want = leaves[r].copy()
        for k, v in zip(idx, new):                       # in batch-slot order: the highest slot wins
            want[k] = v
        assert new.max() > 1.0, "no TD priority above the initial max p: the raise is not exercised"
        got = rb.tree(0, r)
        _assert_tree(got, want, f"replica {r} after the step")
        # max p = max(1, every leaf written so far): a pushed row receives it
        _push(rb, spec, False, 1, 90 + r, r)
        assert rb.priorities([0], r)[0] == max(np.float32(1.0), new.max()), f"replica {r}: max p not raised"
    # set_priorities: 5000 entries, duplicates inside one chunk and across the 2048 / 4096 chunk boundaries
    r = 1
    base = rb.tree(0, r)[cap:2 * cap].copy()
    ix = rng.choice(cap, SET_N, replace=False)
    ix[2050], ix[2060], ix[4100] = ix[2040], ix[10], ix[4090]
    ix[4990] = ix[3000]
    pv = rng.exponential(1.0, SET_N).astype(np.float32)
    others = [rb.tree(0, r0) for r0 in (0, 2)]
    rb.set_priorities(ix, pv, replica=r)
    want = base.copy()
    for k, v in zip(ix, per_ref.leaf_values(pv, PER["alpha"], PER["eps"])):   # in call order: a later entry wins
        want[k] = v
    _assert_tree(rb.tree(0, r), want, "set_priorities with duplicates across chunks")
    for r0, before in zip((0, 2), others):                                  # the other replicas' trees are untouched
        assert np.array_equal(rb.tree(0, r0), before), r0
    rb.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: weighted parity with the autograd oracle across the step plans
# ---------------------------------------------------------------------------------------------------------------------
# id -> (spec, care, precision, replicas)
def _parity_case(name):
    if name == "chained_b37":                 # a tail CTA in every chain launch
        return sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=37), False, 0, 1
    if name == "chained_r3":                  # replicas with their own parameters, priorities, beta; 8 / 8 / 4 rows per CTA
        return (sp.SacSpec(state_dim=9, num_tasks=5, act_dim=3, actor_hidden=[64, 48], critic_hidden=[56, 72], batch=105),
                False, 0, 3)
    if name == "layer_p0_400":                # per-layer fp32 plan at 400 wide
        return (sp.SacSpec(state_dim=39, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=128),
                False, 0, 1)
    if name == "layer_p1_b2048":              # wgmma plan, split-K weight-gradient slices fed with weighted dq
        return (sp.SacSpec(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=2048),
                False, 1, 1)
    if name == "mtsac_t64":                   # 64 tasks, 2 rows each, weighted loss
        return (sp.SacSpec(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=128,
                           num_tasks=64, weighted_loss=True), False, 1, 1)
    if name == "care_o":
        return care_t4(False), True, 1, 1
    return care_t4(), True, 1, 2     # care_m_r2


PARITY = ["chained_b37", "chained_r3", "layer_p0_400", "layer_p1_b2048", "mtsac_t64", "care_o", "care_m_r2"]
PER_ROW = ("y", "q1", "q2", "a_next", "a_cur", "logp_next", "logp_cur")


def _parity_ring(core, spec, care, R, seed):
    """A prioritized ring whose sub-rings hold a number of rows that differs per task, in a pattern that differs per
    replica (the fill N_t does not cancel in the batch-normalised weights, and a weight computed with another replica's
    fill is wrong); skewed priorities with a few very hot slots (drawn several times per batch).  Returns (ring,
    [replica] host table ring index -> rows, [replica] [T] fill per task, cap_per_task)."""
    from distributed_sac_b200.core import Replay
    T = max(spec.num_tasks, 1)
    per = spec.batch // T
    cap_t = max(64, 8 * per)
    rb = Replay(core, T * cap_t, seed=seed, prioritized=dict(PER, beta=1.0))
    rng = np.random.default_rng(seed)
    tables, fills = [], []
    for r in range(R):
        fill = np.array([cap_t - cap_t // 16 * ((r + 1) * t % 5) for t in range(T)])      # >= 3/4 cap_t >= 6 per
        rows = (cp if care else sp).synthetic_batch(spec, seed=seed + 10 * r, batch=T * cap_t)
        tid = _tasks(spec, rows[0])
        rank = np.zeros(T * cap_t, np.int64)
        for t in range(T):
            k = np.nonzero(tid == t)[0]
            rank[k] = np.arange(len(k))
        keep = rank < fill[tid]
        rows = [x[torch.from_numpy(keep)] for x in rows]
        rb.push(*[x.numpy() for x in rows], replica=r)
        tid, rank = tid[keep], rank[keep]
        where = tid * cap_t + rank
        table = [torch.zeros(T * cap_t, x.shape[1]) for x in rows]
        for tb, x in zip(table, rows):
            tb[where] = x
        tables.append(table)
        fills.append(fill)
        slots = np.sort(where)
        prio = rng.exponential(1.0, slots.size) ** 3
        prio[rng.choice(slots.size, 2 * T, replace=False)] = 40.0 * prio.max()
        rb.set_priorities(slots, prio, replica=r)
    return rb, tables, fills, cap_t


@gpu
@pytest.mark.parametrize("name", PARITY)
def test_weighted_parity_envelope(cuda, name):
    """Two PER steps at beta = 1 (R = 3: beta 1, 0.8, 0.6) on skewed priorities: each replica's weights equal
    per_ref.is_weights of the leaves it drew (1 ulp), and each replica's step matches its own autograd oracle given those
    weights (masks, tanh and min routing forced) -- losses (the loss ring's weighted critic loss), every per-row output,
    every parameter, target and Adam moment -- at the 1e-4 bar."""
    from distributed_sac_b200 import _lib
    spec, care, precision, R = _parity_case(name)
    core = _core(spec, care, precision, replicas=R)
    if name == "chained_r3":
        sms = _sms()
        rows3, rows1 = plan_rows(spec.batch, R, sms), plan_rows(spec.batch, 1, sms)
        print(f"[rows] R = 3: {rows3}, R = 1: {rows1} ({sms} SMs)")
        if sms == 132:
            assert list(rows3.values()) == [8, 8, 4]
        assert rows3 != rows1
    rb, tables, fills, cap_t = _parity_ring(core, spec, care, R, seed=17)
    betas = [1.0, 0.8, 0.6][:R]
    for r in range(R):
        rb.set_beta(betas[r], replica=r)
    mod = cp if care else sp
    ports = [(cp.CarePortLearner if care else sp.PortLearner)(spec, mod.init_params(spec, seed=3 + r)) for r in range(R)]
    T = max(spec.num_tasks, 1)
    per = spec.batch // T
    worst = dict(loss=0.0, rows=0.0, state=0.0, flips=0)
    for step in range(2):
        pre = [_leaf_table(rb, spec.num_tasks, cap_t, r) for r in range(R)]
        for r in range(R):
            sync_core_to_port(core, ports[r], r)
        core.step_sampled(rb, 1)
        L = core.read_losses(1)[0]
        for r in range(R):
            what = f"{name} step {step} replica {r}: "
            B, A = spec.batch, spec.act_dim
            idx = core.debug("idx", r).long()
            batch = [tb[idx] for tb in tables[r]]
            eps = core.debug("psave", r).reshape(2 * B, A, 8)[:, :, 5]
            e1, e2, w = eps[:B].clone(), eps[B:].clone(), core.debug("isw", r)
            ix = idx.numpy()
            task, slot = ix // cap_t, ix % cap_t
            assert (task == np.arange(B) // per).all() and (slot < fills[r][task]).all(), what + "drawn outside the filled slots"
            trees, leaves = pre[r]
            want_w = per_ref.is_weights(leaves[task, slot], np.array([tr[1] for tr in trees])[task], fills[r][task], betas[r])
            assert _ulps(w.numpy(), want_w).max() <= 1, what + f"weights off by {_ulps(w.numpy(), want_w).max()} ulp"
            assert float(w.max()) == 1.0 and float(w.min()) < 0.5, what + "the weights are not skewed"
            assert np.bincount(ix).max() >= 2, what + "no index drawn twice"
            forced = cuda_relu_masks(core, spec, r, care=care)
            with per_ref.ImportanceWeights(w), sp.ReluTape(forced) as tape:
                out = (ports[r].update if care else ports[r].update_SAC)(*batch, e1, e2, want_intermediates=True)
            worst["flips"] += sum(check_forced(tape, forced, what).values())
            for j, want in ((0, per_ref.weighted_critic_loss(out, w, spec.weighted_loss)), (1, out["actor_loss"])):
                e = rel_scalar(float(L[r, j]), want)
                assert e <= REL, (what, j, float(L[r, j]), want)
                worst["loss"] = max(worst["loss"], e)
            for k in PER_ROW:
                ref = out[k].detach().double().reshape(B, -1)
                got = core.debug(k, r).double().reshape(ref.shape)
                scale = ref.abs() + ref.abs().mean()
                dev = float(((got - ref).abs() / scale.clamp_min(1e-30)).max())
                assert dev <= REL, f"{what}{k}: {dev:.2e} of |ref| + mean|ref|"
                worst["rows"] = max(worst["rows"], dev)
            check_port_state(core, ports[r], replica=r)
            got = core.get_named(_lib.PARAMS, r)
            worst["state"] = max([worst["state"]] + [rel_l2(got[k], v) for k, v in ports[r].params().items() if k != "log_alpha"])
    if R > 1:
        assert not torch.equal(L[0], L[1])
    rb.close()
    core.close()
    print(f"[parity] {name}: losses {worst['loss']:.1e}, per-row {worst['rows']:.1e}, parameters rel-L2 {worst['state']:.1e}, "
          f"{worst['flips']} mask bits differed from the oracle's own")


# ---------------------------------------------------------------------------------------------------------------------
# 4: multi-step graphs and per-replica beta, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_graphs_and_replica_beta_bit_exact(cuda):
    """R = 3, T = 4: step_sampled(rb, 19) (8 + 8 + 2 + 1-step graphs) equals 19 single steps in all three arenas of every
    replica, every priority and the loss ring; then set_beta(0.3, replica=1) on one handle changes replica 1's weights and
    parameters at the next step and nothing of replicas 0 and 2, against a handle that was never touched."""
    from distributed_sac_b200 import _lib
    spec = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=128, num_tasks=4)
    R = 3
    cores, rings = [], []
    for _ in range(2):
        c = _core(spec, precision=0, replicas=R)
        rb, _tables, _fills, cap_t = _parity_ring(c, spec, False, R, seed=23)
        cores.append(c)
        rings.append(rb)
    cores[0].step_sampled(rings[0], 19)
    for _ in range(19):
        cores[1].step_sampled(rings[1], 1)

    def same(r):
        return all(torch.equal(cores[0].export_arena(w, r), cores[1].export_arena(w, r)) for w in (0, 1, 2))

    for r in range(R):
        assert same(r), f"replica {r}: 19-step graphs differ from single steps"
        for t in range(4):
            assert np.array_equal(rings[0].tree(t, r), rings[1].tree(t, r)), (r, t)
    assert torch.equal(cores[0].read_losses(19), cores[1].read_losses(19))
    rings[0].set_beta(0.3, replica=1)
    for c, rb in zip(cores, rings):
        c.step_sampled(rb, 1)
    for r in (0, 2):
        assert same(r) and torch.equal(cores[0].debug("isw", r), cores[1].debug("isw", r)), f"replica {r} changed"
    assert not torch.equal(cores[0].debug("isw", 1), cores[1].debug("isw", 1))
    assert torch.equal(cores[0].debug("idx", 1), cores[1].debug("idx", 1))
    assert not torch.equal(cores[0].export_arena(_lib.PARAMS, 1), cores[1].export_arena(_lib.PARAMS, 1))
    for c, rb in zip(cores, rings):
        rb.close()
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: the learner surface
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("family", ["LL", "MS"])
def test_learner_on_prioritized_ring(cuda, tmp_path, family, monkeypatch):
    """Learner(replay_where="device", prioritized=...): update() steps from the PER ring (weights not all 1 at beta = 1,
    priorities rewritten), set_per_beta takes effect at the next update, ReplayBuffer.sample() returns a batch, and a host
    ring with prioritized= is refused."""
    import json
    import redis_stub
    from distributed_sac_b200 import learner as L
    from distributed_sac_b200.replay_buffer import MTReplayBuffer, ReplayBuffer
    monkeypatch.chdir(tmp_path)
    per = dict(alpha=0.6, beta=0.0, eps=1e-6)
    if family == "LL":
        cfg = {"device": "cuda", "buffer_size": 1e6, "reward_scale": 1, "batch_size": 256, "gamma": 0.99, "lr_actor": 3e-4,
               "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 5000}
        make = lambda **kw: L.LunarLanderLearner(str(p), write_mode=False, buffer_size=8192,
                                                 server=redis_stub.StrictRedis(host=str(tmp_path) + family), **kw)
        buf_cls, T = ReplayBuffer, 0
    else:
        T = 4
        cfg = {"device": "cuda", "buffer_size": 8192, "reward_scale": 1, "batch_size": 128, "gamma": 0.99, "tau": 0.005,
               "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": T,
               "use_weighted_loss": True,
               "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 4, "action_bound": [-1, 1],
                         "actor_hidden_dim": [64, 64]},
               "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}
        make = lambda **kw: L.MTSACLearner(None, [f"t{i}" for i in range(T)], str(p), write_mode=False,
                                           server=redis_stub.StrictRedis(host=str(tmp_path) + family), **kw)
        buf_cls = MTReplayBuffer
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="device"):
        make(replay_where="host", prioritized=per)
    lrn = make(replay_where="device", prioritized=per)
    assert isinstance(lrn.memory, buf_cls) and lrn.memory.ring.prioritized is not None
    ring = lrn.memory.ring
    ring.fill_synthetic(8192, seed=3)
    n = 8192 // max(T, 1) * max(T, 1)
    ring.set_priorities(np.arange(n), np.random.default_rng(0).exponential(1.0, n) ** 3)
    lrn.update()
    assert (lrn.core.debug("isw") == 1).all(), "beta = 0 gives unit weights"
    lrn.set_per_beta(1.0)
    before = ring.priorities(np.arange(n))
    out = lrn.update()
    assert all(np.isfinite(out))
    w = lrn.core.debug("isw")
    assert float(w.max()) == 1.0 and float(w.min()) < 0.9, "set_per_beta did not reach the next update"
    idx = lrn.core.debug("idx").long().numpy()
    assert not np.array_equal(ring.priorities(idx), before[idx]), "update() did not rewrite the drawn priorities"
    batch = lrn.memory.sample()
    c = lrn.core.cfg
    assert [tuple(x.shape) for x in batch] == [(c.batch, c.obs_dim), (c.batch, c.act_dim), (c.batch, 1), (c.batch, c.obs_dim),
                                               (c.batch, 1)]
    assert all(torch.isfinite(x).all() for x in batch)
    lrn.memory.stop()
