"""Batched inference (b200sac_act, the path players run) over the step envelopes, against the autograd oracle, and the
guarantee that acting never changes training.

The plain SAC / MTSAC act path is: the pitched copy of the observation rows into XA, one gemm_simt_kernel launch per actor
layer, policy_head_kernel on rows [0, n) (rows at or above the batch write the actor-pass buffer XP, a partial last CTA
takes the final n % 8 rows; the head GEMV walks its input in 128-wide rounds) and, for the LunarLander actor's
deterministic action, act_scaled_mu_kernel.  Every case of the chained and per-layer envelopes (the latter at both
precisions) and three replicas with parameters of their own act at every replica, at n in {1, 7, B, B + 1, 2B - 1, 2B},
with injected noise, stochastic = 0 (k tanh(mu)), stochastic = -1 (k mu) and fresh noise.  The masks act used (its own
"hA.<l>" rows) and its tanh(u) are forced into the oracle, the noise it drew is read back (psave entry 5), and actions and
per-row log-probabilities are compared element by element at the envelopes' bar.  test_cases_reach_every_act_branch names
any branch the cases stop reaching.

Acting writes into the step's own work buffers (XA, hA, XT / XP, eps, psave, logp, the action buffer; CARE also XS and the
task ids).  test_acting_never_changes_training runs one training sequence twice, once with act calls between every pair of
step calls of every entry point, and demands bit-identical learner state.
"""
import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import REL, check_forced, core_config
from _harness import CHAIN_CASES, LAYER_CASES, REPLICA_SPEC, REPLICAS, _core, _inputs, _params, _plan, cuda

gpu = pytest.mark.gpu

PARAMS, ADAM_M, ADAM_V = 0, 1, 2

# id -> (SacSpec fields, precision, replicas)
ACT_CASES = {f"chain_{k}": (v, 0, 1) for k, v in CHAIN_CASES.items()}
ACT_CASES.update({f"layer_{k}_{tag}": (v, p, 1) for k, v in LAYER_CASES.items() for p, tag in ((0, "fp32"), (1, "tc"))})
ACT_CASES["replicas3"] = (REPLICA_SPEC, 1, REPLICAS)

MODES = ("eps", "det", "mu", "fresh")          # injected noise, k tanh(mu), k mu, fresh Philox noise


def row_counts(B):
    return sorted({min(max(n, 1), 2 * B) for n in (1, 7, B, B + 1, 2 * B - 1, 2 * B)})


def _obs(spec, seed):
    """2B observation rows (task one-hots included): [s ; s'] of a synthetic minibatch."""
    s, _a, _r, s2, _d = sp.synthetic_batch(spec, seed=seed)
    return torch.cat([s, s2])


def _act(core, obs, mode, eps, replica):
    return core.act(obs, stochastic={"eps": True, "det": False, "mu": False, "fresh": True}[mode], eps=eps,
                    replica=replica, no_tanh=(mode == "mu"))


def act_noise(core, spec, n, replica):
    """The noise the last act call used for rows [0, n): psave entry 5."""
    return core.debug("psave", replica).reshape(2 * spec.batch, spec.act_dim, 8)[:n, :, 5]


def act_masks(core, spec, n, replica):
    """{ReluTape tag: what act used} -- the sign patterns of its own hidden activations and its tanh(u)."""
    B = spec.batch
    m = {f"actor:act:{l}": core.debug(f"hA.{l}", replica).reshape(2 * B, H)[:n] > 0 for l, H in enumerate(spec.actor_hidden)}
    t = core.debug("psave", replica).reshape(2 * B, spec.act_dim, 8)[:n, :, 2]
    # the reference takes log(k (1 - (a / k)^2 + 1e-6)) of its fp32 action a = k tanh(u); where tanh saturates, a / k as
    # fp32 rounds it decides that term, so the fp64 oracle continues with that value (== tanh(u) at k = 1)
    k = torch.tensor(spec.action_scale, dtype=torch.float32)
    m["tanh:act"] = ((k * t) / k).double()
    return m


def close_rows(got, ref, what):
    """|got - ref| <= 1e-4 (|ref| + mean |ref|) element by element; returns the largest |got - ref| / (|ref| + mean |ref|)."""
    got, ref = got.double().reshape(ref.shape), ref.detach().double()
    scale = ref.abs() + ref.abs().mean()
    dev = (got - ref).abs()
    bad = (dev > REL * scale) | ~torch.isfinite(got)
    if bad.any():
        i = tuple(int(x) for x in bad.nonzero()[0])
        rows = sorted({int(x) for x in bad.nonzero()[:, 0]})
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond {REL} (|ref| + mean|ref|), rows {rows[:12]}; first "
                             f"{list(i)} got {float(got[i]):.7g} ref {float(ref[i]):.7g}")
    return float((dev / scale.clamp_min(1e-30)).max())


def check_act(core, spec, p64, obs, got, mode, eps, replica, what):
    """One act call against the oracle with act's masks, tanh(u) and noise forced; returns (forced bits that differed,
    worst deviation)."""
    n, A = obs.shape[0], spec.act_dim
    used = act_noise(core, spec, n, replica)
    if mode == "eps":
        assert torch.equal(used, eps), f"{what}: the head did not use the injected noise"
    elif mode in ("det", "mu"):
        assert (used == 0).all(), f"{what}: deterministic action with nonzero noise"
    forced = act_masks(core, spec, n, replica)
    x = obs.double()
    with sp.ReluTape(forced) as tape:
        with torch.no_grad():
            ref, logp, _ = sp.policy_sample(spec, p64, x, used.double(), tag="act")
            if mode == "mu":
                ref = spec.action_scale * sp.mlp(p64, "actor", x, "act")[:, :A]
    flips = sum(check_forced(tape, forced, f"{what}: ").values())
    got_logp = torch.cat([core.debug("logp_next", replica), core.debug("logp_cur", replica)])[:n]
    worst = close_rows(got, ref, f"{what} actions")
    worst = max(worst, close_rows(got_logp, logp.reshape(-1), f"{what} log-probs"))
    assert got.abs().max() <= spec.action_scale * (1 + 1e-6) or mode == "mu", f"{what}: |action| beyond the action scale"
    return flips, worst


# ---------------------------------------------------------------------------------------------------------------------
# 1: every case, every replica, every row count and mode, element by element against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", list(ACT_CASES))
def test_act_matches_oracle(cuda, name):
    from distributed_sac_b200.core import SacCore
    fields, precision, R = ACT_CASES[name]
    spec = sp.SacSpec(**fields)
    B, A = spec.batch, spec.act_dim
    core = SacCore(core_config(spec, replicas=R, precision=precision), 0, seed=0)
    params = [_params(spec, seed=40 + r) for r in range(R)]
    for r in range(R):
        core.set_named(params[r], PARAMS, r)
    obs_all = _obs(spec, seed=77)
    gen = torch.Generator().manual_seed(5)
    flips, worst = 0, 0.0
    for r in range(R):
        p64 = {k: v.double() for k, v in params[r].items()}
        for n in row_counts(B):
            obs = obs_all[:n]
            for mode in MODES:
                eps = torch.randn(n, A, generator=gen) if mode == "eps" else None
                got = _act(core, obs, mode, eps, r)
                f, w = check_act(core, spec, p64, obs, got, mode, eps, r, f"{name} replica {r} n = {n} {mode}")
                flips, worst = flips + f, max(worst, w)
                if n == 2 * B and mode == "eps":
                    for tag, m in act_masks(core, spec, n, r).items():       # guard: no dead or saturated layer
                        if tag.startswith("actor:"):
                            frac = float(m.float().mean())
                            assert 0.05 <= frac <= 0.95, f"{name} replica {r}: act's {tag} is {100 * frac:.1f}% active"
    if R > 1:
        # replica r of the R-replica handle == an R = 1 handle holding replica r's parameters, bit for bit
        single = SacCore(core_config(spec, precision=precision), 0, seed=0)
        for r in range(R):
            single.set_named(params[r])
            for n in (7, 2 * B):
                eps = torch.randn(n, A, generator=gen)
                a_r, a_1 = core.act(obs_all[:n], eps=eps, replica=r), single.act(obs_all[:n], eps=eps)
                assert torch.equal(a_r.view(torch.int32), a_1.view(torch.int32)), f"replica {r} n = {n}: differs from R = 1"
        single.close()
    for bad_n, bad_r in ((0, 0), (2 * B + 1, 0), (1, R)):
        with pytest.raises(RuntimeError):
            core.act(torch.zeros(bad_n, spec.obs_dim), replica=bad_r)
    core.close()
    print(f"[act] {name}: {flips} forced mask bits differed (all at numerically-zero pre-activations); largest per-element "
          f"|got - ref| / (|ref| + mean|ref|) = {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 2: the fresh noise -- N(0, 1), independent, not the training step's, reproducible
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_fresh_noise_statistics(cuda):
    from scipy import stats
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(**REPLICA_SPEC)
    B, A, R = spec.batch, spec.act_dim, 2
    obs = _obs(spec, seed=3)

    def handle():
        core = SacCore(core_config(spec, replicas=R, precision=1), 0, seed=9)
        for r in range(R):
            core.set_named(_params(spec, seed=60 + r), PARAMS, r)
        return core

    def draw(core, r):
        core.act(obs, replica=r)
        return act_noise(core, spec, 2 * B, r).clone()

    a = handle()
    seq = [draw(a, r) for _ in range(2) for r in range(R)]        # call order: (0, r0), (0, r1), (1, r0), (1, r1)
    z = torch.stack(seq).double()
    N = z.numel()
    flat = z.reshape(-1).numpy()
    assert stats.kstest(flat, "norm").pvalue > 1e-3, "fresh act noise is not N(0, 1) (KS)"
    assert abs(flat.mean()) < 5 / N ** 0.5 and abs(flat.var() - 1) < 5 * (2 / N) ** 0.5, (flat.mean(), flat.var())
    assert abs(stats.skew(flat)) < 5 * (6 / N) ** 0.5 and abs(stats.kurtosis(flat)) < 5 * (24 / N) ** 0.5

    def corr(x, y):
        x, y = x.reshape(-1).double(), y.reshape(-1).double()
        return float(torch.corrcoef(torch.stack([x, y]))[0, 1])

    lim = lambda m: 5 / m ** 0.5
    for k, e in enumerate(seq):
        assert abs(corr(e[1:], e[:-1])) < lim(e[1:].numel()), f"draw {k}: successive rows correlated"
        if A > 1:
            assert abs(corr(e[:, 1:], e[:, :-1])) < lim(e[:, 1:].numel()), f"draw {k}: successive actions correlated"
    assert abs(corr(seq[0], seq[2])) < lim(seq[0].numel()), "successive calls on one replica correlated"
    assert abs(corr(seq[0], seq[1])) < lim(seq[0].numel()), "replicas 0 and 1 correlated"
    for i in range(len(seq)):
        for j in range(i):
            assert not torch.equal(seq[i], seq[j]), f"draws {j} and {i} are equal"

    # the training step's in-kernel noise at the same step index is a different stream
    act_before = draw(a, 0)
    b, _e1, _e2 = _inputs(spec, False, R, 0)
    a.step(*b)
    step_noise = act_noise(a, spec, 2 * B, 0)
    assert not torch.equal(act_before, step_noise)
    assert abs(corr(act_before, step_noise)) < lim(act_before.numel()), "act's noise correlates with the step's"
    act_after = draw(a, 0)
    assert abs(corr(act_after, step_noise)) < lim(act_after.numel())

    # the same seed and call sequence draw the same noise, bit for bit
    c = handle()
    seq_c = [draw(c, r) for _ in range(2) for r in range(R)]
    assert all(torch.equal(x, y) for x, y in zip(seq, seq_c)), "same seed and call sequence, different noise"
    assert torch.equal(draw(c, 0), act_before)
    c.step(*b)
    assert torch.equal(act_noise(c, spec, 2 * B, 0), step_noise)
    assert torch.equal(draw(c, 0), act_after)
    a.close()
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: the cases reach every branch of the act path (CPU)
# ---------------------------------------------------------------------------------------------------------------------
ACT_BRANCHES = {
    "a partial last head CTA (n % 8 != 0)": lambda spec, n: n % 8 != 0,
    "rows at or above the batch (n > B: the XP branch)": lambda spec, n: n > spec.batch,
    "a head input wider than 128 and not a multiple of 32": lambda spec, n: spec.actor_hidden[-1] > 128 and spec.actor_hidden[-1] % 32 != 0,
    "act_dim 1": lambda spec, n: spec.act_dim == 1,
    "act_dim 8": lambda spec, n: spec.act_dim == 8,
    "one actor hidden layer": lambda spec, n: len(spec.actor_hidden) == 1,
    "eight actor hidden layers": lambda spec, n: len(spec.actor_hidden) == 8,
    "more than one replica": lambda spec, n: False,
}


def test_cases_reach_every_act_branch():
    have = set()
    for fields, _precision, R in ACT_CASES.values():
        spec = sp.SacSpec(**fields)
        for n in row_counts(spec.batch):
            have |= {k for k, rule in ACT_BRANCHES.items() if rule(spec, n)}
        if R > 1:
            have.add("more than one replica")
    missing = sorted(set(ACT_BRANCHES) - have)
    assert not missing, f"no act case reaches: {missing}"


# ---------------------------------------------------------------------------------------------------------------------
# 4: acting never changes training, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
NI_PLANS = ["chained_ll", "vs400_tc", "mtsac_t10", "care_m", "care_o"]         # _harness._plan ids


def _ni_handle(name, R):
    from distributed_sac_b200.core import Replay
    spec, care, precision = _plan(name)
    core = _core(spec, care, precision, R, seed=4)
    for r in range(R):
        core.set_named((cp if care else sp).init_params(spec, seed=20 + r), PARAMS, r)
    cap = 8 * spec.batch
    rings = {}
    for where in ("device", "host"):
        rings[where] = Replay(core, cap, where, seed=8)
        rings[where].fill_synthetic(cap, seed=9)
    return core, spec, care, rings


@gpu
@pytest.mark.parametrize("name", NI_PLANS)
def test_acting_never_changes_training(cuda, name):
    R = 2
    plain, spec, care, rings_p = _ni_handle(name, R)
    acting, _, _, rings_a = _ni_handle(name, R)
    B, A = spec.batch, spec.act_dim
    b0 = (cp if care else sp).synthetic_batch(spec, seed=31)
    obs = b0[0] if care else torch.cat([b0[0], b0[3]])
    gen = torch.Generator().manual_seed(6)
    calls = [0]

    def act(core):
        if core is plain:
            return
        for r in range(R):
            for n in ((B, 1) if care else (2 * B, 1)):
                for mode in MODES:
                    _act(core, obs[:n], mode, torch.randn(n, A, generator=gen) if mode == "eps" else None, r)
                    calls[0] += 1

    n_steps = 0
    for core, rings in ((plain, rings_p), (acting, rings_a)):
        n_steps = 0
        act(core)
        for i in range(2):                                   # b200sac_step, injected noise and in-kernel noise
            b, e1, e2 = _inputs(spec, care, R, i)
            core.step(*b, *((e1, e2) if i == 0 else ()))
            act(core)
        for i in range(2, 4):                                # b200sac_step_host
            b, e1, e2 = _inputs(spec, care, R, i)
            core.step_host(*b, *((e1, e2) if i == 2 else ()), want_losses=False)
            act(core)
        n_steps += 4
        core.prepare(rings["device"])                       # device ring: runs cut into 8-, 4-, 2- and 1-step graphs
        for k in (15, 1, 3, 2):
            core.step_sampled(rings["device"], k)
            n_steps += k
            act(core)
        for k in (1, 1, 2, 1):                               # pinned-host ring: the next minibatch is prefetched
            core.step_sampled(rings["host"], k)
            n_steps += k
            act(core)
    assert calls[0] > 0
    torch.cuda.synchronize()
    for r in range(R):
        for which, label in ((PARAMS, "parameters"), (ADAM_M, "Adam m"), (ADAM_V, "Adam v")):
            x, y = plain.export_arena(which, r), acting.export_arena(which, r)
            diff = x.view(torch.int32) != y.view(torch.int32)
            if diff.any():
                i = int(diff.nonzero()[0])
                owner = [k for k, d in plain.table.items() if d[0] <= i < d[0] + d[1] * d[5]]
                raise AssertionError(f"{name} replica {r}: acting changed {int(diff.sum())} floats of the {label}, first "
                                     f"[{i}] ({owner})")
        assert plain.get_steps(r) == acting.get_steps(r), r
    Lp, La = plain.read_losses(n_steps), acting.read_losses(n_steps)
    assert torch.equal(Lp.view(torch.int32), La.view(torch.int32)), f"{name}: acting changed the loss ring"
    for core, rings in ((plain, rings_p), (acting, rings_a)):
        for ring in rings.values():
            ring.close()
        core.close()
