"""What the test modules share: the device fixture and the handle builder, the case tables and named shapes that several
modules run, their input generators, the checkers of a step against the autograd oracle, the bit-exact Adam
specification and CPU stand-ins.  A test module takes these from here, from _golden, the oracle and the library --
never from another test module.  Shapes that differ keep distinct names even where two modules give them the same id."""
import contextlib
import dataclasses
import json
import math

import numpy as np
import pytest
import torch

import care_port as cp
import redis_stub
import sac_port as sp
from _golden import (REL, CareCase, care_core_config, check_port_state, core_config, cuda_relu_masks, kink_checked_step,
                     rel_l2, rel_scalar)

PARAMS, ADAM_M, ADAM_V, GRADS = 0, 1, 2, 3


# ---------------------------------------------------------------------------------------------------------------------
# the device and the handles
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_sac_b200 import _lib
    _lib.load()
    return torch.device("cuda", 0)


def _config(spec, care, precision, replicas=1, **hp):
    """CoreConfig of a SacSpec or (care) a CareSpec; hp: hyperparameters, the CARE-only ones dropped for plain SAC."""
    if not care:
        hp = {k: v for k, v in hp.items() if k not in ("tau_se", "lr_ctx")}
    return (care_core_config if care else core_config)(spec, replicas=replicas, precision=precision, **hp)


def _core(spec, care=False, precision=1, replicas=1, seed=0):
    from distributed_sac_b200.core import SacCore
    return SacCore(_config(spec, care, precision, replicas), 0, seed=seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pad4(x):
    return (x + 3) // 4 * 4


# ---------------------------------------------------------------------------------------------------------------------
# case tables and named shapes
# ---------------------------------------------------------------------------------------------------------------------
# The layer-chained envelope, id -> SacSpec fields.  "mainly covers" of each case, with the rows per CTA of a 132-SM H100
# at one replica (chain_fwd / chain2 / chain_bwd):
#   single   one hidden layer per network, act_dim 1, the CTA that holds both an s' row and an s row     2 / 2 / 2
#   deep8    8 hidden layers each (15-stage chain2 table, 18 critic weight-gradient jobs), widths 4, 252, 256   4 / 2 / 2
#   k32      actor input 27 and critic input 32, both evaluated directly                              8 / 4 / 2
#   k33      critic input 33: the first input layer loaded through the weight pipeline; action scale 1.5  8 / 8 / 4
#   wide_in  a 248-wide critic input (8 chunks, padded pitch), act_dim 8 (kMaxAct), action scale 2.5  8 / 4 / 2
#   tasks33  the upper half of TaskAlpha (task index 32)                                              4 / 2 / 2
#   tasks64  all 64 task slots, weighted loss                                                         4 / 2 / 2
#   big_odd  batch 531: a 19-row final weight-gradient pass, 8 rows per CTA in every chain launch     8 / 8 / 8
CHAIN_CASES = {
    "single": dict(state_dim=5, num_tasks=0, act_dim=1, actor_hidden=[36], critic_hidden=[20], batch=37),
    "deep8": dict(state_dim=9, num_tasks=0, act_dim=2, actor_hidden=[4, 12, 36, 100, 256, 252, 8, 44],
                  critic_hidden=[252, 4, 68, 256, 12, 36, 100, 20], batch=101),
    "k32": dict(state_dim=27, num_tasks=0, act_dim=5, actor_hidden=[64, 48], critic_hidden=[40, 64], batch=203),
    "k33": dict(state_dim=29, num_tasks=0, act_dim=4, actor_hidden=[64, 48], critic_hidden=[40, 64], batch=301,
                action_scale=1.5),
    "wide_in": dict(state_dim=240, num_tasks=0, act_dim=8, actor_hidden=[256, 132], critic_hidden=[196, 256], batch=203,
                    action_scale=2.5),
    "tasks33": dict(state_dim=10, num_tasks=33, act_dim=3, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=99),
    "tasks64": dict(state_dim=6, num_tasks=64, act_dim=2, actor_hidden=[48, 48], critic_hidden=[48, 48], batch=128,
                    weighted_loss=True),
    "big_odd": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[256, 252], critic_hidden=[252, 256], batch=531),
}

# The per-layer envelope, id -> SacSpec fields.  Each case is outside the chained envelope through its own shape (a hidden
# width that is not a multiple of 4 or above 256, or obs + act > 252), so precision 0 takes the per-layer plan too.
#   b1         batch 1: every GEMM on FFMA at both precisions, thin input-layer gradients, one hidden layer each
#   odd67      odd pitches everywhere (no wgmma at precision 1 either), La != Lc, the 8-column critic head at an odd batch;
#              action scale 0.4 (the scale, like the others below that are not 1, is not a power of two: act / k rounds)
#   in45       wgmma on padded first layers (critic 45 in 48, actor 41 in 44) at a batch that is not a multiple of 128
#   in17       input width 17: FFMA (not thin) in a 20-float pitch
#   mixed      precision 1 groups of wgmma-eligible and ineligible problems (one wgmma + one FFMA launch)
#   deep8      8 actor hidden layers (widths 4, 33, 260, 512), one critic hidden layer: La != Lc the other way
#   wide1024   1024-wide layers at batch 640: several column tiles, N tails of 128- and 160-wide tiles; the cost model picks
#              every tile width and split factors 4, 2 and 1
#   split517   batch 517: K slices 160/160/160/37 and head row slices 130/130/130/127; thin input-layer gradients on K slices;
#              action scale 3
#   b512n      the first sliced batch; 8-column critic head with row slices
#   pdout257   policy_dout without gradient slices, just above B * A = 2048; act_dim 8 (policy head backward NO = 16);
#              action scale 1.5
#   pdout256   B * A = 2048 exactly: the policy-head output gradient stays inside head_bwd
#   b2048      the largest batch; 64 tasks, weighted loss; NO = 16 over 512-row slices; 8-column critic head with slices
#   act1_2000  act_dim 1 with the in-kernel policy backward at row slices; a 600-deep thin input gradient (two K passes)
#   tasks33    the upper half of the task table (task index 32) in plain SAC
LAYER_CASES = {
    "b1": dict(state_dim=3, num_tasks=0, act_dim=1, actor_hidden=[37], critic_hidden=[29], batch=1),
    "odd67": dict(state_dim=11, num_tasks=0, act_dim=3, actor_hidden=[37, 61], critic_hidden=[29, 45, 53], batch=67,
                  action_scale=0.4),
    "in45": dict(state_dim=41, num_tasks=0, act_dim=4, actor_hidden=[260, 64], critic_hidden=[64, 260], batch=130),
    "in17": dict(state_dim=15, num_tasks=0, act_dim=2, actor_hidden=[260, 36], critic_hidden=[36, 260], batch=96),
    "mixed": dict(state_dim=36, num_tasks=0, act_dim=4, actor_hidden=[400, 64], critic_hidden=[24, 400], batch=256),
    "deep8": dict(state_dim=9, num_tasks=0, act_dim=2, actor_hidden=[4, 33, 260, 512, 64, 36, 100, 20], critic_hidden=[130],
                  batch=150),
    "wide1024": dict(state_dim=39, num_tasks=0, act_dim=4, actor_hidden=[1024, 520], critic_hidden=[1024, 400], batch=640),
    "split517": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[260, 96], critic_hidden=[96, 260], batch=517,
                     action_scale=3.0),
    "b512n": dict(state_dim=17, num_tasks=0, act_dim=5, actor_hidden=[96, 260], critic_hidden=[72, 131], batch=512),
    "pdout257": dict(state_dim=10, num_tasks=0, act_dim=8, actor_hidden=[64, 66], critic_hidden=[64, 66], batch=257,
                     action_scale=1.5),
    "pdout256": dict(state_dim=10, num_tasks=0, act_dim=8, actor_hidden=[64, 66], critic_hidden=[64, 66], batch=256),
    "b2048": dict(state_dim=30, num_tasks=64, act_dim=8, actor_hidden=[300, 128], critic_hidden=[128, 131], batch=2048,
                  weighted_loss=True),
    "act1_2000": dict(state_dim=12, num_tasks=0, act_dim=1, actor_hidden=[260, 64], critic_hidden=[600, 132], batch=2000),
    "tasks33": dict(state_dim=10, num_tasks=33, act_dim=3, actor_hidden=[66, 64], critic_hidden=[64, 66], batch=99),
}

# three co-scheduled replicas with parameters, minibatches and task ids of their own; at precision 1 the per-layer plan
# picks other tile widths or split factors at R = 3 than at R = 1 for this shape
REPLICA_SPEC = dict(state_dim=9, num_tasks=5, act_dim=3, actor_hidden=[400, 260], critic_hidden=[260, 130], batch=520)
REPLICAS = 3

# one hyperparameter row per replica; every field differs between rows and from the cfg defaults
ROWS = [
    dict(gamma=0.97, reward_scale=0.5, tau=0.01, lr_critic=1e-3, lr_actor=2e-4, lr_alpha=5e-3, tau_se=0.1, lr_ctx=1e-3),
    dict(gamma=0.95, reward_scale=2.0, tau=0.02, lr_critic=5e-4, lr_actor=7e-4, lr_alpha=1e-3, tau_se=0.03, lr_ctx=5e-4),
    dict(gamma=0.9, reward_scale=1.5, tau=0.1, lr_critic=2e-3, lr_actor=1e-4, lr_alpha=3e-3, tau_se=0.2, lr_ctx=2e-4),
]

# a small layer-chained learner (stream order, replica copies, refusals)
SMALL = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=128)

# named shapes (SacSpec fields).  The VSAC shape at batch 128 (VS400: n-step, prioritized, sampled) is another learner than
# the one at batch 300 (VS_LIKE: target and Adam exactness, acting).
VS400 = dict(state_dim=39, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=128)
VS_LIKE = dict(state_dim=39, num_tasks=0, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=300)
# MTSAC at T = 10 (400 wide) and T = 64, weighted loss
MT10 = dict(state_dim=39, num_tasks=10, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=320,
            weighted_loss=True)
MT64 = dict(state_dim=17, num_tasks=64, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=320,
            weighted_loss=True)
# per-layer wgmma with gradient slices (batch >= 512), without tasks and with five per-task temperatures
PER_LAYER = dict(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=640)
PER_LAYER_T5 = dict(PER_LAYER, num_tasks=5)
MTSAC_T4 = dict(state_dim=17, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=160, num_tasks=4,
                weighted_loss=True)
# MTSAC weighted loss on the per-layer FFMA plan (hidden width > 256, forked weight gradients)
MTSAC_WEIGHTED = dict(state_dim=12, act_dim=4, actor_hidden=[260, 64], critic_hidden=[264, 72], batch=200, num_tasks=4,
                      weighted_loss=True)
LL = sp.ll_spec().to_json()

# id -> (SacSpec fields, precision) of the step plans named by the hyperparameter, interval, target, Adam and acting
# tests ("chained" and "chained_ll" are one learner under the ids of two test families)
SAC_PLANS = {
    "chained": (LL, 0),
    "chained_ll": (LL, 0),
    "chained_deep8": (CHAIN_CASES["deep8"], 0),
    "chained_big_odd": (CHAIN_CASES["big_odd"], 0),
    "vs400_fp32": (VS_LIKE, 0),
    "vs400_tc": (VS_LIKE, 1),
    "split517_fp32": (LAYER_CASES["split517"], 0),
    "split517_tc": (LAYER_CASES["split517"], 1),
    "wide1024_tc": (LAYER_CASES["wide1024"], 1),
    "per_layer": (PER_LAYER_T5, 1),
    "mtsac_t10": (MT10, 1),
    "mtsac_t64": (MT64, 1),
    "mtsac_weighted": (MTSAC_WEIGHTED, 0),
}
CARE_PLANS = {"care_m": "care_small_s4", "care_o": "care_o_small_s4"}


def _plan(name):
    """(spec, care, precision) of a SAC_PLANS or CARE_PLANS id; the CARE plans run at precision 1."""
    if name in CARE_PLANS:
        return CareCase(CARE_PLANS[name]).spec, True, 1
    fields, precision = SAC_PLANS[name]
    return sp.SacSpec(**fields), False, precision


def care_t4(modified=True):
    """The CARE fixtures' learner (CARE(M) / CARE(O)) with T = 4."""
    return dataclasses.replace(CareCase("care_small_s4" if modified else "care_o_small_s4").spec, num_tasks=4)


# learner configurations: LunarLander with 10 tasks; the small LL and VS learners of _learner
LL_CFG = {"num_tasks": 10, "device": "cuda", "buffer_size": 1e6, "reward_scale": 1, "batch_size": 256, "gamma": 0.99,
          "lr_actor": 3e-4, "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "num_learn": 1, "num_time_step": 1,
          "random_step": 5000, "start_memory_len": 5000}
LEARNER_CFGS = {
    "LL": {"device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "lr_actor": 3e-4,
           "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 1000},
    "VS": {"device": "cuda", "buffer_size": 10000, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "lr_actor": 3e-4,
           "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 1000, "print_period_learner": 10,
           "update_delay": 1, "actor_hidden_dim": [64, 48], "critic_hidden_dim": [72, 40]},
}


def _learner(family, tmp_path):
    """A LunarLanderLearner ("LL") or VSACLearner ("VS") of LEARNER_CFGS on the Redis stub, not writing."""
    from distributed_sac_b200 import learner as L
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(LEARNER_CFGS[family]))
    kw = dict(write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + family))
    return (L.LunarLanderLearner if family == "LL" else L.VSACLearner)(str(p), **kw)


# ---------------------------------------------------------------------------------------------------------------------
# input generators
# ---------------------------------------------------------------------------------------------------------------------
def _params(spec, seed, care=False, move_targets=False):
    """Xavier weights, small random biases (targets distinct from the locals), and a different temperature per task, so
    that a wrong task's alpha or a wrong network's bias changes the result.  care: care_port.init_params with the mixture
    weights scaled to unit gain (randn weights grow the activations by sqrt(width) per layer -- 10^4 at nine layers).
    move_targets: every target tensor moved off its local as well, so that no target formula can pass by returning
    either operand."""
    p = (cp if care else sp).init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in p:
        if ".mix." in k and k.endswith(".W"):
            p[k] = p[k] * (2.0 / p[k].shape[1]) ** 0.5
        elif k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.num_tasks if care else spec.n_alpha, generator=g)
    if move_targets:
        g = torch.Generator().manual_seed(seed + 2000)
        for k in p:
            if "_target." in k or k.startswith("tse."):
                p[k] = p[k] + 0.02 * torch.randn(p[k].shape, generator=g)
    return p


def _eps(spec, gen):
    return torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen)


def _inputs(spec, care, R, i, noise_seed=1000, batch_seed=0):
    """Step i's minibatch and noise, [R][B][w], a different draw per replica."""
    gen = torch.Generator().manual_seed(noise_seed + i)
    mod = cp if care else sp
    bs = [mod.synthetic_batch(spec, seed=100 * i + r + batch_seed) for r in range(R)]
    b = [torch.stack([x[j] for x in bs]) for j in range(5)]
    e1, e2 = (torch.randn(R, spec.batch, spec.act_dim, generator=gen) for _ in range(2))
    return b, e1, e2


def _tasks(spec, s):
    """The task of each row of observations s (0 without tasks)."""
    return s[:, spec.state_dim:].argmax(1).numpy() if spec.num_tasks > 0 else np.zeros(len(s), np.int64)


def random_pushes(rng, n_pushes, T, streams, max_rows, plain_every=0):
    """Random interleavings: per row a stream, a task (a stream mostly keeps its task), d and cut."""
    task_of = {s: int(rng.integers(T)) for s in range(streams)}
    for p in range(n_pushes):
        n = int(rng.integers(1, max_rows + 1))
        sid = rng.integers(streams, size=n).astype(np.int32)
        for s in np.unique(sid):
            if rng.random() < 0.1:
                task_of[int(s)] = int(rng.integers(T))
        task = np.array([task_of[int(s)] for s in sid])
        d = (rng.random(n) < 0.08).astype(np.float32)
        cut = (rng.random(n) < 0.05).astype(np.uint8)
        r = rng.standard_normal(n).astype(np.float32)
        plain = plain_every and p % plain_every == plain_every - 1
        yield task, r, d, (None if plain else sid), (None if plain else cut)


def _play(rng, n_players, n_rows, time_limit):
    """Interleaved transitions of n_players environments: (player, episode, t) per row plus the pickled payloads."""
    state = [rng.standard_normal(8).astype(np.float32) for _ in range(n_players)]
    ep, t = [0] * n_players, [0] * n_players
    rows = []
    for _ in range(n_rows):
        p = int(rng.integers(n_players))
        nxt = rng.standard_normal(8).astype(np.float32)
        done = bool(rng.random() < 0.1)
        rows.append(((p, ep[p], t[p]), (state[p], rng.standard_normal(2).astype(np.float32), float(rng.standard_normal()), nxt, done)))
        t[p] += 1
        if done or t[p] == time_limit:              # a time-limit reset carries no flag: the next state just does not match
            state[p], ep[p], t[p] = rng.standard_normal(8).astype(np.float32), ep[p] + 1, 0
        else:
            state[p] = nxt
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# the step against the autograd oracle
# ---------------------------------------------------------------------------------------------------------------------
# per-row outputs of the step: debug name of the CUDA buffer == key of the port's intermediates (CARE: without the
# policy-head gradients)
ROW_OUTPUTS = ("q1", "q2", "y", "a_next", "logp_next", "a_cur", "logp_cur", "qmin", "d_action", "d_head")
CARE_ROW_OUTPUTS = ROW_OUTPUTS[:8]


def _bad_elements(got, ref):
    """|got - ref| > 1e-4 (|ref| + mean |ref|) (or not finite), and the largest |got - ref| / (|ref| + mean |ref|)."""
    got, ref = got.double().reshape(ref.shape), ref.double()
    scale = ref.abs() + ref.abs().mean()
    dev = (got - ref).abs()
    return (dev > REL * scale) | ~torch.isfinite(got), float((dev / scale.clamp_min(1e-30)).max())


def _raise_bad(what, bad, got, ref):
    rows = sorted({int(i) for i in bad.nonzero()[:, 0]})
    r, j = (int(x) for x in bad.nonzero()[0])
    raise AssertionError(f"{what}: {int(bad.sum())} elements beyond {REL} (|ref| + mean|ref|), rows {rows[:12]}"
                         f"{'...' if len(rows) > 12 else ''}; first [{r}][{j}] got {float(got[r, j]):.7g} ref {float(ref[r, j]):.7g}")


def check_rows(core, spec, o, replica=0, what="", outputs=ROW_OUTPUTS):
    """Every per-row output of the step, element by element: |got - ref| <= 1e-4 (|ref| + mean |ref|).  Returns the
    largest observed |got - ref| / (|ref| + mean |ref|)."""
    worst = 0.0
    for k in outputs:
        ref = o[k].detach().double().reshape(spec.batch, -1)
        got = core.debug(k, replica).double().reshape(ref.shape)
        bad, w = _bad_elements(got, ref)
        if bad.any():
            _raise_bad(f"{what}{k}", bad, got, ref)
        worst = max(worst, w)
    return worst


def check_losses(core, o, replica=0, what=""):
    L = core.read_losses(1)[0, replica]
    assert torch.isfinite(L).all(), f"{what}losses {L.tolist()}"
    for i, k in ((0, "critic_loss"), (1, "actor_loss"), (3, "entropy")):
        assert rel_scalar(float(L[i]), o[k]) <= REL, f"{what}{k}: {float(L[i])} vs oracle {o[k]}"


def check_active(core, spec, replica=0, what="", care=False, E=2):
    """Every hidden layer of every network (actor on s' and s, Q1/Q2 -- or the E critics of an ensemble -- on (s, a) and
    (s, a~); care: every mixture hidden layer of all three encoder instances too) has between 5 % and 95 % active units in
    the CUDA step's own masks: a sweep over dead or saturated layers would prove little."""
    for tag, m in cuda_relu_masks(core, spec, replica, care, E).items():
        if tag.startswith(("tanh:", "route:", "amin:")):
            continue
        frac = float(m.float().mean())
        assert 0.05 <= frac <= 0.95, f"{what}hidden layer {tag}: {100 * frac:.1f}% active"


def run_checked(core, spec, port, n_steps, seed, what, care=False):
    """n_steps checked steps of `core` against `port`; returns (mask bits flipped at kinks, worst per-row deviation)."""
    gen = torch.Generator().manual_seed(seed)
    flips, worst = 0, 0.0
    for i in range(n_steps):
        b = (cp if care else sp).synthetic_batch(spec, seed=seed + 100 + i)
        e1, e2 = _eps(spec, gen)
        o, f = kink_checked_step(core, port, spec, b, e1, e2, care=care, want_intermediates=True)
        flips += sum(f.values())
        tag = f"{what} step {i}: "
        check_active(core, spec, what=tag, care=care)
        check_losses(core, o, what=tag)
        check_port_state(core, port)               # after step 0, m = (1 - beta1) g: every gradient tensor as well
        worst = max(worst, check_rows(core, spec, o, what=tag, outputs=CARE_ROW_OUTPUTS if care else ROW_OUTPUTS))
    return flips, worst


def plan_labels(core):
    """Kernel labels of one eager step of `core`, sampled from a device ring (the step changes the handle's state)."""
    from distributed_sac_b200.core import Replay
    B = core.cfg.batch
    ring = Replay(core, 4 * B, "device", seed=1)
    ring.fill_synthetic(4 * B, seed=2)
    labels = [n for n, _ in core.profile_step(ring, iters=1)]
    ring.close()
    return labels


def _launches(spec, unfused=False):
    """launches_per_step of a handle for `spec` (exact fp32); unfused: created with B200SAC_FUSE=0."""
    from distributed_sac_b200.core import SacCore
    with pytest.MonkeyPatch.context() as mp:
        if unfused:
            mp.setenv("B200SAC_FUSE", "0")
        core = SacCore(core_config(spec, precision=0), 0, seed=0)
        n = core.launches_per_step
        core.close()
    return n


@pytest.fixture(scope="module")
def chained_launches(cuda):
    """Launches per step of the layer-chained plan (a LunarLander learner), distinct from that learner's per-layer plan."""
    n = _launches(sp.ll_spec())
    assert n != _launches(sp.ll_spec(), unfused=True)
    return n


def chain_rows(rows, groups, R, sms):
    """Rows per CTA of a chain launch (mirror of chain_rows in b200sac.cu): the fewest of 8 / 4 / 2 whose launch of
    groups x ceil(rows / ROWS) CTAs per replica stays within one CTA per SM."""
    bn = 8
    for r in (4, 2):
        if groups * -(-rows // r) * R <= sms:
            bn = r
    return bn


def plan_rows(B, R, sms):
    """{launch: rows per CTA}: chain_fwd runs actor [s';s] + Q1 + Q2 (4B rows, one group), chain2 the twins (B rows, two
    groups), chain_bwd the policy backward (B rows)."""
    return dict(chain_fwd=chain_rows(4 * B, 1, R, sms), chain2=chain_rows(B, 2, R, sms), chain_bwd=chain_rows(B, 1, R, sms))


# ---------------------------------------------------------------------------------------------------------------------
# exactness: parameters as bit patterns, the handles of the exact tests, the Adam specification and its check
# ---------------------------------------------------------------------------------------------------------------------
SLOT_OF_OPT = {0: 0, 1: 1, 2: 2, 3: 4}          # layout table "opt" -> Counters slot
LR_OF_SLOT = {0: "lr_critic", 1: "lr_actor", 2: "lr_alpha", 4: "lr_ctx"}
SLOT_NAME = {0: "critic", 1: "actor", 2: "temperature", 4: "context encoder"}


def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def export(core, replica=0):
    return core.export_arena(PARAMS, replica).numpy().copy()


def _handle(name, R=1, rows=None, seed=0):
    """(core, spec, care) of a _plan id with each replica's own parameters (targets off their locals) and, if given, its
    own hyperparameter row."""
    spec, care, precision = _plan(name)
    core = _core(spec, care, precision, R, seed=seed)
    for r in range(R):
        core.set_named(_params(spec, 11 + 7 * r, care, move_targets=True), PARAMS, r)
        if rows is not None:
            core.set_hparams(r, **rows[r])
    return core, spec, care


def adam_expect(p, m, v, g, lr, b1p, b2p, beta1=0.9, beta2=0.999, eps=1e-8, mode="fp32"):
    """(p', m', v') of adam_scalars + adam_one: step_size = f32(lr / (1 - b1p)) and bc2_sqrt = f32(sqrt(1 - b2p)) in fp64,
    then m' = m + w1*(g - m), v' = v*b2 + (omb2*g)*g, p' = p - step_size*(m' / (sqrtf(v')/bc2_sqrt + eps)), one fp32
    rounding per operation.  mode "fp64": the same formula evaluated in fp64 and rounded once; mode "fma": the multiply-adds
    contracted (the two diagnostics a failing element is tested against)."""
    f = np.float32
    step_size, bc2_sqrt = f(lr / (1.0 - b1p)), f(math.sqrt(1.0 - b2p))
    w1, b2, omb2, e = f(1.0 - beta1), f(beta2), f(1.0 - beta2), f(eps)
    p, m, v, g = (np.asarray(x, dtype=np.float32) for x in (p, m, v, g))
    if mode == "fp64":
        d = np.float64
        m1 = m + d(w1) * (g.astype(d) - m)
        v1 = v * d(b2) + (d(omb2) * g) * g
        p1 = p - d(step_size) * (m1 / (np.sqrt(v1) / d(bc2_sqrt) + d(e)))
        return p1.astype(f), m1.astype(f), v1.astype(f)
    if mode == "fma":
        d = np.float64
        m1 = (d(w1) * (g - m) + m).astype(f)
        v1 = ((omb2 * g).astype(d) * g + v * b2).astype(f)
        q = m1 / (np.sqrt(v1) / bc2_sqrt + e)
        return (p.astype(d) - d(step_size) * q).astype(f), m1, v1
    m1 = m + w1 * (g - m)
    v1 = v * b2 + (omb2 * g) * g
    p1 = p - step_size * (m1 / (np.sqrt(v1) / bc2_sqrt + e))
    return p1, m1, v1


class Counts:
    """fp64 model of one replica's Counters: Adam step and bias-correction products per slot (0 critic, 1 actor,
    2 temperature, 4 context encoder)."""

    def __init__(self, beta1, beta2):
        self.beta1, self.beta2 = beta1, beta2
        self.t, self.b1p, self.b2p = [0] * 5, [1.0] * 5, [1.0] * 5

    def seed(self, steps):
        """b200sac_set_steps: (critic, actor, alpha, context encoder) -> glibc pow, as on the host side"""
        for i, s in enumerate(steps):
            slot = 4 if i == 3 else i
            self.t[slot] = int(s)
            self.b1p[slot], self.b2p[slot] = math.pow(self.beta1, s), math.pow(self.beta2, s)

    def bump(self, actor_every=1):
        """bump_counters: every slot but actor and temperature on a critic-only step; returns 'actor step'."""
        n = self.t[0] + 1
        act = actor_every == 1 or n % actor_every == 0
        for i in range(5):
            if act or i not in (1, 2):
                self.t[i] += 1
                self.b1p[i] *= self.beta1
                self.b2p[i] *= self.beta2
        return act

    def copy(self):
        c = Counts(self.beta1, self.beta2)
        c.t, c.b1p, c.b2p = list(self.t), list(self.b1p), list(self.b2p)
        return c

    def steps(self, n):
        return tuple(self.t[i] for i in (0, 1, 2, 4))[:n]


def new_model(core):
    return [Counts(core.cfg.beta1, core.cfg.beta2) for _ in range(core.cfg.replicas)]


def _slots(core):
    """(slot of every trainable float, -1 in the gaps; [(name, offset, floats, slot)] of the trainable tensors)"""
    if not hasattr(core, "_adam_slots"):
        slot = np.full(core.trainable_floats, -1, np.int8)
        tensors = []
        for name, (off, rows, _cols, tr, opt, pitch) in core.table.items():
            if tr:
                slot[off:off + rows * pitch] = SLOT_OF_OPT[opt]
                tensors.append((name, off, rows * pitch, SLOT_OF_OPT[opt]))
        core._adam_slots = (slot, tensors)
    return core._adam_slots


def snapshot(core, r, with_grads=False):
    """(p[:trainable], m, v[, GRADS]) of replica r as numpy arrays"""
    T = core.trainable_floats
    out = [export(core, r)[:T], core.export_arena(ADAM_M, r).numpy().copy(), core.export_arena(ADAM_V, r).numpy().copy()]
    if with_grads:
        out.append(core.export_arena(GRADS, r).numpy().copy())
    return out


def _slice0(core, r):
    """The gradient arena without the extra split-K slices (b200sac_read_range reads slice 0 only)."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import _ptr, _stream
    out = torch.empty(core.trainable_floats)
    _lib.check(core.lib.b200sac_read_range(core._h, GRADS, r, 0, core.trainable_floats, _ptr(out), _stream()))
    return out.numpy()


def _candidates(core, model, r, s, before, g, sel):
    """{mistake: (p', m', v')} for the elements sel of slot s of replica r"""
    cfg, c = core.cfg, model[r]
    hp = core.get_hparams(r)
    pb, mb, vb = (x[sel] for x in before)
    ex = lambda lr, b1p, b2p, gg=None, mode="fp32": None if b1p >= 1.0 else adam_expect(    # (count 0: no step uses it)
        pb, mb, vb, g[sel] if gg is None else gg, lr, b1p, b2p, cfg.beta1, cfg.beta2, cfg.adam_eps, mode)
    lr, b1p, b2p = hp[LR_OF_SLOT[s]], c.b1p[s], c.b2p[s]
    out = {"no update": (pb, mb, vb)}
    for s2 in (0, 1, 2, 4):
        if s2 != s:
            out[f"the {SLOT_NAME[s2]} slot's rate and count"] = ex(hp[LR_OF_SLOT[s2]], c.b1p[s2], c.b2p[s2])
            out[f"the {SLOT_NAME[s2]} slot's count"] = ex(lr, c.b1p[s2], c.b2p[s2])
    for q in range(cfg.replicas):
        if q != r:
            out[f"replica {q}'s {LR_OF_SLOT[s]}"] = ex(core.get_hparams(q)[LR_OF_SLOT[s]], b1p, b2p)
            out[f"replica {q}'s count"] = ex(lr, model[q].b1p[s], model[q].b2p[s])
    out["count t - 1"] = ex(lr, b1p / cfg.beta1, b2p / cfg.beta2)
    out["count t + 1"] = ex(lr, b1p * cfg.beta1, b2p * cfg.beta2)
    out["pow(beta, t) instead of the running product"] = ex(lr, math.pow(cfg.beta1, c.t[s]), math.pow(cfg.beta2, c.t[s]))
    out["the gradient without its split-K slices"] = ex(lr, b1p, b2p, _slice0(core, r)[sel])
    out["fp64 evaluation"] = ex(lr, b1p, b2p, mode="fp64")
    out["FMA-contracted evaluation"] = ex(lr, b1p, b2p, mode="fma")
    return {k: c for k, c in out.items() if c is not None}


def check_adam(core, model, r, before, after, act, what):
    """Every trainable element of replica r after one step == adam_expect of its slot (actor and temperature untouched on
    a critic-only step), p, m and v bit for bit; the gaps between tensors unchanged.  model[r] holds the counters the step
    used (bumped).  Returns {slot: elements whose parameter moved}."""
    cfg = core.cfg
    slot, tensors = _slots(core)
    hp = core.get_hparams(r)
    got = after[:3]
    g = after[3]
    want = [np.empty_like(x) for x in before]
    for s in (0, 1, 2, 4):
        sel = slot == s
        if not sel.any():
            continue
        if s in (1, 2) and not act:
            res = [x[sel] for x in before]
        else:
            res = adam_expect(before[0][sel], before[1][sel], before[2][sel], g[sel], hp[LR_OF_SLOT[s]], model[r].b1p[s],
                              model[r].b2p[s], cfg.beta1, cfg.beta2, cfg.adam_eps)
        for w, x in zip(want, res):
            w[sel] = x
    gap = slot < 0
    for w, b in zip(want, before):
        w[gap] = b[gap]
    bad = []
    for name, off, n, s in tensors:
        sl = slice(off, off + n)
        diff = np.zeros(n, bool)
        for x, w in zip(got, want):
            diff |= _bits(x[sl]) != _bits(w[sl])
        if not diff.any():
            continue
        sel = np.zeros(core.trainable_floats, bool)
        sel[sl] = True
        cands = _candidates(core, model, r, s, before, g, sel)
        hit = [k for k, c in cands.items() if all(np.array_equal(_bits(x[sl]), _bits(y)) for x, y in zip(got, c))]
        i = int(np.argmax(diff))
        bad.append(f"{name} ({SLOT_NAME[s]} slot, t = {model[r].t[s]}, {LR_OF_SLOT[s]} = {hp[LR_OF_SLOT[s]]}; it got "
                   f"{' / '.join(hit) or 'no candidate'}): {int(diff.sum())} of {n} elements differ, first [{i}] "
                   f"g = {g[off + i]!r}: (p, m, v) = {tuple(float(x[off + i]) for x in got)} want "
                   f"{tuple(float(w[off + i]) for w in want)}")
    assert not bad, f"{what}: " + "; ".join(bad[:6])
    changed = gap & ((_bits(got[0]) != _bits(before[0])) | (_bits(got[1]) != _bits(before[1])) |
                     (_bits(got[2]) != _bits(before[2])))
    assert not changed.any(), f"{what}: {int(changed.sum())} floats between tensors changed, first [{int(np.argmax(changed))}]"
    return {s: int(((slot == s) & (got[0] != before[0])).sum()) for s in (0, 1, 2, 4) if (slot == s).any()}


def capture_grads(port):
    """{name: gradient} as each optimizer's step() consumes it (the critic's before pi_loss.backward() adds to it)."""
    grads = {}
    names = {id(t): k for k, t in port.p.items()}
    for opt in (port.opt_critic, port.opt_actor, port.opt_alpha, getattr(port, "opt_ctx", None)):
        if opt is None:
            continue

        def step(*a, _opt=opt, _orig=opt.step, **kw):
            for grp in _opt.param_groups:
                for t in grp["params"]:
                    grads[names[id(t)]] = torch.zeros_like(t) if t.grad is None else t.grad.detach().clone()
            return _orig(*a, **kw)
        opt.step = step
    return grads


def check_grads(core, ref, what, r=0):
    """GRADS == the oracle's consumed gradients to 1e-4 per tensor (log_alpha: or 1e-6 absolute)."""
    got = core.get_named(GRADS, r)
    bad = []
    for k, g in got.items():
        assert k in ref, f"{what}: the oracle has no gradient for {k}"
        err = rel_l2(g, ref[k].reshape(g.shape))
        if err > REL and not (k == "log_alpha" and float((g - ref[k].reshape(g.shape)).abs().max()) <= 1e-6):
            bad.append((k, float(f"{err:.2e}")))
    assert not bad, f"{what}: gradients differ from the oracle's beyond {REL} (CUDA masks forced): {bad[:8]}"
    return len(got)


# ---------------------------------------------------------------------------------------------------------------------
# CPU stand-ins
# ---------------------------------------------------------------------------------------------------------------------
class BlobStubLib:
    """CPU stand-in for b200sac_blob_*: emulates the device gather (payload float j = arena[src[j]] -> image bytes at dst[j])."""

    def __init__(self, arena):
        self.arena = arena

    def b200sac_blob_template(self, h, replica, image, image_bytes, n_floats, src, dst):
        import ctypes as C
        import numpy as np
        self.image = np.ctypeslib.as_array(C.cast(image, C.POINTER(C.c_uint8)), shape=(image_bytes,)).copy()
        self.src = np.ctypeslib.as_array(C.cast(src, C.POINTER(C.c_int32)), shape=(n_floats,)).copy()
        self.dst = np.ctypeslib.as_array(C.cast(dst, C.POINTER(C.c_int32)), shape=(n_floats,)).copy()
        return 0

    def b200sac_blob_begin(self, h, stream):
        import numpy as np
        out = self.image.copy()
        vals = np.ascontiguousarray(self.arena[self.src], dtype=np.float32).view(np.uint8).reshape(-1, 4)
        for b in range(4):
            out[self.dst + b] = vals[:, b]
        self.out = out
        return 0

    def b200sac_blob_wait(self, h, ptr, n):
        import ctypes as C
        C.cast(ptr, C.POINTER(C.c_void_p))[0] = self.out.ctypes.data
        C.cast(n, C.POINTER(C.c_int64))[0] = self.out.size
        return 0


# ---------------------------------------------------------------------------------------------------------------------
# stream order
# ---------------------------------------------------------------------------------------------------------------------
def _stream_run(mode, change, sync_before_change, result):
    """16 sampled steps of a SMALL learner at R = 2 from a ring: mode "stream" enqueues them on a torch side stream,
    "legacy" on the legacy default stream (bridged onto the handle's own stream), "host" runs them one b200sac_update
    each from a pinned-host ring.  change(core), unless None, is enqueued right behind step 8 (after a synchronisation
    if sync_before_change); returns result(core) after step 16."""
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(SMALL, replicas=2), 0, seed=7)
    rb = Replay(core, capacity=4096, where="host" if mode == "host" else "device", seed=3)
    stream = torch.cuda.Stream() if mode == "stream" else None
    with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
        rb.fill_synthetic(4096, seed=9)
        core.prepare(rb)

        def eight():
            if mode == "host":
                for _ in range(8):
                    core.update_sampled(rb)          # b200sac_update: one staged-graph step + its losses
            else:
                core.step_sampled(rb, 8)             # one 8-step graph launch
        eight()
        if sync_before_change:
            torch.cuda.synchronize()
        if change is not None:
            change(core)
        eight()
        out = result(core)
    rb.close()
    core.close()
    return out
