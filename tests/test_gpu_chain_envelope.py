"""GPU: the layer-chained step (chain.cuh, chain2.cuh; build_plan_fused in b200sac.cu) over its whole eligibility envelope
against the autograd oracle.

The chained plan takes every exact-fp32, non-CARE learner whose hidden widths are multiples of 4 and at most 256, with at
most 8 hidden layers per network and state + tasks + act <= 252.  The cases below walk the edges of that space, where the
kernels branch: a CTA that gets fewer rows than its rows per CTA (odd batches), one hidden layer (no directly evaluated
input layer, a policy backward without dense stages), eight hidden layers (the longest stage tables), width-4 and 252/256-wide
layers, input widths 32 / 33 / 248, act_dim 1 and 8, more than 32 tasks, and co-scheduled replicas with parameters of their
own.  Every step is checked with the masks of the CUDA step forced into the oracle (tests/_golden.py::kink_checked_step):
losses, every parameter / target / Adam moment, and every per-row output of the step element by element, so that a single
wrong tail row fails.
"""
import pytest
import torch

import sac_port as sp
from _golden import (REL, check_forced, check_port_state, core_config, cuda_relu_masks, kink_checked_step, rel_scalar,
                     sync_core_to_port)

pytestmark = pytest.mark.gpu

# id -> SacSpec fields.  "mainly covers" of each case, with the rows per CTA of a 132-SM H100 at one replica
# (chain_fwd / chain2 / chain_bwd):
#   single   one hidden layer per network, act_dim 1, the CTA that holds both an s' row and an s row     2 / 2 / 2
#   deep8    8 hidden layers each (15-stage chain2 table, 18 critic weight-gradient jobs), widths 4, 252, 256   4 / 2 / 2
#   k32      actor input 27 and critic input 32, both evaluated directly                              8 / 4 / 2
#   k33      critic input 33: the first input layer loaded through the weight pipeline                 8 / 8 / 4
#   wide_in  a 248-wide critic input (8 chunks, padded pitch), act_dim 8 (kMaxAct)                    8 / 4 / 2
#   tasks33  the upper half of TaskAlpha (task index 32)                                              4 / 2 / 2
#   tasks64  all 64 task slots, weighted loss                                                         4 / 2 / 2
#   big_odd  batch 531: a 19-row final weight-gradient pass, 8 rows per CTA in every chain launch     8 / 8 / 8
CASES = {
    "single": dict(state_dim=5, num_tasks=0, act_dim=1, actor_hidden=[36], critic_hidden=[20], batch=37),
    "deep8": dict(state_dim=9, num_tasks=0, act_dim=2, actor_hidden=[4, 12, 36, 100, 256, 252, 8, 44],
                  critic_hidden=[252, 4, 68, 256, 12, 36, 100, 20], batch=101),
    "k32": dict(state_dim=27, num_tasks=0, act_dim=5, actor_hidden=[64, 48], critic_hidden=[40, 64], batch=203),
    "k33": dict(state_dim=29, num_tasks=0, act_dim=4, actor_hidden=[64, 48], critic_hidden=[40, 64], batch=301),
    "wide_in": dict(state_dim=240, num_tasks=0, act_dim=8, actor_hidden=[256, 132], critic_hidden=[196, 256], batch=203),
    "tasks33": dict(state_dim=10, num_tasks=33, act_dim=3, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=99),
    "tasks64": dict(state_dim=6, num_tasks=64, act_dim=2, actor_hidden=[48, 48], critic_hidden=[48, 48], batch=128,
                    weighted_loss=True),
    "big_odd": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[256, 252], critic_hidden=[252, 256], batch=531),
}

# Just outside the envelope: each must take the per-layer fp32 plan (and still match the oracle there).
OUTSIDE = {
    "width260": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[64, 48], critic_hidden=[260, 40], batch=64),
    # (a batch that is not a multiple of 4: head_bwd4_kernel's scratch follows the batch's head gradients in shared memory)
    "width260_b67": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[64, 48], critic_hidden=[260, 40], batch=67),
    "width254": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[254, 40], critic_hidden=[64, 48], batch=64),
    "input253": dict(state_dim=245, num_tasks=4, act_dim=4, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=48),
}

# per-row outputs of the step: debug name of the CUDA buffer == key of the port's intermediates
ROW_OUTPUTS = ("q1", "q2", "y", "a_next", "logp_next", "a_cur", "logp_cur", "qmin", "d_action", "d_head")
LAUNCHES = ("chain_fwd", "chain2", "chain_bwd")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_sac_b200 import _lib
    _lib.load()
    return torch.device("cuda", 0)


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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _params(spec, seed):
    """Xavier weights, small random biases (targets distinct from the locals), and a different temperature per task, so
    that a wrong task's alpha or a wrong network's bias changes the result."""
    p = sp.init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in p:
        if k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


def _eps(spec, gen):
    return torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen)


def check_rows(core, spec, o, replica=0, what=""):
    """Every per-row output of the step, element by element: |got - ref| <= 1e-4 (|ref| + mean |ref|).  Returns the
    largest observed |got - ref| / (|ref| + mean |ref|)."""
    worst = 0.0
    for k in ROW_OUTPUTS:
        ref = o[k].detach().double().reshape(spec.batch, -1)
        got = core.debug(k, replica).double().reshape(ref.shape)
        scale = ref.abs() + ref.abs().mean()
        dev = (got - ref).abs()
        bad = (dev > REL * scale) | ~torch.isfinite(got)
        if bad.any():
            rows = sorted({int(i) for i in bad.nonzero()[:, 0]})
            r, j = (int(x) for x in bad.nonzero()[0])
            raise AssertionError(f"{what}{k}: {int(bad.sum())} elements beyond {REL} (|ref| + mean|ref|), rows {rows[:12]}"
                                 f"{'...' if len(rows) > 12 else ''}; first [{r}][{j}] got {float(got[r, j]):.7g} "
                                 f"ref {float(ref[r, j]):.7g}")
        worst = max(worst, float((dev / scale.clamp_min(1e-30)).max()))
    return worst


def check_losses(core, o, replica=0, what=""):
    L = core.read_losses(1)[0, replica]
    assert torch.isfinite(L).all(), f"{what}losses {L.tolist()}"
    for i, k in ((0, "critic_loss"), (1, "actor_loss"), (3, "entropy")):
        assert rel_scalar(float(L[i]), o[k]) <= REL, f"{what}{k}: {float(L[i])} vs oracle {o[k]}"


def check_active(core, spec, replica=0, what=""):
    """Every hidden layer of every network (actor on s' and s, Q1/Q2 on (s, a) and (s, a~)) has between 5 % and 95 %
    active units in the CUDA step's own masks: a sweep over dead or saturated layers would prove little."""
    for tag, m in cuda_relu_masks(core, spec, replica).items():
        if tag.startswith(("tanh:", "route:")):
            continue
        frac = float(m.float().mean())
        assert 0.05 <= frac <= 0.95, f"{what}hidden layer {tag}: {100 * frac:.1f}% active"


def run_checked(core, spec, port, n_steps, seed, what):
    """n_steps checked steps of `core` against `port`; returns (mask bits flipped at kinks, worst per-row deviation)."""
    gen = torch.Generator().manual_seed(seed)
    flips, worst = 0, 0.0
    for i in range(n_steps):
        b = sp.synthetic_batch(spec, seed=seed + 100 + i)
        e1, e2 = _eps(spec, gen)
        o, f = kink_checked_step(core, port, spec, b, e1, e2, want_intermediates=True)
        flips += sum(f.values())
        tag = f"{what} step {i}: "
        check_active(core, spec, what=tag)
        check_losses(core, o, what=tag)
        check_port_state(core, port)               # after step 0, m = (1 - beta1) g: every gradient tensor as well
        worst = max(worst, check_rows(core, spec, o, what=tag))
    return flips, worst


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2: the oracle sweep, with the guards that it ran the chained plan on non-degenerate networks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_chained_step_matches_oracle(cuda, chained_launches, name):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(**CASES[name])
    p = _params(spec, seed=7)
    port = sp.PortLearner(spec, p)
    core = SacCore(core_config(spec, precision=0), 0, seed=0)
    assert core.launches_per_step == chained_launches, (name, core.launches_per_step, chained_launches)
    assert _launches(spec, unfused=True) != chained_launches, name
    # (data seed: with 11, wide_in's third step leaves Q2's head-bias Adam moment at 1.5e-5 out of 0.9 m + 0.1 g with both
    # terms near 0.07 -- a one-element cancellation that no fp32 evaluation order meets at 1e-4)
    flips, worst = run_checked(core, spec, port, 3, seed=13, what=name)
    got = core.get_named(_lib.PARAMS)
    for k in sp.param_names(spec, sp.TRAINABLE_NETS):
        assert torch.isfinite(got[k]).all(), (name, k)
        assert not torch.equal(got[k], p[k]), f"{name}: {k} did not change in three steps"
    core.close()
    print(f"[kinks] {name}: {flips} mask bits differed, all at numerically-zero pre-activations")
    print(f"[rows] {name}: largest per-row |got - ref| / (|ref| + mean|ref|) = {worst:.2e}  (rows per CTA {plan_rows(spec.batch, 1, _sms())})")


# ---------------------------------------------------------------------------------------------------------------------
# 3: the sweep puts a partial CTA into every chain launch at every rows-per-CTA value
# ---------------------------------------------------------------------------------------------------------------------
def test_sweep_covers_a_tail_cta_at_every_rows_per_cta(cuda):
    sms = _sms()
    have = set()
    for c in CASES.values():
        for launch, rows in plan_rows(c["batch"], 1, sms).items():
            if c["batch"] % rows:
                have.add((launch, rows))
    missing = sorted({(launch, rows) for launch in LAUNCHES for rows in (2, 4, 8)} - have)
    assert not missing, f"on {sms} SMs no case gives these (launch, rows per CTA) pairs a partial CTA: {missing}; add a batch"


# ---------------------------------------------------------------------------------------------------------------------
# 4: co-scheduled replicas with parameters and minibatches of their own
# ---------------------------------------------------------------------------------------------------------------------
def test_replicas_with_different_parameters_match_their_oracles(cuda, chained_launches):
    """Three replicas, each its own parameter draw and minibatch: every replica follows its own oracle, and equals bit for
    bit an R = 1 handle given the same state and inputs -- whose launches use other rows per CTA (each row's sums have
    a fixed order that does not depend on them)."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    # (batch 105, a multiple of the 5 tasks: each replica's minibatch has task ids of its own; 105 rows leave a partial CTA
    # at every rows-per-CTA value either handle uses)
    spec = sp.SacSpec(state_dim=9, num_tasks=5, act_dim=3, actor_hidden=[64, 48], critic_hidden=[56, 72], batch=105)
    R, sms = 3, _sms()
    rows3, rows1 = plan_rows(spec.batch, R, sms), plan_rows(spec.batch, 1, sms)
    print(f"[rows] R = 3: {rows3}, R = 1: {rows1} ({sms} SMs)")
    if sms == 132:
        assert list(rows3.values()) == [8, 8, 4] and list(rows1.values()) == [4, 2, 2]
    assert rows3 != rows1
    params = [_params(spec, seed=30 + r) for r in range(R)]
    ports = [sp.PortLearner(spec, p) for p in params]
    batches = [sp.synthetic_batch(spec, seed=300 + r) for r in range(R)]
    gen = torch.Generator().manual_seed(3)
    eps = [_eps(spec, gen) for _ in range(R)]

    core = SacCore(core_config(spec, replicas=R, precision=0), 0, seed=0)
    assert core.launches_per_step == chained_launches
    for r in range(R):
        sync_core_to_port(core, ports[r], r)
    core.step(*[torch.stack([b[j] for b in batches]) for j in range(5)],
              torch.stack([e[0] for e in eps]), torch.stack([e[1] for e in eps]))
    for r in range(R):
        forced = cuda_relu_masks(core, spec, r)
        with sp.ReluTape(forced) as tape:
            o = ports[r].update_SAC(*batches[r], *eps[r], want_intermediates=True)
        check_forced(tape, forced, f"replica {r}: ")
        check_active(core, spec, r, f"replica {r}: ")
        check_losses(core, o, r, f"replica {r}: ")
        check_port_state(core, ports[r], replica=r)
        check_rows(core, spec, o, r, f"replica {r}: ")
    L3 = core.read_losses(1)[0]
    assert not torch.equal(L3[0], L3[1]) and not torch.equal(L3[1], L3[2])

    single = SacCore(core_config(spec, precision=0), 0, seed=0)
    for r in range(R):
        sync_core_to_port(single, sp.PortLearner(spec, params[r]))
        single.step(*batches[r], *eps[r])
        diff = [f"{which}:{k}" for which, arena in (("params", _lib.PARAMS), ("grads", _lib.GRADS), ("adam_m", _lib.ADAM_M),
                                                     ("adam_v", _lib.ADAM_V))
                for a, b in [(core.get_named(arena, r), single.get_named(arena))] for k in a if not torch.equal(a[k], b[k])]
        assert not diff, f"replica {r} of the R = 3 handle differs from the R = 1 handle in {diff[:8]}"
        assert torch.equal(L3[r], single.read_losses(1)[0, 0]), (r, L3[r].tolist(), single.read_losses(1)[0, 0].tolist())
    single.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: just outside the envelope -- the per-layer fp32 plan, still matching the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(OUTSIDE))
def test_outside_the_envelope_takes_the_per_layer_plan(cuda, chained_launches, name):
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(**OUTSIDE[name])
    port = sp.PortLearner(spec, _params(spec, seed=5))
    core = SacCore(core_config(spec, precision=0), 0, seed=0)
    assert core.launches_per_step != chained_launches, name
    assert core.launches_per_step == _launches(spec, unfused=True), name
    flips, worst = run_checked(core, spec, port, 1, seed=21, what=name)
    core.close()
    print(f"[kinks] {name}: {flips} mask bits differed, all at numerically-zero pre-activations")
    print(f"[rows] {name}: largest per-row |got - ref| / (|ref| + mean|ref|) = {worst:.2e}")
