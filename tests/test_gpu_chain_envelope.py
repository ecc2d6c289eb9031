"""GPU: the layer-chained step (chain.cuh, chain2.cuh; build_plan_fused in b200sac.cu) over its whole eligibility envelope
against the autograd oracle.

The chained plan takes every exact-fp32, non-CARE learner whose hidden widths are multiples of 4 and at most 256, with at
most 8 hidden layers per network and state + tasks + act <= 252.  The cases (_harness.CHAIN_CASES) walk the edges of that space, where the
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
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, sync_core_to_port
from _harness import (CHAIN_CASES, _eps, _launches, _params, _sms, chained_launches, check_active, check_losses, check_rows,
                      cuda, plan_rows, run_checked)

pytestmark = pytest.mark.gpu

# Just outside the envelope: each must take the per-layer fp32 plan (and still match the oracle there).
OUTSIDE = {
    "width260": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[64, 48], critic_hidden=[260, 40], batch=64),
    # (a batch that is not a multiple of 4: head_bwd4_kernel's scratch follows the batch's head gradients in shared memory)
    "width260_b67": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[64, 48], critic_hidden=[260, 40], batch=67),
    "width254": dict(state_dim=8, num_tasks=0, act_dim=2, actor_hidden=[254, 40], critic_hidden=[64, 48], batch=64),
    "input253": dict(state_dim=245, num_tasks=4, act_dim=4, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=48),
}

LAUNCHES = ("chain_fwd", "chain2", "chain_bwd")


# ---------------------------------------------------------------------------------------------------------------------
# 1 + 2: the oracle sweep, with the guards that it ran the chained plan on non-degenerate networks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CHAIN_CASES))
def test_chained_step_matches_oracle(cuda, chained_launches, name):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec = sp.SacSpec(**CHAIN_CASES[name])
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
    for c in CHAIN_CASES.values():
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
