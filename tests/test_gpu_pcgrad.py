"""GPU: PCGrad gradient surgery (cfg.pcgrad) on the per-layer plan.  The task slices against the autograd oracle's per-task
gradients (the step's ReLU masks, saturated tanh and min routing forced into the oracle), the Gram matrix against fp64
from the exported slices and across handles and replica counts, the weights against the host Gram-form solve, Adam bit
for bit on the weighted slice sum, whole steps against the PCGrad oracle on the device's permutations (a constructed
conflict, the full-size MT10 shape), prioritized and linked n-step rings, the switches between prepared graphs,
critic-only steps, the task order checks, the learners and the plan's launch count."""
import dataclasses
import json

import numpy as np
import pytest
import torch

import pcgrad_ref as pr
import sac_port as sp
import redis_stub
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, sync_core_to_port
from _harness import ADAM_M, ADAM_V, GRADS, PARAMS, _params, adam_expect, cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def _spec(T, B=None):
    B = B or {2: 96, 3: 96, 10: 320}[T]
    return sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[64, 48], critic_hidden=[48, 64], batch=B, num_tasks=T,
                      weighted_loss=True)


def _core(spec, precision=0, R=1, seed=0, **kw):
    from distributed_sac_b200.core import SacCore
    return SacCore(dataclasses.replace(core_config(spec, replicas=R, precision=precision), pcgrad=True, **kw), 0, seed=seed)


def _data(spec, R, step=0, seed=0):
    bs = [pr.block_batch(spec, seed=500 + 37 * r + 1000 * step + seed) for r in range(R)]
    b = [torch.stack([x[j] for x in bs]) for j in range(5)]
    g = torch.Generator().manual_seed(77 + step + seed)
    e1, e2 = (torch.randn(R, spec.batch, spec.act_dim, generator=g) for _ in range(2))
    return b, e1, e2


def _opt_range(core, which):
    """(begin, end) of optimizer `which`'s slice of the trainable arena."""
    lo, hi = None, 0
    for name, (off, rows, _c, trainable, opt, pitch) in core.table.items():
        if trainable and opt == which:
            lo = off if lo is None else min(lo, off)
            hi = max(hi, off + rows * pitch)
    return lo, hi


def _unflat(core, flat, names):
    return {n: core._unpack(n, flat, core.table[n][0]) for n in names}


def _rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _check_adam(core, spec, r, before, after, slices, rec, what):
    """Both optimizers' p, m and v after the step == adam_expect on the weighted slice sum, bit for bit."""
    k = core.get_steps(r)
    for which in (0, 1):
        lo, hi = _opt_range(core, which)
        ghat = pr.combine_fp32(slices[:, lo:hi], rec["w"][which])
        lr = spec.lr_critic if which == 0 else spec.lr_actor
        n = k[which]
        pe, me, ve = adam_expect(before[PARAMS][lo:hi], before[ADAM_M][lo:hi], before[ADAM_V][lo:hi], ghat, lr,
                                 spec.beta1 ** n, spec.beta2 ** n)
        assert np.array_equal(after[PARAMS][lo:hi].view(np.uint32), pe.view(np.uint32)), (what, which)
        assert np.array_equal(after[ADAM_M][lo:hi].view(np.uint32), me.view(np.uint32)), (what, which)
        assert np.array_equal(after[ADAM_V][lo:hi].view(np.uint32), ve.view(np.uint32)), (what, which)


def _state(core, r):
    return {k: core.export_arena(k, r).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)}


def _check_step(core, spec, r, before, b, e1, e2, what):
    """One pcgrad step of replica r against the oracle and the kernel's exact arithmetic."""
    T = spec.num_tasks
    rec = core.read_pcgrad(r)
    slices = np.stack([core.export_task_grad(t, r).numpy() for t in range(T)])
    after = {k: core.export_arena(k, r).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)}
    assert rec["task_mismatch"] == 0, what
    batch = [x[r] for x in b]
    p0 = _unflat(core, before[PARAMS], list(core.table))
    p1 = _unflat(core, after[PARAMS], list(core.table))
    for which in (0, 1):
        lo, hi = _opt_range(core, which)
        sl = slices[:, lo:hi].astype(np.float64)
        # Gram matrix: fp64 from the slices the device wrote (pad entries are zero on both sides)
        G = rec["gram"][which]
        ref = sl @ sl.T
        assert np.allclose(G, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max()), (what, which)
        # weights: the host Gram-form solve from the device's G and permutations, every decision and weight identical
        c, w, taken = pr.gram_solve(G, rec["perm"][which])
        assert np.array_equal(rec["projected"][which], taken), (what, which)
        assert np.array_equal(rec["w"][which], w.astype(np.float32)), (what, which, rec["w"][which], w)
        # per-task slices against the oracle (the actor's through the critics the step's critic update left)
        src = dict(p0)
        if which == 1:
            for n in sp.param_names(spec, ("q1", "q2"), False):
                src[n] = p1[n]
        forced = cuda_relu_masks(core, spec, r)
        with sp.ReluTape(forced) as tape:
            ref_t = pr.task_grads(spec, src, batch, e1[r], e2[r], which)
        check_forced(tape, {k: v for k, v in forced.items() if k in tape.z}, what)     # the tags this pass evaluates
        for t in range(T):
            got = _unflat(core, slices[t], pr.opt_names(spec, which))
            for n in pr.opt_names(spec, which):
                assert _rel(got[n].numpy(), ref_t[t][n].numpy()) < 1e-4, (what, which, t, n)
    _check_adam(core, spec, r, before, after, slices, rec, what)
    # Polyak targets from the new critics, fp32 per operation
    tau, omt = np.float32(spec.tau), np.float32(1.0 - spec.tau)
    for n in sp.param_names(spec, ("q1", "q2"), False):
        tn = n.replace("q1.", "q1_target.").replace("q2.", "q2_target.")
        exp = tau * p1[n].numpy() + omt * p0[tn].numpy()
        assert np.array_equal(p1[tn].numpy().view(np.uint32), exp.astype(np.float32).view(np.uint32)), (what, tn)
    return rec


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("T", [2, 3, 10])
@pytest.mark.parametrize("R", [1, 3])
def test_pcgrad_step(cuda, precision, T, R):
    spec = _spec(T)
    core = _core(spec, precision, R)
    for r in range(R):
        core.set_named(_params(spec, 11 + 7 * r, move_targets=True), PARAMS, r)
    before = [{k: core.export_arena(k, r).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)} for r in range(R)]
    b, e1, e2 = _data(spec, R)
    core.step(*b, e1, e2)
    torch.cuda.synchronize()
    for r in range(R):
        _check_step(core, spec, r, before[r], b, e1, e2, f"p{precision} T{T} R{R} r{r}")
    # the unprojected gradient stays what GRADS exports: the slices summed in index order
    slices = [core.export_task_grad(t, 0).numpy() for t in range(T)]
    acc = slices[0].copy()
    for s_ in slices[1:]:
        acc = acc + s_
    assert np.array_equal(core.export_arena(GRADS, 0).numpy().view(np.uint32), acc.view(np.uint32))


def test_gram_reproducible_across_handles_and_replicas(cuda):
    spec = _spec(3)
    b, e1, e2 = _data(spec, 3, seed=9)
    grams = []
    for R in (3, 3):
        core = _core(spec, 1, R)
        for r in range(R):
            core.set_named(_params(spec, 5 + r, move_targets=True), PARAMS, r)
        core.step(*b, e1, e2)
        grams.append([core.read_pcgrad(r)["gram"] for r in range(R)])
    for r in range(3):
        one = _core(spec, 1, 1)
        one.set_named(_params(spec, 5 + r, move_targets=True), PARAMS, 0)
        one.step(*[x[r:r + 1] for x in b], e1[r:r + 1], e2[r:r + 1])
        g1 = one.read_pcgrad(0)["gram"]
        assert np.array_equal(grams[0][r].view(np.uint64), grams[1][r].view(np.uint64))
        assert np.array_equal(grams[0][r].view(np.uint64), g1.view(np.uint64))


def _conflict_batch(spec, step):
    """Two tasks with the same states, actions and next states, and rewards of opposite sign."""
    b, e1, e2 = _data(spec, 1, step=step)
    P = spec.batch // 2
    for j in (0, 1, 3):
        b[j][0, P:] = b[j][0, :P]
    for j in (0, 3):                          # the one-hot stays the row's own task
        b[j][0, P:, spec.state_dim:] = b[j][0, :P, spec.state_dim:].flip(-1)
    b[2][0, :P] = 5.0 + b[2][0, :P].abs()
    b[2][0, P:] = -b[2][0, :P]
    return b, e1, e2


def _oracle_steps(core, spec, batches, what):
    """Each (b, e1, e2) of `batches` stepped on the device and on the PCGrad oracle, the oracle run on the device's
    permutations with the step's ReLU masks, tanh values and min routing forced; after every step the whole state agrees
    to 1e-4 and the weights to 1e-4 relative.  Returns the device records."""
    port = sp.PortLearner(spec, sp.init_params(spec))
    sync_core_to_port(core, port, 0)
    recs = []
    for i, (b, e1, e2) in enumerate(batches):
        core.step(*b, e1, e2)
        rec = core.read_pcgrad(0)
        forced = cuda_relu_masks(core, spec, 0)
        with sp.ReluTape(forced) as tape:
            ref = pr.pcgrad_update(port, *[x[0] for x in b], e1[0], e2[0], rec["perm"])
        check_forced(tape, forced, f"{what} step {i}")
        for which in (0, 1):
            G, w32, taken = ref[which]
            assert np.array_equal(rec["projected"][which], taken), (what, i, which)
            assert np.allclose(rec["w"][which], w32, rtol=1e-4, atol=1e-4), (what, i, which)
            assert np.allclose(rec["gram"][which], G, rtol=2e-4, atol=1e-4 * np.abs(G).max()), (what, i, which)
        check_port_state(core, port, 0)
        recs.append(rec)
    return recs


def test_conflict_projects_and_matches_oracle(cuda):
    """Five steps on conflicting tasks: the critic projects on every step, and the whole state follows the oracle."""
    spec = _spec(2)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 3, move_targets=True), PARAMS, 0)
    before = _state(core, 0)
    b0 = _conflict_batch(spec, 0)
    recs = _oracle_steps(core, spec, [b0] + [_conflict_batch(spec, k) for k in range(1, 5)], "conflict")
    assert all(rec["projected"][0].any() for rec in recs)
    # the first step once more, bit for bit, on a fresh handle
    core2 = _core(spec, 0, 1)
    core2.set_named(_params(spec, 3, move_targets=True), PARAMS, 0)
    b, e1, e2 = b0
    core2.step(*b, e1, e2)
    _check_step(core2, spec, 0, before, b, e1, e2, "conflict step 0")


def test_full_size_ms_matches_oracle(cuda):
    """The MT10 MTSAC shape (39 + 10 inputs, 4 actions, 400^3, batch 1280, T 10) at precision 1: two steps."""
    spec = sp.ms_spec()
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 4, move_targets=True), PARAMS, 0)
    _oracle_steps(core, spec, [_data(spec, 1, step=k) for k in range(2)], "MS")


@pytest.mark.parametrize("ring", ["prioritized", "linked"])
def test_sampled_rings(cuda, ring):
    """Sampled steps on a prioritized ring and on a linked ring at n = 3: rows in task blocks, and every step's Adam bit
    for bit on the weighted slices."""
    from distributed_sac_b200.core import Replay
    spec = _spec(3)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 6, move_targets=True), PARAMS, 0)
    n = 3000
    rb = Replay(core, 4096, "device", seed=5, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-3) if ring == "prioritized" else None,
                trajectories=ring == "linked")
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=8, batch=n)
    if ring == "linked":
        rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy(), stream=s[:, spec.state_dim:].argmax(1).numpy())
        rb.set_nstep(3)
    else:
        rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    try:
        for k in range(3):
            before = _state(core, 0)
            core.step_sampled(rb, 1)
            rec = core.read_pcgrad(0)
            assert rec["task_mismatch"] == 0 and np.isfinite(rec["w"]).all(), (ring, k)
            slices = np.stack([core.export_task_grad(t, 0).numpy() for t in range(3)])
            _check_adam(core, spec, 0, before, _state(core, 0), slices, rec, f"{ring} step {k}")
    finally:
        rb.close()


def test_switch_off_and_stream_order(cuda):
    spec = _spec(3)
    core = _core(spec, 0, 2)
    for r in range(2):
        core.set_named(_params(spec, 21 + r, move_targets=True), PARAMS, r)
    assert core.get_pcgrad(1) == {"critic": True, "actor": True}
    core.set_pcgrad(critic=False, actor=False, replica=1)
    assert core.get_pcgrad(1) == {"critic": False, "actor": False} and core.get_pcgrad(0)["critic"]
    b, e1, e2 = _data(spec, 2, seed=3)
    before = {k: core.export_arena(k, 1).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)}
    core.step(*b, e1, e2)
    rec = core.read_pcgrad(1)
    assert np.array_equal(rec["w"], np.ones((2, 3), np.float32)) and not rec["projected"].any()
    assert np.isfinite(rec["gram"]).all()
    slices = np.stack([core.export_task_grad(t, 1).numpy() for t in range(3)])
    after = core.export_arena(PARAMS, 1).numpy()
    for which in (0, 1):
        lo, hi = _opt_range(core, which)
        g = slices[0, lo:hi] + slices[1, lo:hi] + slices[2, lo:hi]
        lr = spec.lr_critic if which == 0 else spec.lr_actor
        pe, _, _ = adam_expect(before[PARAMS][lo:hi], before[ADAM_M][lo:hi], before[ADAM_V][lo:hi], g, lr, spec.beta1, spec.beta2)
        assert np.array_equal(after[lo:hi].view(np.uint32), pe.view(np.uint32)), which


def test_switch_between_prepared_graphs(cuda):
    """Switches set between launches of prepared graphs apply to the next step and to no earlier one.  The ring holds
    rewards of opposite sign for the two tasks, so the critic's task gradients conflict."""
    from distributed_sac_b200.core import Replay
    spec = _spec(2)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 3, move_targets=True), PARAMS, 0)
    rb = Replay(core, 4096, "device", seed=3)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=4, batch=2000)
    r = torch.where(s[:, spec.state_dim:spec.state_dim + 1] > 0, 5.0 + r.abs(), -5.0 - r.abs())     # [n][1]
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    ones = np.ones((2, 2), np.float32)
    try:
        core.prepare(rb)
        core.step_sampled(rb, 1)
        assert core.read_pcgrad(0)["projected"][0].any()
        core.set_pcgrad(critic=False, actor=False)
        core.step_sampled(rb, 1)
        rec = core.read_pcgrad(0)
        assert np.array_equal(rec["w"], ones) and not rec["projected"].any()
        core.set_pcgrad(critic=True, actor=True)
        core.step_sampled(rb, 1)
        rec = core.read_pcgrad(0)
        assert rec["projected"][0].any() and not np.array_equal(rec["w"], ones)
    finally:
        rb.close()


def test_critic_only_step_leaves_actor(cuda):
    spec = _spec(2)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 8, move_targets=True), PARAMS, 0)
    core.set_update_intervals(actor_every=2)
    lo, hi = _opt_range(core, 1)
    p0 = core.export_arena(PARAMS, 0).numpy().copy()
    b, e1, e2 = _data(spec, 1)
    core.step(*b, e1, e2)
    rec = core.read_pcgrad(0)
    assert np.isnan(rec["w"][1]).all() and np.isfinite(rec["w"][0]).all()
    assert np.array_equal(core.export_arena(PARAMS, 0).numpy()[lo:hi].view(np.uint32), p0[lo:hi].view(np.uint32))


def test_task_order_checks(cuda):
    spec = _spec(3)
    core = _core(spec, 0, 1)
    b, e1, e2 = _data(spec, 1)
    perm = torch.randperm(spec.batch, generator=torch.Generator().manual_seed(1))
    shuffled = [x[:, perm] for x in b]
    wrong = int((shuffled[0][0, :, spec.state_dim:].argmax(1) != torch.arange(spec.batch) // (spec.batch // 3)).sum())
    assert wrong > 0
    with pytest.raises(RuntimeError):
        core.step_host(*shuffled, e1, e2)
    assert core.read_pcgrad(0)["task_mismatch"] == 0 and np.isnan(core.read_pcgrad(0)["gram"]).all()
    core.step(*shuffled, e1, e2)
    assert core.read_pcgrad(0)["task_mismatch"] == wrong
    core.step_host(*b, e1, e2)
    assert core.read_pcgrad(0)["task_mismatch"] == 0


def test_refusals_and_launch_count(cuda):
    from distributed_sac_b200.core import SacCore
    spec = _spec(2)
    for bad in (dict(num_tasks=1, batch=96), dict(grad_clip=True)):
        with pytest.raises(RuntimeError):
            SacCore(dataclasses.replace(core_config(spec, precision=1), pcgrad=True, **bad), 0)
    plain = SacCore(core_config(spec, precision=1), 0)
    with pytest.raises(RuntimeError):
        plain.set_pcgrad(critic=False)
    assert _core(spec, 1).launches_per_step == plain.launches_per_step + 2


MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


def test_mtsac_learner_host_ring(cuda, tmp_path):
    """MTSACLearner(pcgrad=True).update() through the pinned-host ring (the learner's default): the draw keeps the task
    blocks, the record is finite, and set_pcgrad turns the surgery off for the next update."""
    from distributed_sac_b200.learner import MTSACLearner
    p = tmp_path / "ms.json"
    p.write_text(json.dumps(MS_CFG))
    lrn = MTSACLearner(None, ["t0", "t1", "t2"], str(p), write_mode=False, replay_where="host", pcgrad=True,
                       server=redis_stub.StrictRedis(host=str(tmp_path) + "ms"))
    try:
        lrn.memory.ring.fill_synthetic(4096, seed=1)
        for _ in range(3):
            assert all(x == x for x in lrn.update())
            rec = lrn.core.read_pcgrad(0)
            assert rec["task_mismatch"] == 0 and np.isfinite(rec["gram"]).all() and np.isfinite(rec["w"]).all()
        lrn.set_pcgrad(critic=False, actor=False)
        lrn.update()
        assert np.array_equal(lrn.core.read_pcgrad(0)["w"], np.ones((2, 3), np.float32))
        s, *_ = lrn.memory.ring.sample()          # the ring's own draw is in task blocks too
        assert torch.equal(s[:, 12:].argmax(1), torch.arange(60) // 20)
    finally:
        lrn.memory.stop()


def test_learner_refusals(cuda, tmp_path):
    """The single-task learners and CARE cannot run PCGrad: ValueError before any handle is built."""
    from _harness import LEARNER_CFGS
    from distributed_sac_b200 import learner as L
    p = tmp_path / "LL.json"
    p.write_text(json.dumps(LEARNER_CFGS["LL"]))
    with pytest.raises(ValueError):
        L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "LL"), pcgrad=True)
    pc = tmp_path / "care.json"
    pc.write_text(json.dumps(dict(MS_CFG, encoder={}, use_modified_care=True)))
    with pytest.raises(ValueError):
        L.CARELearner(None, ["t0", "t1", "t2"], str(pc), write_mode=False, pcgrad=True,
                      server=redis_stub.StrictRedis(host=str(tmp_path) + "care"))
