"""GPU: gradient surgery (PCGrad, CAGrad) on the CARE learners, CARE(M) and CARE(O).  The task slices of the critic range
(q1, q2 and every cse.mix / trunk / ctx tensor), of the actor and of the CARE(O) context encoder against the autograd
oracle's per-task gradients (the step's masks forced into it), the Gram matrix against fp64 from the exported slices, the
weights against the host solve, Adam of all three optimizers and the Polyak targets bit for bit, whole steps against the
surgery oracle (a constructed conflict, the full-size C10 shape, plain / PCGrad / CAGrad replicas side by side), settings
changed between prepared graphs, critic-only steps, the sampled rings, rows out of task order, the refusals, the plan's
launches and the learners."""
import dataclasses
import json
import math
import re

import numpy as np
import pytest
import torch

import cagrad_ref as cr
import care_port as cp
import care_surgery_ref as cs
import pcgrad_ref as pr
import redis_stub
import sac_port as sp
from _golden import care_core_config, check_forced, check_port_state, cuda_relu_masks, sync_core_to_port
from _harness import ADAM_M, ADAM_V, GRADS, PARAMS, _params, adam_expect, cuda, plan_labels  # noqa: F401

pytestmark = pytest.mark.gpu

VARIANTS = pytest.mark.parametrize("modified", [True, False], ids=["CARE(M)", "CARE(O)"])
C_DEF = 0.5


def _spec(T, modified, B=None):
    """Small CARE shapes: three mixture layers of K = 3 encoders, a two-layer trunk and context net."""
    B = B or {2: 96, 3: 96, 10: 320}[T]
    return cp.CareSpec(state_dim=6, act_dim=2, num_tasks=T, actor_hidden=[64, 48], critic_hidden=[48, 64], batch=B,
                       num_encoders=3, mix_hidden=[16, 12], mix_out=10, ctx_in=20, ctx_hidden=[12], ctx_out=10, emb_dim=10,
                       modified=modified, weighted_loss=modified)


def _core(spec, precision=0, R=1, seed=0, **kw):
    from distributed_sac_b200.core import SacCore
    return SacCore(dataclasses.replace(care_core_config(spec, replicas=R, precision=precision), pcgrad=True, **kw), 0,
                   seed=seed)


def _block_batch(spec, seed):
    s, a, r, s2, d = cp.synthetic_batch(spec, seed=seed)
    order = torch.argsort(torch.argmax(s[:, -spec.num_tasks:], 1), stable=True)
    return s[order], a[order], r[order], s2[order], d[order]


def _data(spec, R, step=0, seed=0):
    bs = [_block_batch(spec, 500 + 37 * r + 1000 * step + seed) for r in range(R)]
    b = [torch.stack([x[j] for x in bs]) for j in range(5)]
    g = torch.Generator().manual_seed(77 + step + seed)
    e1, e2 = (torch.randn(R, spec.batch, spec.act_dim, generator=g) for _ in range(2))
    return b, e1, e2


def _opt_range(core, which):
    """(begin, end) of layout-table optimizer `which`'s slice of the trainable arena (0 critic, 1 actor, 3 context
    encoder)."""
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


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _state(core, r):
    return {k: core.export_arena(k, r).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)}


def _slices(core, T, r):
    return np.stack([core.export_task_grad(t, r).numpy() for t in range(T)])


def _check_adam(core, spec, r, before, after, slices, w, what, actor=True):
    """p, m and v of the critic and actor after the step == adam_expect on sum_t fp32(w_t g_t), and of the CARE(O)
    context encoder on the plain slice sum, bit for bit."""
    k = core.get_steps(r)
    T = spec.num_tasks
    opts = [(0, w[0], spec.lr_critic, k[0])] + ([(1, w[1], spec.lr_actor, k[1])] if actor else [])
    if not spec.modified:
        opts.append((3, np.ones(T, np.float32), spec.lr_ctx, k[3]))
    for which, ww, lr, n in opts:
        lo, hi = _opt_range(core, which)
        ghat = pr.combine_fp32(slices[:, lo:hi], ww)
        pe, me, ve = adam_expect(before[PARAMS][lo:hi], before[ADAM_M][lo:hi], before[ADAM_V][lo:hi], ghat, lr,
                                 spec.beta1 ** n, spec.beta2 ** n)
        for arena, exp in ((PARAMS, pe), (ADAM_M, me), (ADAM_V, ve)):
            assert np.array_equal(after[arena][lo:hi].view(np.uint32), exp.view(np.uint32)), (what, which, arena)


def _check_targets(core, spec, p0, p1, what):
    """q targets with tau and the target state encoder with tau_se, fp32 per operation, bit for bit."""
    for n in core.table:
        if n.startswith(("q1_target.", "q2_target.")):
            rate, ln = spec.tau, n.replace("_target.", ".", 1)
        elif n.startswith("tse."):
            rate, ln = spec.tau_se, "cse." + n[4:]
        else:
            continue
        exp = np.float32(rate) * p1[ln].numpy() + np.float32(1.0 - rate) * p0[n].numpy()
        assert np.array_equal(p1[n].numpy().view(np.uint32), exp.astype(np.float32).view(np.uint32)), (what, n)


def _check_step(core, spec, r, before, b, e1, e2, mode, what):
    """One step of replica r against the oracle and the kernels' exact arithmetic.  mode: "pcgrad", "cagrad" (c = C_DEF)
    or "plain" (switches off, c = 0)."""
    T = spec.num_tasks
    rec = core.read_pcgrad(r)
    slices = _slices(core, T, r)
    after = _state(core, r)
    assert rec["task_mismatch"] == 0, what
    batch = [x[r] for x in b]
    p0 = _unflat(core, before[PARAMS], list(core.table))
    p1 = _unflat(core, after[PARAMS], list(core.table))
    port = cp.CarePortLearner(spec, p0)
    forced = cuda_relu_masks(core, spec, r, care=True)
    with sp.ReluTape(forced) as tape:
        ref0 = cs.task_grads(port, batch, e1[r], e2[r], 0)
        with torch.no_grad():             # the actor's gradient goes through the critics the step's critic update left
            for n in port.critic_names:
                port.p[n].copy_(p1[n])
        ref1 = cs.task_grads(port, batch, e1[r], e2[r], 1)
    check_forced(tape, {k: v for k, v in forced.items() if k in tape.z}, what)
    for which, ref_t in ((0, ref0), (1, ref1)):
        lo, hi = _opt_range(core, which)
        sl = slices[:, lo:hi].astype(np.float64)
        G = rec["gram"][which]
        gref = sl @ sl.T
        assert np.allclose(G, gref, rtol=1e-12, atol=1e-12 * np.abs(gref).max()), (what, which)
        if mode == "cagrad":
            host = cr.solve(G, C_DEF)
            cg = core.read_cagrad(r)
            assert cg["ibest"][which] == host["ibest"], (what, which)
            assert np.max(np.abs(cg["p"][which] - host["p"])) <= 1e-12, (what, which)
            assert _ulps(rec["w"][which], host["w32"]).max() <= 1, (what, which)
            assert not rec["projected"].any(), what
        else:
            _, w, taken = pr.gram_solve(G, rec["perm"][which], mode == "pcgrad")
            assert np.array_equal(rec["projected"][which], taken), (what, which)
            assert np.array_equal(rec["w"][which], w.astype(np.float32)), (what, which, rec["w"][which], w)
        names = cs.loss_names(port, which)
        for t in range(T):
            got = _unflat(core, slices[t], names)
            for n in names:
                assert _rel(got[n].numpy(), ref_t[t][n].numpy()) < 1e-4, (what, which, t, n)
    _check_adam(core, spec, r, before, after, slices, rec["w"], what)
    _check_targets(core, spec, p0, p1, what)
    return rec


def _set_mode(core, r, mode):
    core.set_pcgrad(critic=mode == "pcgrad", actor=mode == "pcgrad", replica=r)
    core.set_cagrad(critic=C_DEF if mode == "cagrad" else 0.0, actor=C_DEF if mode == "cagrad" else 0.0, replica=r)


@VARIANTS
@pytest.mark.parametrize("mode", ["pcgrad", "cagrad"])
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("T", [2, 3, 10])
@pytest.mark.parametrize("R", [1, 3])
def test_care_surgery_step(cuda, modified, mode, precision, T, R):
    spec = _spec(T, modified)
    core = _core(spec, precision, R)
    for r in range(R):
        core.set_named(_params(spec, 11 + 7 * r, care=True, move_targets=True), PARAMS, r)
        _set_mode(core, r, mode)
    before = [_state(core, r) for r in range(R)]
    b, e1, e2 = _data(spec, R)
    core.step(*b, e1, e2)
    torch.cuda.synchronize()
    for r in range(R):
        _check_step(core, spec, r, before[r], b, e1, e2, mode, f"{mode} p{precision} T{T} R{R} r{r}")
    # GRADS stays the unprojected gradient: the slices summed in index order
    sl = _slices(core, T, 0)
    assert np.array_equal(core.export_arena(GRADS, 0).numpy().view(np.uint32), pr.combine_fp32(sl, np.ones(T)).view(np.uint32))
    core.close()


def test_replicas_plain_pcgrad_cagrad_side_by_side(cuda):
    """One R = 3 CARE(O) handle: replica 0 the plain sum, 1 PCGrad, 2 CAGrad, each against its own expectation."""
    spec = _spec(3, False)
    core = _core(spec, 1, 3)
    modes = ["plain", "pcgrad", "cagrad"]
    for r, m in enumerate(modes):
        core.set_named(_params(spec, 31 + r, care=True, move_targets=True), PARAMS, r)
        _set_mode(core, r, m)
    before = [_state(core, r) for r in range(3)]
    b, e1, e2 = _data(spec, 3, seed=4)
    core.step(*b, e1, e2)
    recs = [_check_step(core, spec, r, before[r], b, e1, e2, m, f"side by side {m}") for r, m in enumerate(modes)]
    assert np.array_equal(recs[0]["w"], np.ones((2, 3), np.float32))
    assert (core.read_cagrad(2)["ibest"] >= 0).all() and (core.read_cagrad(0)["ibest"] == -1).all()
    core.close()


def _conflict_batch(spec, step):
    """Two tasks with the same states, actions and next states, and rewards of opposite sign."""
    b, e1, e2 = _data(spec, 1, step=step)
    P = spec.batch // 2
    for j in (0, 1, 3):
        b[j][0, P:] = b[j][0, :P]
    for j in (0, 3):                          # the one-hot stays the row's own task
        b[j][0, P:, spec.state_dim:] = b[j][0, :P, spec.state_dim:].flip(-1)
    b[2][0, :P] = 20.0 + b[2][0, :P].abs()
    b[2][0, P:] = -b[2][0, :P]
    return b, e1, e2


def _oracle_steps(core, spec, batches, what, c=None):
    """Each (b, e1, e2) stepped on the device and on the surgery oracle (PCGrad on the device's permutations, or CAGrad
    with c), the step's masks forced; after every step the whole state agrees to 1e-4.  Returns the device records."""
    port = cp.CarePortLearner(spec, _unflat(core, core.export_arena(PARAMS, 0).numpy(), list(core.table)))
    sync_core_to_port(core, port, 0)
    recs = []
    for i, (b, e1, e2) in enumerate(batches):
        core.step(*b, e1, e2)
        rec = core.read_pcgrad(0)
        forced = cuda_relu_masks(core, spec, 0, care=True)
        with sp.ReluTape(forced) as tape:
            ref = cs.surgery_update(port, *[x[0] for x in b], e1[0], e2[0], rec["perm"], c=c)
        check_forced(tape, forced, f"{what} step {i}")
        for which in (0, 1):
            G, w32, taken = ref[which]
            if c is None:
                assert np.array_equal(rec["projected"][which], taken), (what, i, which)
            assert np.allclose(rec["w"][which], w32, rtol=1e-4, atol=1e-4), (what, i, which, rec["w"][which], w32)
            assert np.allclose(rec["gram"][which], G, rtol=2e-4, atol=1e-4 * np.abs(G).max()), (what, i, which)
        check_port_state(core, port, 0)
        recs.append(rec)
    return recs


@VARIANTS
def test_conflict_follows_oracle(cuda, modified):
    """Four steps on conflicting tasks: the critic projects, and the whole state follows the PCGrad oracle."""
    spec = _spec(2, modified)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 3, care=True, move_targets=True), PARAMS, 0)
    recs = _oracle_steps(core, spec, [_conflict_batch(spec, k) for k in range(4)], "conflict")
    assert any(rec["projected"][0].any() for rec in recs)
    core.close()


@VARIANTS
@pytest.mark.parametrize("mode", ["pcgrad", "cagrad"])
def test_full_size_c10(cuda, modified, mode):
    """BASELINE config 5's shape (39 + 10 inputs, K = 6 encoders, 768-d context, 400^3 MLPs, batch 1280, T 10) at
    precision 1: two steps against the surgery oracle."""
    spec = cp.CareSpec(modified=modified, weighted_loss=modified)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 4, care=True, move_targets=True), PARAMS, 0)
    if mode == "cagrad":
        _set_mode(core, 0, "cagrad")
    batches = []
    for k in range(2):
        b = _block_batch(spec, 60 + k)
        g = torch.Generator().manual_seed(90 + k)
        batches.append(([x[None] for x in b], torch.randn(1, spec.batch, spec.act_dim, generator=g),
                        torch.randn(1, spec.batch, spec.act_dim, generator=g)))
    _oracle_steps(core, spec, batches, f"C10 {mode}", c=C_DEF if mode == "cagrad" else None)
    core.close()


def _ring(core, spec, n=3000, seed=4, **kw):
    from distributed_sac_b200.core import Replay
    rb = Replay(core, 4096, kw.pop("where", "device"), seed=seed, **kw)
    s, a, r, s2, d = cp.synthetic_batch(spec, seed=seed, batch=n)
    r = torch.where(s[:, spec.state_dim:spec.state_dim + 1] > 0, 5.0 + r.abs(), -5.0 - r.abs())
    return rb, (s, a, r, s2, d)


@VARIANTS
def test_settings_between_prepared_graphs(cuda, modified):
    """Switches and c set between launches of prepared graphs apply to the next step and to no earlier one."""
    spec = _spec(2, modified)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 3, care=True, move_targets=True), PARAMS, 0)
    rb, (s, a, r, s2, d) = _ring(core, spec)
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    ones = np.ones((2, 2), np.float32)
    try:
        core.prepare(rb)
        core.step_sampled(rb, 1)
        rec = core.read_pcgrad(0)
        for which in (0, 1):
            assert np.array_equal(rec["w"][which], pr.gram_solve(rec["gram"][which], rec["perm"][which])[1].astype(np.float32))
        core.set_pcgrad(critic=False, actor=False)
        core.step_sampled(rb, 1)
        rec = core.read_pcgrad(0)
        assert np.array_equal(rec["w"], ones) and not rec["projected"].any()
        assert (core.read_cagrad(0)["ibest"] == -1).all()
        core.set_cagrad(critic=C_DEF, actor=C_DEF)
        core.step_sampled(rb, 1)
        rec, cg = core.read_pcgrad(0), core.read_cagrad(0)
        assert (cg["ibest"] >= 0).all() and not rec["projected"].any()
        for which in (0, 1):
            assert _ulps(rec["w"][which], cr.solve(rec["gram"][which], C_DEF)["w32"]).max() <= 1
        core.set_cagrad(critic=0.0, actor=0.0)
        core.step_sampled(rb, 1)
        assert np.array_equal(core.read_pcgrad(0)["w"], ones) and (core.read_cagrad(0)["ibest"] == -1).all()
    finally:
        rb.close()
        core.close()


@VARIANTS
def test_critic_only_step(cuda, modified):
    """On a critic-only step the actor is untouched and its record NaN; the CARE(O) context encoder's Adam still runs on
    the plain slice sum."""
    spec = _spec(3, modified)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 8, care=True, move_targets=True), PARAMS, 0)
    core.set_update_intervals(actor_every=2)
    lo, hi = _opt_range(core, 1)
    before = _state(core, 0)
    b, e1, e2 = _data(spec, 1)
    core.step(*b, e1, e2)
    rec = core.read_pcgrad(0)
    after = _state(core, 0)
    assert np.isnan(rec["w"][1]).all() and np.isfinite(rec["w"][0]).all()
    assert np.array_equal(after[PARAMS][lo:hi].view(np.uint32), before[PARAMS][lo:hi].view(np.uint32))
    _check_adam(core, spec, 0, before, after, _slices(core, 3, 0), rec["w"], "critic-only", actor=False)
    if not modified:
        clo, chi = _opt_range(core, 3)
        assert not np.array_equal(after[PARAMS][clo:chi], before[PARAMS][clo:chi])
    core.close()


@VARIANTS
@pytest.mark.parametrize("ring", ["uniform", "prioritized", "linked", "host"])
def test_sampled_rings(cuda, modified, ring):
    """Sampled steps from the device ring (uniform, prioritized, linked n-step) and the pinned-host ring: rows in task
    blocks, and every step's Adam bit for bit on the weighted slices."""
    spec = _spec(3, modified)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 6, care=True, move_targets=True), PARAMS, 0)
    kw = dict(where="host") if ring == "host" else dict(prioritized=dict(alpha=0.6, beta=0.4, eps=1e-3)) \
        if ring == "prioritized" else dict(trajectories=True) if ring == "linked" else {}
    rb, (s, a, r, s2, d) = _ring(core, spec, seed=8, **kw)
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
            _check_adam(core, spec, 0, before, _state(core, 0), _slices(core, 3, 0), rec["w"], f"{ring} step {k}")
    finally:
        rb.close()
        core.close()


@VARIANTS
def test_out_of_order_rows(cuda, modified):
    """b200sac_step with shuffled rows counts them, and GRADS (the slice sum) is still the oracle's total gradient."""
    spec = _spec(3, modified)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 9, care=True, move_targets=True), PARAMS, 0)
    p0 = _unflat(core, core.export_arena(PARAMS, 0).numpy(), list(core.table))
    b, e1, e2 = _data(spec, 1)
    perm = torch.randperm(spec.batch, generator=torch.Generator().manual_seed(1))
    sh = [x[:, perm] for x in b]
    wrong = int((sh[0][0, :, -spec.num_tasks:].argmax(1) != torch.arange(spec.batch) // (spec.batch // 3)).sum())
    assert wrong > 0
    core.step(*sh, e1, e2)
    assert core.read_pcgrad(0)["task_mismatch"] == wrong
    p1 = _unflat(core, core.export_arena(PARAMS, 0).numpy(), list(core.table))
    grads = core.export_arena(GRADS, 0).numpy()
    port = cp.CarePortLearner(spec, p0)
    batch = [x[0] for x in sh]
    forced = cuda_relu_masks(core, spec, 0, care=True)
    with sp.ReluTape(forced) as tape:
        ref0 = cs.task_grads(port, batch, e1[0], e2[0], 0)
        with torch.no_grad():
            for n in port.critic_names:
                port.p[n].copy_(p1[n])
        ref1 = cs.task_grads(port, batch, e1[0], e2[0], 1)
    check_forced(tape, {k: v for k, v in forced.items() if k in tape.z}, "shuffled")
    for which, ref_t in ((0, ref0), (1, ref1)):
        names = cs.loss_names(port, which)
        got = _unflat(core, grads, names)
        for n in names:
            tot = sum(t[n] for t in ref_t)
            assert _rel(got[n].numpy(), tot.numpy()) < 1e-4, (which, n)
    core.close()


def _norm(label):
    """A launch label without what the task slicing changes: the K split, head_bwd's row slices and the wgmma tile."""
    label = re.sub(r", split \d+", "", label)
    label = re.sub(r"row slices \d+", "row slices", label)
    return re.sub(r"wgmma 128x\d+( paired)?", "wgmma", label)


@VARIANTS
@pytest.mark.parametrize("precision", [0, 1])
def test_refusals_and_plan_shape(cuda, modified, precision):
    """CARE with T = 1 or grad_clip is still refused.  The plan is the default CARE plan plus pcgrad{critic} before
    adam_critic+polyak, pcgrad{actor} before adam_actor+alpha and the gemm launches the group limit adds."""
    from distributed_sac_b200.core import SacCore
    spec = _spec(10, modified)
    for bad in (dict(num_tasks=1, batch=96), dict(grad_clip=True)):
        with pytest.raises(RuntimeError):
            SacCore(dataclasses.replace(care_core_config(spec, precision=precision), pcgrad=True, **bad), 0)
    plain = SacCore(care_core_config(spec, precision=precision), 0)
    surg = _core(spec, precision)
    L0, L1 = plan_labels(plain), plan_labels(surg)
    for opt, nxt in (("critic", "adam_critic+polyak"), ("actor", "adam_actor+alpha")):
        i = L1.index(f"pcgrad{{{opt}}}")
        assert L1[i + 1] == nxt, (opt, L1[i + 1])
    rest = [_norm(x) for x in L1 if not x.startswith("pcgrad{")]
    want = [_norm(x) for x in L0]
    extra, j = [], 0
    for x in rest:
        if j < len(want) and x == want[j]:
            j += 1
        else:
            extra.append(x)
    assert j == len(want), (want[j:], rest)
    assert all(x.startswith("gemm_") for x in extra), extra
    assert surg.launches_per_step == plain.launches_per_step + 2 + len(extra)
    plain.close()
    surg.close()


def _learner_cfg(tmp_path, modified, T=3):
    names_ = [f"task-{i}" for i in range(T)]
    rng = np.random.default_rng(0)
    (tmp_path / "emb.json").write_text(json.dumps({n: rng.standard_normal(64).round(4).tolist() for n in names_}))
    (tmp_path / "names.json").write_text(json.dumps(names_))
    cfg = {"use_modified_care": modified, "num_tasks": T, "device": "cuda", "buffer_size": 4096, "reward_scale": 1,
           "batch_size": 60, "log_alpha": 0, "tau": 0.005, "update_delay": 1, "start_memory_len": 1000,
           "print_period_learner": 10, "gamma": 0.99,
           "actor": {"state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "lr_actor": 3e-4, "actor_hidden_dim": [64, 64]},
           "critic": {"state_dim": 12, "action_dim": 3, "lr_critic": 3e-4, "critic_hidden_dim": [64, 64]},
           "encoder": {"state_dim": 12, "pretrained_embedding_json_path": str(tmp_path / "emb.json"),
                       "task_name_json_path": str(tmp_path / "names.json"), "hidden_dims_contextEnc": [20],
                       "embedding_dim_contextEnc": 16, "output_dim_contextEnc": 16, "RoBERTa_embedding_dim": 64,
                       "lr_contextEnc": 3e-4, "hidden_dims_mixtureEnc": [24], "output_dim_mixtureEnc": 16, "num_encoders": 3,
                       "num_tasks": T, "state_encoder_tau": 0.05}}
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(cfg))
    return str(p), names_


@VARIANTS
@pytest.mark.parametrize("mode", ["pcgrad", "cagrad"])
def test_care_learner_host_ring(cuda, tmp_path, monkeypatch, modified, mode):
    """CARELearner(pcgrad=True) / (cagrad=0.5).update() through the pinned-host ring: the record is finite and in task
    order, set_pcgrad / set_cagrad(0) give the plain sum on the next update, and the exported actor encoder is the
    critic's."""
    from distributed_sac_b200.learner import CARELearner
    monkeypatch.chdir(tmp_path)
    path, names_ = _learner_cfg(tmp_path, modified)
    kw = dict(pcgrad=True) if mode == "pcgrad" else dict(cagrad=C_DEF)
    lrn = CARELearner(None, names_, path, write_mode=False, replay_where="host",
                      server=redis_stub.StrictRedis(host=str(tmp_path) + mode), **kw)
    try:
        lrn.memory.ring.fill_synthetic(4096, seed=1)
        for _ in range(2):
            assert all(math.isfinite(x) for x in lrn.update())
            rec = lrn.core.read_pcgrad(0)
            assert rec["task_mismatch"] == 0 and np.isfinite(rec["gram"]).all() and np.isfinite(rec["w"]).all()
        if mode == "cagrad":
            assert (lrn.core.read_cagrad(0)["ibest"] >= 0).all()
            lrn.set_cagrad(0)
        else:
            lrn.set_pcgrad(critic=False, actor=False)
        lrn.update()
        assert np.array_equal(lrn.core.read_pcgrad(0)["w"], np.ones((2, 3), np.float32))
        sd = lrn._module_state_dict("actor")      # the actor's encoder is exported from the critic's
        crit = lrn.core.get_named()
        enc = {k: v for k, v in lrn._key_map("actor").items() if v.startswith("cse.")}
        assert enc and all(torch.equal(sd[k].reshape(-1), crit[v].reshape(-1)) for k, v in enc.items())
    finally:
        lrn.memory.stop()


def test_care_learner_refusals(cuda, tmp_path, monkeypatch):
    """The MT1 CARE learner (T = 1) still refuses surgery, and an 'encoder' block without the learner's keys raises an
    error that is both a KeyError and a ValueError, naming the keys."""
    from distributed_sac_b200.learner import CARELearner
    monkeypatch.chdir(tmp_path)
    path, names_ = _learner_cfg(tmp_path, True, T=1)
    for kw in (dict(pcgrad=True), dict(cagrad=C_DEF)):
        with pytest.raises(ValueError):
            CARELearner(None, names_, path, write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "t1"), **kw)
    cfg = json.loads(open(path).read())
    del cfg["encoder"]["lr_contextEnc"]
    (tmp_path / "bad.json").write_text(json.dumps(cfg))
    with pytest.raises(KeyError, match="lr_contextEnc") as e:
        CARELearner(None, names_, str(tmp_path / "bad.json"), write_mode=False,
                    server=redis_stub.StrictRedis(host=str(tmp_path) + "bad"))
    assert isinstance(e.value, ValueError)
