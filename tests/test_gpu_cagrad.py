"""GPU: CAGrad (b200sac_set_cagrad) on pcgrad handles.  The one-warp solve against the host restatement on a set of Gram
matrices (degenerate ones included); whole steps with the record against the host solve of the device's own G, the task
slices against the autograd oracle, Adam and the Polyak targets bit for bit; several steps against the CAGrad oracle (a
constructed conflict and the full-size MT10 shape); plain, PCGrad and CAGrad replicas side by side in one handle; the
coefficient between prepared graphs; critic-only steps; prioritized and linked rings; refusals, the launch count and the
MTSAC learner."""
import ctypes as C
import dataclasses
import json
import math

import numpy as np
import pytest
import torch

import cagrad_ref as cr
import pcgrad_ref as pr
import sac_port as sp
import redis_stub
from _cagrad import gram_sets
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, sync_core_to_port
from _harness import ADAM_M, ADAM_V, GRADS, PARAMS, _params, adam_expect, cuda  # noqa: F401

pytestmark = pytest.mark.gpu

C_DEF = 0.5


def _spec(T, B=None):
    B = B or {2: 96, 3: 96, 10: 320}[T]
    return sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[64, 48], critic_hidden=[48, 64], batch=B, num_tasks=T,
                      weighted_loss=True)


def _core(spec, precision=0, R=1, seed=0, c=C_DEF):
    """A pcgrad handle with PCGrad off and CAGrad at c on both optimizers of every replica."""
    from distributed_sac_b200.core import SacCore
    core = SacCore(dataclasses.replace(core_config(spec, replicas=R, precision=precision), pcgrad=True), 0, seed=seed)
    core.set_pcgrad(critic=False, actor=False)
    core.set_cagrad(critic=c, actor=c)
    return core


def _data(spec, R, step=0, seed=0):
    bs = [pr.block_batch(spec, seed=500 + 37 * r + 1000 * step + seed) for r in range(R)]
    b = [torch.stack([x[j] for x in bs]) for j in range(5)]
    g = torch.Generator().manual_seed(77 + step + seed)
    e1, e2 = (torch.randn(R, spec.batch, spec.act_dim, generator=g) for _ in range(2))
    return b, e1, e2


def _opt_range(core, which):
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


def _state(core, r):
    return {k: core.export_arena(k, r).numpy().copy() for k in (PARAMS, ADAM_M, ADAM_V)}


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _check_record(rec, k, ref, what):
    """Device record entry k (0 critic, 1 actor) against a host solve record."""
    assert rec["ibest"][k] == ref["ibest"], (what, k, rec["ibest"][k], ref["ibest"])
    for name, key in (("lambda", "lam"), ("best", "best"), ("first", "first"), ("scale", "scale")):
        assert abs(rec[name][k] - ref[key]) <= 1e-12 * max(1.0, abs(ref[key])), (what, k, name, rec[name][k], ref[key])
    assert np.max(np.abs(rec["p"][k] - ref["p"])) <= 1e-12, (what, k)


def _check_adam(core, spec, r, before, after, slices, w, what):
    """Both optimizers' p, m and v after the step == adam_expect on sum_t fp32(w_t g_t), bit for bit."""
    k = core.get_steps(r)
    for which in (0, 1):
        lo, hi = _opt_range(core, which)
        ghat = pr.combine_fp32(slices[:, lo:hi], w[which])
        lr = spec.lr_critic if which == 0 else spec.lr_actor
        n = k[which]
        pe, me, ve = adam_expect(before[PARAMS][lo:hi], before[ADAM_M][lo:hi], before[ADAM_V][lo:hi], ghat, lr,
                                 spec.beta1 ** n, spec.beta2 ** n)
        for arena, exp in ((PARAMS, pe), (ADAM_M, me), (ADAM_V, ve)):
            assert np.array_equal(after[arena][lo:hi].view(np.uint32), exp.view(np.uint32)), (what, which, arena)


# ---- the solver alone ---------------------------------------------------------------------------------------------
def _device_solve(G, c):
    from distributed_sac_b200 import _lib
    lib = _lib.load()
    T = G.shape[0]
    G = np.ascontiguousarray(G, np.float64)
    w, p = np.empty(T, np.float32), np.empty(T, np.float64)
    sc = {k: C.c_double() for k in ("lambda", "best", "first", "scale")}
    ib = C.c_int32()
    _lib.check(lib.b200sac_cagrad_solve_test(T, G.ctypes.data, float(c), w.ctypes.data, p.ctypes.data,
                                             *[C.addressof(sc[k]) for k in ("lambda", "best", "first", "scale")],
                                             C.addressof(ib)))
    rec = {k: np.array([v.value]) for k, v in sc.items()}
    rec.update(p=p[None], ibest=np.array([ib.value]), w=w)
    return rec


@pytest.mark.parametrize("T,kind,c,G", gram_sets(), ids=[f"T{T}-{k}-c{c}" for T, k, c, _ in gram_sets()])
def test_solver_matches_host(cuda, T, kind, c, G):
    rec = _device_solve(G, c)
    ref = cr.solve(G, c)
    _check_record(rec, 0, ref, f"T{T} {kind}")
    assert _ulps(rec["w"], ref["w32"]).max() <= 1, (T, kind, rec["w"], ref["w32"])


def test_solver_degenerate(cuda):
    for G in (np.zeros((3, 3)), np.array([[1.0, np.nan], [np.nan, 1.0]]), np.diag([np.inf, 1.0, 2.0])):
        rec = _device_solve(G, 0.5)
        ref = cr.solve(G, 0.5)
        assert rec["ibest"][0] == -2 and np.array_equal(rec["w"], np.ones(G.shape[0], np.float32))
        assert np.isnan(rec["p"]).all() and np.isnan(rec["lambda"][0])
        assert (math.isnan(ref["scale"]) and math.isnan(rec["scale"][0])) or rec["scale"][0] == ref["scale"]


# ---- whole steps ------------------------------------------------------------------------------------------------------
def _check_step(core, spec, r, before, b, e1, e2, what):
    """One CAGrad step of replica r against the oracle and the kernel's exact arithmetic."""
    T = spec.num_tasks
    pc = core.read_pcgrad(r)
    cg = core.read_cagrad(r)
    slices = np.stack([core.export_task_grad(t, r).numpy() for t in range(T)])
    after = _state(core, r)
    assert pc["task_mismatch"] == 0 and not pc["projected"].any(), what
    batch = [x[r] for x in b]
    p0 = _unflat(core, before[PARAMS], list(core.table))
    p1 = _unflat(core, after[PARAMS], list(core.table))
    for which in (0, 1):
        lo, hi = _opt_range(core, which)
        sl = slices[:, lo:hi].astype(np.float64)
        G = pc["gram"][which]
        ref = sl @ sl.T
        assert np.allclose(G, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max()), (what, which)
        host = cr.solve(G, C_DEF)
        _check_record(cg, which, host, what)
        assert _ulps(pc["w"][which], host["w32"]).max() <= 1, (what, which)
        src = dict(p0)
        if which == 1:
            for n in sp.param_names(spec, ("q1", "q2"), False):
                src[n] = p1[n]
        forced = cuda_relu_masks(core, spec, r)
        with sp.ReluTape(forced) as tape:
            ref_t = pr.task_grads(spec, src, batch, e1[r], e2[r], which)
        check_forced(tape, {k: v for k, v in forced.items() if k in tape.z}, what)
        for t in range(T):
            got = _unflat(core, slices[t], pr.opt_names(spec, which))
            for n in pr.opt_names(spec, which):
                assert _rel(got[n].numpy(), ref_t[t][n].numpy()) < 1e-4, (what, which, t, n)
    _check_adam(core, spec, r, before, after, slices, pc["w"], what)
    tau, omt = np.float32(spec.tau), np.float32(1.0 - spec.tau)
    for n in sp.param_names(spec, ("q1", "q2"), False):
        tn = n.replace("q1.", "q1_target.").replace("q2.", "q2_target.")
        exp = tau * p1[n].numpy() + omt * p0[tn].numpy()
        assert np.array_equal(p1[tn].numpy().view(np.uint32), exp.astype(np.float32).view(np.uint32)), (what, tn)
    return pc, cg


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("T", [2, 3, 10])
@pytest.mark.parametrize("R", [1, 3])
def test_cagrad_step(cuda, precision, T, R):
    spec = _spec(T)
    core = _core(spec, precision, R)
    for r in range(R):
        core.set_named(_params(spec, 11 + 7 * r, move_targets=True), PARAMS, r)
    before = [_state(core, r) for r in range(R)]
    b, e1, e2 = _data(spec, R)
    core.step(*b, e1, e2)
    torch.cuda.synchronize()
    for r in range(R):
        _, cg = _check_step(core, spec, r, before[r], b, e1, e2, f"p{precision} T{T} R{R} r{r}")
        assert (cg["ibest"] >= 0).all()


def _conflict_batch(spec, step):
    """Two tasks with the same states, actions and next states, and rewards of opposite sign."""
    b, e1, e2 = _data(spec, 1, step=step)
    P = spec.batch // 2
    for j in (0, 1, 3):
        b[j][0, P:] = b[j][0, :P]
    for j in (0, 3):
        b[j][0, P:, spec.state_dim:] = b[j][0, :P, spec.state_dim:].flip(-1)
    b[2][0, :P] = 5.0 + b[2][0, :P].abs()
    b[2][0, P:] = -b[2][0, :P]
    return b, e1, e2


def _oracle_steps(core, spec, batches, what, c=C_DEF, r=0, port=None):
    """Each (b, e1, e2) stepped on the device and on cagrad_update with the step's ReLU masks, tanh values and min
    routing forced; after every step the whole state agrees to 1e-4."""
    if port is None:
        port = sp.PortLearner(spec, sp.init_params(spec))
        sync_core_to_port(core, port, r)
    recs = []
    for i, (b, e1, e2) in enumerate(batches):
        core.step(*b, e1, e2)
        pc, cg = core.read_pcgrad(r), core.read_cagrad(r)
        forced = cuda_relu_masks(core, spec, r)
        with sp.ReluTape(forced) as tape:
            ref = cr.cagrad_update(port, *[x[r] for x in b], e1[r], e2[r], c)
        check_forced(tape, forced, f"{what} step {i}")
        for which in (0, 1):
            G, w32, _ = ref[which]
            assert np.allclose(pc["w"][which], w32, rtol=1e-4, atol=1e-4), (what, i, which)
            assert np.allclose(pc["gram"][which], G, rtol=2e-4, atol=1e-4 * np.abs(G).max()), (what, i, which)
        check_port_state(core, port, r)
        recs.append((pc, cg))
    return recs


def test_conflict_matches_oracle(cuda):
    """Five steps on conflicting tasks against the CAGrad oracle; the weights move away from 1."""
    spec = _spec(2)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 3, move_targets=True), PARAMS, 0)
    recs = _oracle_steps(core, spec, [_conflict_batch(spec, k) for k in range(5)], "conflict")
    assert all((cg["ibest"] >= 0).all() for _, cg in recs)
    assert any(not np.allclose(pc["w"][0], 1.0) for pc, _ in recs)


def test_full_size_ms_matches_oracle(cuda):
    """The MT10 MTSAC shape (39 + 10 inputs, 4 actions, 400^3, batch 1280, T 10) at precision 1: two steps."""
    spec = sp.ms_spec()
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 4, move_targets=True), PARAMS, 0)
    _oracle_steps(core, spec, [_data(spec, 1, step=k) for k in range(2)], "MS")


def test_plain_pcgrad_cagrad_side_by_side(cuda):
    """One handle, three replicas: plain sum (PCGrad off, c = 0), PCGrad, CAGrad; two steps, each against its oracle."""
    spec = _spec(3)
    core = _core(spec, 0, 3, c=0.0)
    core.set_pcgrad(critic=True, actor=True, replica=1)
    core.set_cagrad(critic=C_DEF, actor=C_DEF, replica=2)
    ports = []
    for r in range(3):
        core.set_named(_params(spec, 31 + r, move_targets=True), PARAMS, r)
        ports.append(sp.PortLearner(spec, sp.init_params(spec)))
        sync_core_to_port(core, ports[r], r)
    for step in range(2):
        b, e1, e2 = _data(spec, 3, step=step, seed=40)
        core.step(*b, e1, e2)
        for r in range(3):
            pc, cg = core.read_pcgrad(r), core.read_cagrad(r)
            forced = cuda_relu_masks(core, spec, r)
            args = [x[r] for x in b] + [e1[r], e2[r]]
            with sp.ReluTape(forced) as tape:
                if r == 1:
                    ref = pr.pcgrad_update(ports[r], *args, pc["perm"])
                else:
                    ref = cr.cagrad_update(ports[r], *args, 0.0 if r == 0 else C_DEF)
            check_forced(tape, forced, f"r{r} step {step}")
            if r == 0:
                assert np.array_equal(pc["w"], np.ones((2, 3), np.float32)) and list(cg["ibest"]) == [-1, -1]
                assert np.isnan(cg["p"]).all() and np.isnan(cg["lambda"]).all()
            elif r == 1:
                assert list(cg["ibest"]) == [-1, -1]
                for which in (0, 1):
                    assert np.array_equal(pc["projected"][which], ref[which][2])
            else:
                assert (cg["ibest"] >= 0).all() and not pc["projected"].any()
                for which in (0, 1):
                    _check_record(cg, which, cr.solve(pc["gram"][which], C_DEF), f"r2 step {step}")
            check_port_state(core, ports[r], r)


def _ring_core(spec, c):
    """A precision-1 CAGrad handle at c with a prepared device ring whose two tasks have rewards of opposite sign."""
    from distributed_sac_b200.core import Replay
    core = _core(spec, 1, 1, c=c)
    core.set_named(_params(spec, 3, move_targets=True), PARAMS, 0)
    rb = Replay(core, 4096, "device", seed=3)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=4, batch=2000)
    r = torch.where(s[:, spec.state_dim:spec.state_dim + 1] > 0, 5.0 + r.abs(), -5.0 - r.abs())
    rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    core.prepare(rb)
    return core, rb


def test_coefficient_between_prepared_graphs(cuda):
    """c set in stream order between two launches of prepared graphs, with no host synchronisation between them, applies
    to the second step and not to the first: the result equals a run that synchronised before the change, bit for bit,
    and differs from a run that had c from the start."""
    spec = _spec(2)
    runs = {}
    for mode in ("enqueued", "synced", "from_start"):
        core, rb = _ring_core(spec, C_DEF if mode == "from_start" else 0.0)
        stream = torch.cuda.Stream()
        try:
            with torch.cuda.stream(stream):
                core.step_sampled(rb, 1)
                if mode == "synced":
                    stream.synchronize()
                core.set_cagrad(critic=C_DEF, actor=0.0)
                assert core.get_cagrad(0) == {"critic": C_DEF, "actor": 0.0}
                core.step_sampled(rb, 1)
            stream.synchronize()
            runs[mode] = (_state(core, 0), core.read_pcgrad(0), core.read_cagrad(0))
        finally:
            rb.close()
    for mode, (_, pc, cg) in runs.items():
        assert cg["ibest"][0] >= 0 and cg["ibest"][1] == -1, mode
        assert np.array_equal(pc["w"][1], np.ones(2, np.float32)), mode
        _check_record(cg, 0, cr.solve(pc["gram"][0], C_DEF), mode)
    for k in (PARAMS, ADAM_M, ADAM_V):
        assert np.array_equal(runs["enqueued"][0][k].view(np.uint32), runs["synced"][0][k].view(np.uint32)), k
    assert not np.array_equal(runs["enqueued"][0][PARAMS], runs["from_start"][0][PARAMS])


def test_critic_only_step_leaves_actor(cuda):
    spec = _spec(2)
    core = _core(spec, 1, 1)
    core.set_named(_params(spec, 8, move_targets=True), PARAMS, 0)
    core.set_update_intervals(actor_every=2)
    lo, hi = _opt_range(core, 1)
    p0 = core.export_arena(PARAMS, 0).numpy().copy()
    b, e1, e2 = _data(spec, 1)
    core.step(*b, e1, e2)
    pc, cg = core.read_pcgrad(0), core.read_cagrad(0)
    assert np.isnan(pc["w"][1]).all() and np.isfinite(pc["w"][0]).all()
    assert cg["ibest"][0] >= 0 and cg["ibest"][1] == -1
    assert np.isnan(cg["p"][1]).all() and all(np.isnan(cg[k][1]) for k in ("lambda", "best", "first", "scale"))
    assert np.array_equal(core.export_arena(PARAMS, 0).numpy()[lo:hi].view(np.uint32), p0[lo:hi].view(np.uint32))


@pytest.mark.parametrize("ring", ["prioritized", "linked"])
def test_sampled_rings(cuda, ring):
    """Sampled steps on a prioritized ring and on a linked ring at n = 3: rows in task blocks, the record against the
    host solve, and Adam bit for bit on the weighted slices."""
    from distributed_sac_b200.core import Replay
    spec = _spec(3)
    core = _core(spec, 0, 1)
    core.set_named(_params(spec, 6, move_targets=True), PARAMS, 0)
    rb = Replay(core, 4096, "device", seed=5, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-3) if ring == "prioritized" else None,
                trajectories=ring == "linked")
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=8, batch=3000)
    if ring == "linked":
        rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy(), stream=s[:, spec.state_dim:].argmax(1).numpy())
        rb.set_nstep(3)
    else:
        rb.push(s.numpy(), a.numpy(), r.numpy(), s2.numpy(), d.numpy())
    try:
        for k in range(3):
            before = _state(core, 0)
            core.step_sampled(rb, 1)
            pc, cg = core.read_pcgrad(0), core.read_cagrad(0)
            assert pc["task_mismatch"] == 0 and (cg["ibest"] >= 0).all(), (ring, k)
            for which in (0, 1):
                _check_record(cg, which, cr.solve(pc["gram"][which], C_DEF), f"{ring} step {k}")
            slices = np.stack([core.export_task_grad(t, 0).numpy() for t in range(3)])
            _check_adam(core, spec, 0, before, _state(core, 0), slices, pc["w"], f"{ring} step {k}")
    finally:
        rb.close()


def test_refusals_and_launch_count(cuda):
    from distributed_sac_b200.core import SacCore
    spec = _spec(2)
    plain = SacCore(core_config(spec, precision=1), 0)
    with pytest.raises(RuntimeError):
        plain.set_cagrad(critic=0.5)
    core = _core(spec, 1, 2)
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(RuntimeError):
            core.set_cagrad(critic=bad, replica=1)
        assert core.get_cagrad(1) == {"critic": C_DEF, "actor": C_DEF}
    with pytest.raises(RuntimeError):
        core.set_cagrad(critic=0.5, replica=2)
    pcg = SacCore(dataclasses.replace(core_config(spec, precision=1), pcgrad=True), 0)
    assert pcg.get_cagrad(0) == {"critic": 0.0, "actor": 0.0}
    rec = pcg.read_cagrad(0)
    assert list(rec["ibest"]) == [-1, -1] and np.isnan(rec["p"]).all()
    assert core.launches_per_step == pcg.launches_per_step
    # copy_replica leaves dst's coefficients as they were
    core.set_cagrad(critic=0.25, actor=0.0, replica=1)
    core.copy_replica(0, 1)
    assert core.get_cagrad(1) == {"critic": 0.25, "actor": 0.0}


MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


def test_mtsac_learner_host_ring(cuda, tmp_path):
    """MTSACLearner(cagrad=0.5).update() through the pinned-host ring (the learner's default): both PCGrad switches off,
    c on both optimizers, a finite record; set_cagrad(0) gives the plain sum on the next update."""
    from distributed_sac_b200.learner import MTSACLearner
    p = tmp_path / "ms.json"
    p.write_text(json.dumps(MS_CFG))
    lrn = MTSACLearner(None, ["t0", "t1", "t2"], str(p), write_mode=False, replay_where="host", cagrad=0.5,
                       server=redis_stub.StrictRedis(host=str(tmp_path) + "ms"))
    try:
        assert lrn.core.get_pcgrad(0) == {"critic": False, "actor": False}
        assert lrn.core.get_cagrad(0) == {"critic": 0.5, "actor": 0.5}
        lrn.memory.ring.fill_synthetic(4096, seed=1)
        for _ in range(3):
            assert all(x == x for x in lrn.update())
            pc, cg = lrn.core.read_pcgrad(0), lrn.core.read_cagrad(0)
            assert pc["task_mismatch"] == 0 and np.isfinite(pc["w"]).all() and (cg["ibest"] >= 0).all()
            for which in (0, 1):
                _check_record(cg, which, cr.solve(pc["gram"][which], 0.5), "learner")
        lrn.set_cagrad(0.0)
        lrn.update()
        assert np.array_equal(lrn.core.read_pcgrad(0)["w"], np.ones((2, 3), np.float32))
    finally:
        lrn.memory.stop()


def test_learner_refusals(cuda, tmp_path):
    """cagrad= with pcgrad=True, on the single-task learners or on CARE: ValueError before any handle is built."""
    from _harness import LEARNER_CFGS
    from distributed_sac_b200 import learner as L
    srv = lambda tag: redis_stub.StrictRedis(host=str(tmp_path) + tag)     # noqa: E731
    ms = tmp_path / "ms.json"
    ms.write_text(json.dumps(MS_CFG))
    for kw in (dict(pcgrad=True, cagrad=0.5), dict(cagrad=-1.0), dict(cagrad=float("nan"))):
        with pytest.raises(ValueError):
            L.MTSACLearner(None, ["t0", "t1", "t2"], str(ms), write_mode=False, server=srv("ms"), **kw)
    for fam, cls in (("LL", L.LunarLanderLearner), ("VS", L.VSACLearner)):
        p = tmp_path / f"{fam}.json"
        p.write_text(json.dumps(LEARNER_CFGS[fam]))
        with pytest.raises(ValueError):
            cls(str(p), write_mode=False, server=srv(fam), cagrad=0.5)
    pc = tmp_path / "care.json"
    pc.write_text(json.dumps(dict(MS_CFG, encoder={}, use_modified_care=True)))
    with pytest.raises(ValueError):
        L.CARELearner(None, ["t0", "t1", "t2"], str(pc), write_mode=False, cagrad=0.5, server=srv("care"))
