"""Every Adam step, bit for bit, and the gradients it reads against the autograd oracle.

One Adam step moves an element by at most about lr (3e-4 here), about 0.5 % of a Xavier weight's norm: the 1e-4
relative-L2 bar of the parity tests accepts an error of up to ~2 % of the update, and a larger one on a few elements.  No
bar is needed.  The library is built with -fmad=false and without fast-math, and every writer of the update -- adam_kernel
of the per-layer and CARE plans (split-K gradient slices added in index order, replica strides, counter slots 0 critic,
1 actor, 4 CARE(O) context encoder), the fused optimizer epilogue of the layer-chained plan's wgrad_kernel (float4 body,
bias rows), the temperature Adam of the TAIL_ALPHA_AND_LOSSES job -- evaluates adam_scalars / adam_one with one rounding
per operation, in source order, from readable state: p, m, v before the step, the gradient it consumed (GRADS after the
step; b200sac_export adds the split-K slices in adam_kernel's order), the replica's learning rate and the fp64 bias
corrections Counters::b1p / b2p.  The counters are modelled here as the library keeps them: pow(beta, t) after
b200sac_set_steps, then one multiplication by beta per step that advances the slot (critic-only steps skip the actor and
the temperature).  So every trainable element must equal adam_expect() of its own slot as a bit pattern, and the gaps
between tensors must not change.  A failing tensor is tested against the mistakes that would explain it (another slot's
rate or count, another replica's row, t - 1 / t + 1, the gradient without its split-K slices, fp64 or FMA evaluation), and
the message names the one that reproduces it.

Bit-exactness on top of wrong gradients would prove nothing, so the first checked step of every plan also compares GRADS
with the gradients the oracle's optimizers consume (captured at each optimizer's step(), CUDA masks forced) at 1e-4 per
tensor.  The CPU test at the end ties adam_expect to torch.optim.Adam, the reference's optimizer.
"""
import numpy as np
import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import kink_checked_step
from _harness import (ADAM_M, ADAM_V, LEARNER_CFGS, ROWS, _bits, _handle, _inputs, _learner, adam_expect, capture_grads,
                      check_adam, check_grads, cuda, new_model, snapshot)


def set_steps(core, model, r, steps):
    core.set_steps(steps, r)
    got = core.get_steps(r)
    model[r].seed(list(got) + [0] * (4 - len(got)))      # set_steps reseeds every slot it does not name from its count


def plant_edges(core, r):
    """Three real elements per trainable tensor: m = v = 0 (a fresh element), a denormal v, a tiny m."""
    m, v = core.export_arena(ADAM_M, r).numpy().copy(), core.export_arena(ADAM_V, r).numpy().copy()
    for name, (off, rows, cols, tr, _o, pitch) in core.table.items():
        if not tr:
            continue
        n = rows * cols
        for j, (mm, vv) in enumerate(((0.0, 0.0), (None, 1e-41), (1e-30, None))):
            r_, c_ = divmod((j * (n // 3 + 1) + 1) % n, cols)
            i = off + r_ * pitch + c_
            if mm is not None:
                m[i] = mm
            if vv is not None:
                v[i] = vv
    core.import_arena(torch.from_numpy(m), ADAM_M, r)
    core.import_arena(torch.from_numpy(v), ADAM_V, r)


def checked_steps(core, spec, care, model, n_steps, what, step_fn=None, actor_every=1, first=0):
    """n_steps steps (default: b200sac_step on _inputs), each replica checked after each; returns {slot: moved elements}
    summed over replicas and steps, and the actor steps seen per replica."""
    R = core.cfg.replicas
    moved, acts = {}, [0] * R
    for i in range(n_steps):
        before = [snapshot(core, r) for r in range(R)]
        if step_fn is None:
            b, e1, e2 = _inputs(spec, care, R, first + i)
            core.step(*b, e1, e2)
        else:
            step_fn(i)
        for r in range(R):
            act = model[r].bump(actor_every)
            acts[r] += act
            assert core.get_steps(r) == model[r].steps(len(core.get_steps(r))), (what, i, r)
            for s, k in check_adam(core, model, r, before[r], snapshot(core, r, True), act,
                                   f"{what} step {i} replica {r}").items():
                moved[s] = moved.get(s, 0) + k
    return moved, acts


def assert_moved(moved, care_o, what):
    want = (0, 1, 2) + ((4,) if care_o else ())
    assert all(moved.get(s, 0) > 0 for s in want), f"{what}: a slot never moved a parameter ({moved}): the case is vacuous"


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's gradients
# ---------------------------------------------------------------------------------------------------------------------
def _port_of(core, spec, care, r=0):
    """An oracle learner holding replica r's state, rates and counts."""
    named = core.get_named(0, r)
    st = {"m": core.get_named(ADAM_M, r), "v": core.get_named(ADAM_V, r), "step": core.get_steps(r)}
    port = cp.CarePortLearner(spec, named, st) if care else sp.PortLearner(spec, named, st)
    hp = core.get_hparams(r)
    for opt, key in ((port.opt_critic, "lr_critic"), (port.opt_actor, "lr_actor"), (port.opt_alpha, "lr_alpha"),
                     (getattr(port, "opt_ctx", None), "lr_ctx")):
        if opt is not None:
            for grp in opt.param_groups:
                grp["lr"] = hp[key]
    return port


def oracle_checked_step(core, spec, care, model, i, what):
    """One step of replica 0 checked twice: GRADS against the oracle's consumed gradients, and the update exactly."""
    port = _port_of(core, spec, care)
    ref = capture_grads(port)
    set_steps(core, model, 0, core.get_steps(0))     # kink_checked_step reseeds the counters from the oracle's counts
    before = snapshot(core, 0)
    b, e1, e2 = _inputs(spec, care, 1, 100 + i)
    kink_checked_step(core, port, spec, [x[0] for x in b], e1[0], e2[0], care=care)
    act = model[0].bump()
    after = snapshot(core, 0, True)
    check_grads(core, ref, what)
    return check_adam(core, model, 0, before, after, act, what)


# ---------------------------------------------------------------------------------------------------------------------
# 1: every plan and writer: counts of their own per slot, edge elements, gradients against the oracle
# ---------------------------------------------------------------------------------------------------------------------
PLANS = ["chained_ll", "chained_deep8", "chained_big_odd", "vs400_fp32", "vs400_tc", "split517_fp32", "split517_tc",
         "wide1024_tc", "mtsac_t10", "mtsac_t64", "care_m", "care_o"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", PLANS)
def test_adam_is_exact(cuda, name):
    core, spec, care = _handle(name)
    care_o = care and core.cfg.care_original
    model = new_model(core)
    checked_steps(core, spec, care, model, 2, f"{name} warm-up")
    set_steps(core, model, 0, (7, 1, 10 ** 6, 3))
    plant_edges(core, 0)
    moved = oracle_checked_step(core, spec, care, model, 0, f"{name} oracle step")
    more, _ = checked_steps(core, spec, care, model, 2, name, first=10)
    for s, k in more.items():
        moved[s] = moved.get(s, 0) + k
    assert_moved(moved, care_o, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: three replicas, each its own rates (one at lr = 0) and its own counts 0, 1, 7, 10^6 per slot
# ---------------------------------------------------------------------------------------------------------------------
R3_PLANS = ["chained_ll", "chained_big_odd", "vs400_tc", "split517_fp32", "mtsac_t10", "care_m", "care_o"]
R3_COUNTS = [(10 ** 6, 7, 1, 0), (1, 0, 7, 10 ** 6), (7, 10 ** 6, 0, 1)]   # replica 1 trains at lr = 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", R3_PLANS)
def test_adam_is_exact_per_replica(cuda, name):
    rows = [dict(ROWS[0]), dict(ROWS[1], lr_critic=0.0, lr_actor=0.0, lr_alpha=0.0, lr_ctx=0.0), dict(ROWS[2])]
    core, spec, care = _handle(name, R=3, rows=rows)
    model = new_model(core)
    for r in range(3):
        set_steps(core, model, r, R3_COUNTS[r])
        plant_edges(core, r)
    p1 = snapshot(core, 1)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} R = 3")
    assert_moved(moved, care and core.cfg.care_original, name)
    after = snapshot(core, 1)
    assert np.array_equal(_bits(after[0]), _bits(p1[0])), "replica 1 (lr = 0) moved a parameter"
    assert not np.array_equal(after[1], p1[1]), "replica 1 (lr = 0) did not update its moments"
    assert model[0].b2p[0] == 0.0 and model[2].b2p[1] == 0.0, "b2p did not underflow at 10^6 steps"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: actor every 3rd, targets every 2nd step: the critic exact on every step, actor and temperature on actor steps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "vs400_tc", "split517_fp32", "mtsac_t10", "care_o"])
def test_adam_is_exact_under_update_intervals(cuda, name):
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    core.set_update_intervals(actor_every=3, target_every=2)
    model = new_model(core)
    set_steps(core, model, 1, (4, 1, 1, 4))
    moved, acts = checked_steps(core, spec, care, model, 6, f"{name} actor_every = 3", actor_every=3)
    assert acts == [2, 2], f"expected two actor steps per replica in six, saw {acts}"
    assert_moved(moved, care and core.cfg.care_original, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: state carried over: copy_replica, a Learner checkpoint restore
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "split517_tc", "care_o"])
def test_adam_is_exact_after_copy_replica(cuda, name):
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    checked_steps(core, spec, care, model, 2, f"{name} warm-up")
    set_steps(core, model, 0, (7, 1, 10 ** 6, 3))
    core.copy_replica(0, 1)
    model[1] = model[0].copy()
    assert core.get_steps(1) == core.get_steps(0)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} after copy_replica", first=20)
    assert_moved(moved, care and core.cfg.care_original, name)
    core.close()


@pytest.mark.gpu
def test_adam_is_exact_after_checkpoint_restore(cuda, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    a = _learner("LL", tmp_path)
    spec = sp.ll_spec(batch=LEARNER_CFGS["LL"]["batch_size"])
    try:
        for i in range(3):
            b, e1, e2 = _inputs(spec, False, 1, i)
            a.core.step(*b, e1, e2)
        path = a.save_checkpoint(5)
    finally:
        a.memory.stop()
    lrn = _learner("LL", tmp_path)
    try:
        lrn.load_checkpoint(path)
        core = lrn.core
        assert core.get_steps() == (3, 3, 3)
        model = new_model(core)
        model[0].seed(list(core.get_steps()) + [0])         # load_checkpoint -> set_steps: pow(beta, t)
        moved, _ = checked_steps(core, spec, False, model, 2, "LL after load_checkpoint", first=30)
        assert_moved(moved, False, "checkpoint restore")
    finally:
        lrn.memory.stop()


# ---------------------------------------------------------------------------------------------------------------------
# 5: the other entry points: step_sampled from a device ring (graph path), step_host
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "split517_tc", "care_o"])
def test_sampled_step_adam_is_exact(cuda, name):
    from distributed_sac_b200.core import Replay
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    set_steps(core, model, 1, (7, 1, 10 ** 6, 3))
    cap = 4 * spec.batch * max(spec.num_tasks, 1)
    ring = Replay(core, cap, "device", seed=5)
    ring.fill_synthetic(cap, seed=6)
    moved, _ = checked_steps(core, spec, care, model, 3, f"{name} step_sampled", step_fn=lambda i: core.step_sampled(ring, 1))
    assert_moved(moved, care and core.cfg.care_original, name)
    ring.close()
    core.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["vs400_fp32"])
def test_host_step_adam_is_exact(cuda, name):
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    set_steps(core, model, 0, (7, 1, 10 ** 6))

    def step(i):
        b, e1, e2 = _inputs(spec, care, 2, 40 + i)
        core.step_host(*b, e1, e2)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} step_host", step_fn=step)
    assert_moved(moved, False, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6 (CPU): the specification against the reference's optimizer
# ---------------------------------------------------------------------------------------------------------------------
def test_adam_expect_follows_torch_adam():
    """adam_expect against torch.optim.Adam (CPU defaults) over six steps of random fp32 state with tiny and zero
    gradients.  torch contracts lerp_ / addcmul_ into FMAs, so m and v may differ in the last bits; p must agree to
    1e-3 of the update bound lr, m and v to a few ulp of the magnitudes they are formed from."""
    lr, beta1, beta2, eps = 3e-4, 0.9, 0.999, 1e-8
    rng = np.random.default_rng(7)
    n = 200_000
    p0 = (rng.standard_normal(n) * 0.0625).astype(np.float32)
    param = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([param], lr=lr, betas=(beta1, beta2), eps=eps)
    p, m, v = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    ulp = np.finfo(np.float32).eps
    differ = 0
    for t in range(1, 7):
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 0, n)).astype(np.float32)
        g[rng.random(n) < 0.05] = 0.0
        g[rng.random(n) < 0.02] = np.float32(1e-30) * rng.standard_normal()
        param.grad = torch.from_numpy(g.copy())
        opt.step()
        scale_m = np.abs(m) + np.abs(g) * np.float32(1 - beta1)
        scale_v = np.abs(v) + np.float32(1 - beta2) * g * g
        p, m, v = adam_expect(p, m, v, g, lr, beta1 ** t, beta2 ** t, beta1, beta2, eps)
        st = opt.state[param]
        tm, tv, tp = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy(), param.detach().numpy()
        assert np.abs(tp.astype(np.float64) - p).max() <= 1e-3 * lr, t
        assert (np.abs(tm.astype(np.float64) - m) <= 2 * ulp * scale_m).all(), t
        assert (np.abs(tv.astype(np.float64) - v) <= 2 * ulp * scale_v).all(), t
        differ += int((tm != m).sum())
        # keep the two trajectories from drifting apart: continue from torch's state
        p, m, v = tp.copy(), tm.copy(), tv.copy()
    assert differ > 0, "torch and adam_expect agree bit for bit: the bars are not exercised"
