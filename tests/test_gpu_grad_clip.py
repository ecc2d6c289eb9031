"""GPU: gradient-norm clipping per replica and optimizer (b200sac_cfg.grad_clip, b200sac_set_grad_clip) and the gradient
norms of every step (b200sac_read_grad_norms).

A grad_clip handle runs torch.nn.utils.clip_grad_norm_(params, max_norm) right before each optimizer's step(): the
critic, the actor and the CARE(O) context encoder, not the temperature.  Checked here, over the layer-chained plan, the
per-layer plan at both precisions (with and without split-K gradient slices, MTSAC with forked weight gradients) and both
CARE variants:
  * the clipped steps follow the autograd oracle given the same thresholds (CUDA masks forced), from a state with non-zero
    Adam moments -- from zero moments Adam is nearly scale-invariant, so a dropped coefficient would barely show -- and the
    same steps unclipped end far away from there;
  * the step is exact: the reported norm is the fp64 norm of the exported gradient, the coefficient is the host formula
    applied to it, and Adam's update equals adam_expect on fp32(g * coef) bit for bit;
  * +inf and never-binding thresholds leave every bit as a handle without grad_clip leaves it;
  * replicas clip independently, critic-only steps skip the actor, set_grad_clip is stream-ordered, runs repeat bit for bit;
  * bad arguments are refused without a change, and the Learner classes expose it through max_grad_norm=.
"""
import json
import math

import numpy as np
import pytest
import torch

import care_port as cp
import redis_stub
import sac_port as sp
from _clip import clip_oracle
from _golden import REL, check_port_state, core_config, kink_checked_step, rel_l2
from _harness import (ADAM_M, ADAM_V, LEARNER_CFGS, PARAMS, SMALL, _bits, _config, _inputs, _params, _plan, _slots, check_adam,
                      cuda, new_model, plan_labels, snapshot)

pytestmark = pytest.mark.gpu

PLANS = ["chained", "chained_deep8", "vs400_fp32", "vs400_tc", "split517_tc", "mtsac_weighted", "care_m", "care_o"]
COLS = (("critic", 0, 0), ("actor", 1, 1), ("ctx", 2, 4))     # (oracle key, norm column, Counters slot)
INF = math.inf


def _clip_handle(name, R=1, seed=0, grad_clip=True):
    """(core, spec, care) of a _plan id created with grad_clip, each replica with its own parameters (targets off their
    locals)."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = _plan(name)
    core = SacCore(_config(spec, care, precision, R, grad_clip=grad_clip), 0, seed=seed)
    for r in range(R):
        core.set_named(_params(spec, 11 + 7 * r, care, move_targets=True), PARAMS, r)
    return core, spec, care


def _port_of(core, spec, care, max_grad_norm=None, r=0):
    """An oracle learner holding replica r's state, rates and counts, clipped at max_grad_norm (None: unclipped)."""
    named = core.get_named(PARAMS, r)
    st = {"m": core.get_named(ADAM_M, r), "v": core.get_named(ADAM_V, r), "step": core.get_steps(r)}
    port = clip_oracle((cp.CarePortLearner if care else sp.PortLearner)(spec, named, st), max_grad_norm)
    hp = core.get_hparams(r)
    for opt, key in ((port.opt_critic, "lr_critic"), (port.opt_actor, "lr_actor"), (port.opt_alpha, "lr_alpha"),
                     (getattr(port, "opt_ctx", None), "lr_ctx")):
        if opt is not None:
            for grp in opt.param_groups:
                grp["lr"] = hp[key]
    return port


def _steps(core, spec, care, first, n):
    for i in range(first, first + n):
        b, e1, e2 = _inputs(spec, care, core.cfg.replicas, i)
        core.step(*b, e1, e2)


def _binding(core, r=0, scale=0.25):
    """{critic, actor, ctx}: scale x the norms of the last step (inf where an optimizer did not step)."""
    n = core.read_grad_norms(1)[0, r]
    return {k: (scale * float(n[col]) if math.isfinite(float(n[col])) else INF) for k, col, _ in COLS}


def _check_clipped_step(core, model, before, act, what, r=0, binding=True):
    """One step of replica r, exactly: every reported norm against the fp64 norm of the exported gradient (rel 1e-6), the
    coefficient against the host formula (1 ulp), then every Adam write bit for bit with g' = fp32(g * coef) of its
    optimizer (the temperature unclipped).  Returns the coefficients."""
    after = snapshot(core, r, True)
    slot, _ = _slots(core)
    g = after[3].copy()
    norms = core.read_grad_norms(1)[0, r]
    coef = core.debug("clip", r).numpy()
    thr = core.get_grad_clip(r)
    for k, col, s in COLS:
        sel = slot == s
        if not sel.any() or (s == 1 and not act):
            assert math.isnan(float(norms[col])), f"{what}: {k} did not step but reports norm {float(norms[col])}"
            continue
        want = math.sqrt(float(np.sum(np.square(g[sel].astype(np.float64)))))
        got = float(norms[col])
        assert abs(got - want) <= 1e-6 * want, f"{what}: {k} norm {got!r}, fp64 norm of GRADS {want!r}"
        c_host = np.float32(min(1.0, thr[k] / (want + 1e-6)))
        ulps = abs(int(_bits([coef[col]])[0]) - int(_bits([c_host])[0]))
        assert ulps <= 1, f"{what}: {k} coefficient {coef[col]!r}, host formula {c_host!r}"
        if binding:
            assert coef[col] < 1.0, f"{what}: {k} threshold {thr[k]} not binding at norm {want}"
        g[sel] = g[sel] * np.float32(coef[col])          # one fp32 multiply
    check_adam(core, model, r, before, after[:3] + [g], act, what)
    return coef


# ---------------------------------------------------------------------------------------------------------------------
# 1: the oracle, from non-zero Adam moments, with thresholds binding on every step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PLANS)
def test_clipped_steps_match_oracle(cuda, name):
    core, spec, care = _clip_handle(name)
    _steps(core, spec, care, 0, 2)                          # unclipped warm-up: Adam moments of every optimizer != 0
    batches = [_inputs(spec, care, 1, 100 + i) for i in range(4)]
    unpack = lambda bt: ([x[0] for x in bt[0]], bt[1][0], bt[2][0])
    probe = _port_of(core, spec, care, max_grad_norm=INF)
    b, e1, e2 = unpack(batches[0])
    (probe.update if care else probe.update_SAC)(*b, e1, e2)
    thr = 0.25 * min(probe.grad_norms.values())
    core.set_grad_clip(critic=thr, actor=thr, ctx=thr)
    port, free = _port_of(core, spec, care, max_grad_norm=thr), _port_of(core, spec, care)
    for i, bt in enumerate(batches):
        b, e1, e2 = unpack(bt)
        kink_checked_step(core, port, spec, b, e1, e2, care=care)
        (free.update if care else free.update_SAC)(*b, e1, e2)
        check_port_state(core, port)
        got = core.read_grad_norms(1)[0, 0]
        for k, col, _ in COLS:
            if k not in port.grad_norms:
                assert math.isnan(float(got[col])), (name, i, k)
                continue
            ref = port.grad_norms[k]
            assert ref > thr, f"{name} step {i}: {k} norm {ref} below the threshold {thr}: the step is not clipped"
            assert abs(float(got[col]) - ref) <= REL * ref, f"{name} step {i}: {k} norm {float(got[col])} vs oracle {ref}"
    # the same steps without clipping end elsewhere, in the critic and in the actor
    cs, fs = port.adam_state(), free.adam_state()
    cp_, fp_ = port.params(), free.params()
    for net, pick in (("critic", lambda k: k.startswith(("q1.", "q2.", "cse."))), ("actor", lambda k: k.startswith("actor."))):
        dev = max(max(rel_l2(cp_[k], fp_[k]), rel_l2(cs["m"][k], fs["m"][k]), rel_l2(cs["v"][k], fs["v"][k]))
                  for k in cs["m"] if pick(k))
        assert dev >= 100 * REL, f"{name}: the unclipped {net} state is only {dev:.2e} away: the test is vacuous"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: one step, exactly
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PLANS)
def test_clipped_step_is_exact(cuda, name):
    core, spec, care = _clip_handle(name)
    model = new_model(core)
    _steps(core, spec, care, 0, 2)
    model[0].bump(), model[0].bump()
    core.set_grad_clip(**_binding(core))
    for i in range(2):
        before = snapshot(core, 0)
        _steps(core, spec, care, 10 + i, 1)
        act = model[0].bump()
        _check_clipped_step(core, model, before, act, f"{name} step {i}")
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: +inf and never-binding thresholds change nothing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ring", ["uniform", "prioritized"])
@pytest.mark.parametrize("thr", [INF, 1e30], ids=["inf", "1e30"])
@pytest.mark.parametrize("name", ["chained", "vs400_tc", "care_o"])
def test_unbounded_thresholds_leave_every_bit(cuda, name, thr, ring):
    """20 sampled steps (actor every 2nd, targets every 3rd step) of a grad_clip handle == a handle without grad_clip:
    parameters, targets, Adam moments, counters and losses torch.equal."""
    from distributed_sac_b200.core import Replay
    cores, rings = [], []
    for g in (False, True):
        core, spec, care = _clip_handle(name, grad_clip=g)
        core.set_update_intervals(2, 3)
        cap = 4 * spec.batch * max(spec.num_tasks, 1)
        rb = Replay(core, cap, "device", seed=5, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-3) if ring == "prioritized" else None)
        rb.fill_synthetic(cap, seed=6)
        cores.append(core)
        rings.append(rb)
    cores[1].set_grad_clip(critic=thr, actor=thr, ctx=thr)
    for core, rb in zip(cores, rings):
        core.step_sampled(rb, 20)
    for which in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(cores[0].export_arena(which), cores[1].export_arena(which)), (name, which)
    assert cores[0].get_steps() == cores[1].get_steps()
    assert torch.equal(cores[0].read_losses(20).nan_to_num(7.0), cores[1].read_losses(20).nan_to_num(7.0))
    n = cores[1].read_grad_norms(20)[:, 0]
    actor_step = torch.tensor([(i + 1) % 2 == 0 for i in range(20)])
    assert torch.isfinite(n[:, 0]).all() and (n[:, 0] > 0).all()
    assert torch.equal(torch.isfinite(n[:, 1]), actor_step)
    assert torch.isfinite(n[:, 2]).all() if name == "care_o" else torch.isnan(n[:, 2]).all()
    for rb in rings:
        rb.close()
    for core in cores:
        core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: replicas clip independently
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chained", "mtsac_weighted"])
def test_replicas_clip_independently(cuda, name):
    """R = 3 with thresholds (inf, binding, another binding value): each replica == an R = 1 handle holding its state,
    thresholds and inputs, bit for bit, norms included (exact fp32 plans: their sums do not depend on R)."""
    core, spec, care = _clip_handle(name, R=3)
    singles = []
    for r in range(3):
        c1, _, _ = _clip_handle(name)
        c1.set_named(_params(spec, 11 + 7 * r, care, move_targets=True), PARAMS, 0)
        singles.append(c1)
    _steps(core, spec, care, 0, 1)
    thr = [dict(critic=INF, actor=INF, ctx=INF), _binding(core, 1, 0.1), _binding(core, 2, 0.2)]
    for r in range(3):
        core.set_grad_clip(replica=r, **thr[r])
        b, e1, e2 = _inputs(spec, care, 3, 0)
        singles[r].step(*[x[r:r + 1] for x in b], e1[r:r + 1], e2[r:r + 1])
        singles[r].set_grad_clip(**thr[r])
    for i in range(1, 4):
        b, e1, e2 = _inputs(spec, care, 3, i)
        core.step(*b, e1, e2)
        for r in range(3):
            singles[r].step(*[x[r:r + 1] for x in b], e1[r:r + 1], e2[r:r + 1])
    n3, L3 = core.read_grad_norms(4), core.read_losses(4)
    for r, c1 in enumerate(singles):
        for which in (PARAMS, ADAM_M, ADAM_V):
            assert torch.equal(core.export_arena(which, r), c1.export_arena(which)), (name, r, which)
        assert torch.equal(n3[:, r].nan_to_num(7.0), c1.read_grad_norms(4)[:, 0].nan_to_num(7.0)), (name, r)
        assert torch.equal(L3[:, r], c1.read_losses(4)[:, 0]), (name, r)
        assert core.get_steps(r) == c1.get_steps()
        coef = core.debug("clip", r)[:2]
        assert (coef == 1.0).all() if r == 0 else (coef < 1.0).all(), (name, r, coef)
    for c in [core] + singles:
        c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: critic-only steps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chained", "split517_tc", "care_o"])
def test_critic_only_steps_clip_the_critic_alone(cuda, name):
    """Actor every 2nd step: on the critic-only steps the actor norm and coefficient are NaN, the actor side is bit-identical,
    and the critic is clipped exactly; on the actor steps both are."""
    core, spec, care = _clip_handle(name)
    model = new_model(core)
    _steps(core, spec, care, 0, 2)
    model[0].bump(), model[0].bump()
    core.set_grad_clip(**_binding(core))
    core.set_update_intervals(actor_every=2)
    slot, _ = _slots(core)
    for i in range(4):
        before = snapshot(core, 0)
        _steps(core, spec, care, 20 + i, 1)
        act = model[0].bump(2)
        assert act == (i % 2 == 1)
        coef = _check_clipped_step(core, model, before, act, f"{name} step {i}")
        if not act:
            assert math.isnan(coef[1])
            after = snapshot(core, 0)
            for x, y in zip(before, after):
                assert np.array_equal(_bits(x[slot == 1]), _bits(y[slot == 1])), f"{name} step {i}: the actor moved"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6: stream order, determinism
# ---------------------------------------------------------------------------------------------------------------------
def _graph_run(change):
    """16 sampled steps of a SMALL grad_clip learner at R = 2 as two prepared 8-step graph launches; change(core), unless
    None, is enqueued between them.  Returns (norms with NaN read as 7, losses, parameters of replica 1)."""
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(SMALL, replicas=2, grad_clip=True), 0, seed=7)
    rb = Replay(core, capacity=4096, where="device", seed=3)
    rb.fill_synthetic(4096, seed=9)
    core.prepare(rb)
    core.step_sampled(rb, 8)
    if change is not None:
        change(core)
    core.step_sampled(rb, 8)
    out = core.read_grad_norms(16).nan_to_num(7.0), core.read_losses(16), core.export_arena(PARAMS, 1)
    rb.close()
    core.close()
    return out


def test_set_grad_clip_is_stream_ordered(cuda):
    nx, lx, px = _graph_run(None)
    thr = 0.5 * float(nx[8, 1, 0])
    ny, ly, py = _graph_run(lambda core: core.set_grad_clip(critic=thr, replica=1))
    n2, l2, p2 = _graph_run(None)
    assert torch.equal(nx, n2) and torch.equal(lx, l2) and torch.equal(px, p2)        # a run repeats bit for bit
    assert torch.equal(nx[:8], ny[:8]) and torch.equal(lx[:8], ly[:8])   # steps 1-8: unchanged
    assert torch.equal(nx[8, 1, 0], ny[8, 1, 0]) and torch.equal(lx[8, 1, 0], ly[8, 1, 0])   # step 9's critic gradient too
    assert torch.equal(nx[:, 0], ny[:, 0]) and torch.equal(lx[:, 0], ly[:, 0])   # replica 0 was not touched
    assert not torch.equal(nx[9:, 1, 0], ny[9:, 1, 0])                   # step 9's critic update was clipped


@pytest.mark.parametrize("name", ["chained", "split517_tc", "care_o"])
def test_clipped_runs_repeat_bit_for_bit(cuda, name):
    runs = []
    for _ in range(2):
        core, spec, care = _clip_handle(name, R=2)
        _steps(core, spec, care, 0, 1)
        for r in range(2):
            core.set_grad_clip(replica=r, **_binding(core, r, 0.4))
        _steps(core, spec, care, 1, 3)
        runs.append([core.read_grad_norms(4)] + [core.export_arena(w, r) for w in (PARAMS, ADAM_M, ADAM_V) for r in range(2)])
        core.close()
    assert torch.equal(runs[0][0].nan_to_num(7.0), runs[1][0].nan_to_num(7.0))
    assert all(torch.equal(x, y) for x, y in zip(runs[0][1:], runs[1][1:]))


# ---------------------------------------------------------------------------------------------------------------------
# 7: the plans
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chained", "vs400_tc", "care_m", "care_o"])
def test_clip_plans_add_the_norm_launches(cuda, name):
    """The layer-chained plan: weight gradients stored, then norm and Adam per optimizer (4 launches more); the per-layer
    plan: a norm launch in front of every clipped Adam launch."""
    labels, counts = [], []
    for g in (False, True):
        core, _, _ = _clip_handle(name, grad_clip=g)
        counts.append(core.launches_per_step)
        labels.append(plan_labels(core))
        core.close()
    plain, clip = labels
    if name == "chained":
        want = [l.replace("wgrad+adam+polyak{q1,q2}", "wgrad{q1,q2};grad_norm{critic};adam_critic+polyak")
                 .replace("wgrad+adam{actor}", "wgrad{actor};grad_norm{actor};adam_actor") for l in plain]
        assert clip == ";".join(want).split(";"), clip
        assert counts[1] == counts[0] + 4
    else:
        norms = {"grad_norm{critic}": "adam_critic+polyak", "grad_norm{actor}": "adam_actor+alpha",
                 "grad_norm{context_encoder}": "adam_context_encoder"}
        assert [l for l in clip if l not in norms] == plain
        at = [i for i, l in enumerate(clip) if l in norms]
        assert all(clip[i + 1] == norms[clip[i]] for i in at), clip
        assert len(at) == (3 if name == "care_o" else 2) and counts[1] == counts[0] + len(at)


# ---------------------------------------------------------------------------------------------------------------------
# 8: refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_bad_arguments_are_refused(cuda):
    from distributed_sac_b200.core import SacCore
    plain = SacCore(core_config(SMALL), 0, seed=0)
    for call in (lambda: plain.set_grad_clip(critic=1.0), lambda: plain.get_grad_clip(), lambda: plain.read_grad_norms(1)):
        with pytest.raises(RuntimeError, match="error -4"):
            call()
    with pytest.raises(RuntimeError, match="error -1"):
        plain.debug("clip")
    plain.close()
    core = SacCore(core_config(SMALL, replicas=2, grad_clip=True), 0, seed=0)
    assert core.get_grad_clip(0) == core.get_grad_clip(1) == dict(critic=INF, actor=INF, ctx=INF)
    core.set_grad_clip(critic=2.0, actor=3.0, ctx=4.0, replica=1)
    want = [core.get_grad_clip(r) for r in range(2)]
    assert want[1] == dict(critic=2.0, actor=3.0, ctx=4.0)
    for bad in (math.nan, 0.0, -1.0, -INF):
        for k in ("critic", "actor", "ctx"):
            with pytest.raises(RuntimeError, match="error -1"):
                core.set_grad_clip(replica=1, **{k: bad})
    for r in (-1, 2):
        assert core.lib.b200sac_set_grad_clip(core._h, r, 1.0, 1.0, 1.0, None) == -1
    with pytest.raises(RuntimeError, match="error -1"):
        core.read_grad_norms(1)                      # no step yet
    assert [core.get_grad_clip(r) for r in range(2)] == want
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9: the Learner surface
# ---------------------------------------------------------------------------------------------------------------------
def _ll(tmp_path, tag, **kw):
    from distributed_sac_b200.learner import LunarLanderLearner
    p = tmp_path / "ll.json"
    p.write_text(json.dumps(LEARNER_CFGS["LL"]))
    return LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + tag), **kw)


@pytest.mark.parametrize("where", ["host", "device"])
def test_lunarlander_learner_max_grad_norm(cuda, tmp_path, monkeypatch, where):
    monkeypatch.chdir(tmp_path)
    lrn = _ll(tmp_path, "a", replay_where=where, max_grad_norm=1e-4, seed=1)
    try:
        assert lrn.core.cfg.grad_clip and lrn.core.get_grad_clip() == dict(critic=1e-4, actor=1e-4, ctx=1e-4)
        lrn.memory.ring.fill_synthetic(4000, seed=2)
        for _ in range(3):
            out = lrn.update()
            assert len(out) == 2 and all(math.isfinite(x) for x in out)
        L = lrn.update_many(4)
        assert L.shape == (4, 2) and torch.isfinite(L).all()
        n = lrn.core.read_grad_norms(7)[:, 0]
        assert torch.isfinite(n[:, :2]).all() and torch.isnan(n[:, 2]).all()
        assert (n[:, :2] > 1e-4).all() and (lrn.core.debug("clip")[:2] < 1).all()
        lrn.set_max_grad_norm(INF)
        assert lrn.core.get_grad_clip() == dict(critic=INF, actor=INF, ctx=INF)
        lrn.update()
        assert (lrn.core.debug("clip")[:2] == 1).all()
        path = lrn.save_checkpoint(7)
        before = lrn.core.export_arena()
    finally:
        lrn.memory.stop()
    lrn2 = _ll(tmp_path, "b", replay_where=where, max_grad_norm=1.0, seed=5, checkpoint_path=path)
    try:
        assert torch.equal(lrn2.core.export_arena(), before) and lrn2.core.get_steps() == (8, 8, 8)
        assert lrn2.core.get_grad_clip()["critic"] == 1.0          # the thresholds are the learner's, not the checkpoint's
    finally:
        lrn2.memory.stop()
    plain = _ll(tmp_path, "c")
    try:
        assert not plain.core.cfg.grad_clip
        with pytest.raises(ValueError):
            plain.set_max_grad_norm(1.0)
    finally:
        plain.memory.stop()


def test_care_learner_max_grad_norm(cuda, tmp_path, monkeypatch):
    """CARE(O): the context encoder is clipped too."""
    from distributed_sac_b200.learner import CARELearner
    monkeypatch.chdir(tmp_path)
    names_ = [f"task-{i}" for i in range(4)]
    rng = np.random.default_rng(0)
    (tmp_path / "emb.json").write_text(json.dumps({n: rng.standard_normal(64).round(4).tolist() for n in names_}))
    (tmp_path / "names.json").write_text(json.dumps(names_))
    cfg = {"use_modified_care": False, "num_tasks": 4, "device": "cuda", "buffer_size": 4000, "reward_scale": 1,
           "batch_size": 64, "log_alpha": 0, "tau": 0.005, "update_delay": 6, "start_memory_len": 1000,
           "print_period_learner": 10, "gamma": 0.99,
           "actor": {"state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "lr_actor": 3e-4, "actor_hidden_dim": [64, 64]},
           "critic": {"state_dim": 12, "action_dim": 3, "lr_critic": 3e-4, "critic_hidden_dim": [64, 64]},
           "encoder": {"state_dim": 12, "pretrained_embedding_json_path": str(tmp_path / "emb.json"),
                       "task_name_json_path": str(tmp_path / "names.json"), "hidden_dims_contextEnc": [20],
                       "embedding_dim_contextEnc": 16, "output_dim_contextEnc": 16, "RoBERTa_embedding_dim": 64,
                       "lr_contextEnc": 3e-4, "hidden_dims_mixtureEnc": [24], "output_dim_mixtureEnc": 16, "num_encoders": 3,
                       "num_tasks": 4, "state_encoder_tau": 0.05}}
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(cfg))
    lrn = CARELearner(None, names_, str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "c"),
                      replay_where="device", max_grad_norm=1e-6)
    try:
        lrn.memory.ring.fill_synthetic(4000, seed=1)
        for _ in range(2):
            out = lrn.update()
            assert len(out) == 3 and all(math.isfinite(x) for x in out)
        L = lrn.update_many(3)
        assert L.shape == (3, 3) and torch.isfinite(L).all()
        n = lrn.core.read_grad_norms(5)[:, 0]
        assert torch.isfinite(n).all() and (n > 1e-6).all()
        assert (lrn.core.debug("clip") < 1).all()
    finally:
        lrn.memory.stop()
