"""GPU: dropout Q-functions (b200sac_cfg.critic_dropout; include/b200sac.h "Dropout Q-functions").

  1  p = 0 equals a critic_ln handle bit for bit (every arena, the losses), every mask all ones;
  2  the masks ("mQ/mT/mP") equal oracle/philox_ref.py bit for bit for every pass, layer, net and replica;
  3  the step against the DroQ oracle (oracle/droq_port.py) with the CUDA ReLU masks forced, every gradient checked;
  4  z' and h against an fp64 recomputation;
  5  the keep fraction and the independence of the masks;
  6  per-replica rates; 7 stream order of set_critic_dropout and its refusals; 8 the plan;
  9  critic-only steps, gradient clipping, resets, a sampled step from a prioritized, linked device ring and multi-step
     graphs; 10 learners and checkpoints.
"""
import json
import math

import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import droq_port as dq
import philox_ref as pr
import redis_stub
import sac_port as sp
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, sync_core_to_port
from _harness import (LEARNER_CFGS, _eps, _inputs, capture_grads, check_grads, cuda, kink_checked_step, plan_labels,
                      run_checked)

pytestmark = pytest.mark.gpu

SHAPES = {      # the LayerNorm tests' sizes
    "LL": dict(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=64),
    "VS": dict(state_dim=39, act_dim=4, actor_hidden=[96, 96, 96], critic_hidden=[96, 80, 96], batch=128),
    "MS": dict(state_dim=39, act_dim=4, actor_hidden=[96, 96, 96], critic_hidden=[96, 96, 96], batch=160, num_tasks=10,
               weighted_loss=True),
}
PARAMS, ADAM_M, ADAM_V, GRADS = 0, 1, 2, 3
KINDS = {"Q": "cur", "T": "next", "P": "pi"}          # debug buffer -> pass


def _spec(shape):
    return sp.SacSpec(**SHAPES[shape])


def _core(spec, precision=0, replicas=1, seed=0, p=None, dropout=True, **kw):
    from distributed_sac_b200.core import SacCore
    core = SacCore(core_config(spec, replicas=replicas, precision=precision, critic_layer_norm=True,
                               critic_dropout=dropout, **kw), 0, seed=seed)
    if p is not None:
        core.set_critic_dropout(p)
    return core


def _ln_params(spec, seed):
    """Xavier weights, small random biases, LayerNorm weights near 1 and biases near 0, a temperature per task."""
    p = lnp.init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in p:
        if k.endswith(".ln.weight"):
            p[k] = 1.0 + 0.1 * torch.randn(p[k].shape, generator=g)
        elif k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    for k in list(p):
        if "_target." in k:
            p[k] = p[k.replace("_target", "")].clone()
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


def _masks(core, spec, kind, l, replica=0):
    return core.debug(f"m{kind}.{l}", replica).reshape(2, spec.batch, spec.critic_hidden[l])


def _arenas_equal(a, b, ra=0, rb=0, what=""):
    for w in (PARAMS, ADAM_M, ADAM_V, GRADS):
        assert torch.equal(a.export_arena(w, ra), b.export_arena(w, rb)), (what, w)


# ---- 1: p = 0 is the critic_ln step ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("shape", ["LL", "VS", "MS"])
def test_zero_rate_equals_layer_norm_handle(cuda, shape, precision):
    spec = _spec(shape)
    drop, ln = _core(spec, precision, seed=3), _core(spec, precision, seed=3, dropout=False)
    assert drop.get_critic_dropout() == 0.0
    for c in (drop, ln):
        c.set_named(_ln_params(spec, 5), PARAMS)
    for i in range(3):
        b, e1, e2 = _inputs(spec, False, 1, i)
        drop.step(*b, e1, e2)
        ln.step(*b, e1, e2)
    _arenas_equal(drop, ln, what=shape)
    assert torch.equal(drop.read_losses(3), ln.read_losses(3))
    for kind in KINDS:
        for l in range(len(spec.critic_hidden)):
            assert (_masks(drop, spec, kind, l) == 1).all(), (kind, l)
            assert torch.equal(drop.debug(f"z{kind}.{l}"), ln.debug(f"z{kind}.{l}")), (kind, l)
    drop.close()
    ln.close()


# ---- 2: the masks are philox_ref's ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.01, 0.1, 0.5])
def test_masks_equal_philox_reference(cuda, p):
    spec, R, seed = _spec("VS"), 3, 0x5EED_0000_0000_0017
    core = _core(spec, 0, replicas=R, seed=seed, p=p)
    B = spec.batch
    for step in range(1, 4):
        b, e1, e2 = _inputs(spec, False, R, step)
        core.step(*b, e1, e2)
        for r in range(R):
            for kind, tag in KINDS.items():
                for l, H in enumerate(spec.critic_hidden):
                    got = _masks(core, spec, kind, l, r).numpy() == 1
                    for net in (0, 1):
                        want = pr.drop_masks(seed, r, step, tag, l, net, B, H, p)
                        assert np.array_equal(got[net], want), (p, step, r, kind, l, net, int((got[net] != want).sum()))
    core.close()


# ---- 3: parity with the DroQ oracle ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,precision,p", [(s, q, 0.1) for s in ("LL", "VS", "MS") for q in (0, 1)] + [("VS", 1, 0.5)])
def test_step_matches_droq_oracle(cuda, shape, precision, p):
    spec = _spec(shape)
    seed = 11
    core = _core(spec, precision, seed=seed, p=p)
    port = dq.DroqPortLearner(spec, _ln_params(spec, 7), p, seed)
    gen = torch.Generator().manual_seed(3)
    for i in range(3):
        b = sp.synthetic_batch(spec, seed=300 + i)
        e1, e2 = _eps(spec, gen)
        ref = capture_grads(port)
        kink_checked_step(core, port, spec, b, e1, e2, want_intermediates=True)
        check_grads(core, ref, f"{shape} p{precision} rate {p} step {i}")
    flips, worst = run_checked(core, spec, port, 2, 11, f"{shape} p{precision} rate {p}")
    print(f"[critic_dropout] {shape} precision {precision} p {p}: {flips} kink flips, worst row deviation {worst:.2e}")
    core.close()


# ---- 4: z' and h ---------------------------------------------------------------------------------------------------------------
def test_dropped_values_and_normalization(cuda):
    spec, p = _spec("VS"), 0.1
    core = _core(spec, 0, p=p)
    params = _ln_params(spec, 5)
    core.set_named(params, PARAMS)
    b, e1, e2 = _inputs(spec, False, 1, 0)
    core.step(*b, e1, e2)
    B, s = spec.batch, np.float64(pr.scale(p))
    x = torch.cat([b[0][0], b[1][0]], 1).double().numpy()          # pass A's input (s, a)
    for l, H in enumerate(spec.critic_hidden):
        z = core.debug(f"zQ.{l}").reshape(2, B, H).double().numpy()
        h = core.debug(f"hQ.{l}").reshape(2, B, H).double().numpy()
        m = _masks(core, spec, "Q", l).numpy() == 1
        xin = x if l == 0 else core.debug(f"hQ.{l - 1}").reshape(2, B, -1).double().numpy()
        for n in range(2):
            W = params[f"q{n + 1}.{l}.weight"].double().numpy()
            c = params[f"q{n + 1}.{l}.bias"].double().numpy().reshape(-1)
            ref = s * ((xin if l == 0 else xin[n]) @ W.T + c)
            assert (z[n][~m[n]] == 0).all(), (l, n)
            err = np.abs(z[n] - ref)[m[n]] / (np.abs(ref[m[n]]) + np.abs(ref).mean())
            assert err.max() <= 1e-5, (l, n, float(err.max()))
            want, _, _ = lnp.ln_forward(z[n], params[f"q{n + 1}.{l}.ln.weight"].double().numpy().reshape(-1),
                                        params[f"q{n + 1}.{l}.ln.bias"].double().numpy().reshape(-1))
            e2_ = np.abs(h[n] - want) / np.maximum(np.abs(want), 1.0)
            assert e2_.max() <= 1e-6, (l, n, float(e2_.max()))
    core.close()


# ---- 5: distribution ------------------------------------------------------------------------------------------------------------
def test_keep_fraction_and_independence(cuda):
    spec, R, p = _spec("VS"), 3, 0.1
    core = _core(spec, 0, replicas=R, seed=21, p=p)
    seen = {}
    for step in range(2):
        b, e1, e2 = _inputs(spec, False, R, step)
        core.step(*b, e1, e2)
        for r in range(R):
            for kind in KINDS:
                m = _masks(core, spec, kind, 0, r)
                for net in (0, 1):
                    seen[(step, r, kind, net)] = m[net].reshape(-1).double()
    allm = torch.cat(list(seen.values()))
    n = allm.numel()
    keep = float(allm.mean())
    assert abs(keep - (1 - p)) <= 5 * math.sqrt(p * (1 - p) / n), keep
    base = seen[(0, 0, "Q", 0)]
    for other in [(1, 0, "Q", 0), (0, 1, "Q", 0), (0, 0, "T", 0), (0, 0, "P", 0), (0, 0, "Q", 1)]:
        o = seen[other]
        assert not torch.equal(base, o), other
        a_, b_ = base - base.mean(), o - o.mean()
        corr = float((a_ * b_).mean() / (a_.std() * b_.std()))
        assert abs(corr) <= 5 / math.sqrt(base.numel()), (other, corr)
    core.close()


# ---- 6: per-replica rates ----------------------------------------------------------------------------------------------------------
def test_per_replica_rates(cuda):
    spec, R, seed = _spec("LL"), 3, 8
    rates = (0.0, 0.1, 0.5)
    core = _core(spec, 0, replicas=R, seed=seed)
    for r, p in enumerate(rates):
        core.set_critic_dropout(p, replica=r)
    assert [core.get_critic_dropout(r) for r in range(R)] == list(rates)
    ln = _core(spec, 0, replicas=R, seed=seed, dropout=False)
    one = _core(spec, 0, replicas=1, seed=seed, p=0.0)
    ports = {r: dq.DroqPortLearner(spec, _ln_params(spec, 30 + r), rates[r], seed, replica=r) for r in (1, 2)}
    for i in range(3):
        b, e1, e2 = _inputs(spec, False, R, i)
        for r, port in ports.items():
            sync_core_to_port(core, port, r)
        core.step(*b, e1, e2)
        ln.step(*b, e1, e2)
        one.step(*[t[:1] for t in b], e1[:1], e2[:1])
        for r, port in ports.items():
            forced = cuda_relu_masks(core, spec, r)
            with sp.ReluTape(forced) as tape:
                port.update_SAC(*[t[r] for t in b], e1[r], e2[r])
            check_forced(tape, forced, f"replica {r} step {i}: ")
            check_port_state(core, port, r)
    _arenas_equal(core, ln, what="replica 0 vs critic_ln")
    _arenas_equal(core, one, what="replica 0 vs R = 1")
    for c in (core, ln, one):
        c.close()


# ---- 7: stream order and refusals ----------------------------------------------------------------------------------------------
def _prepared_run(mode, change, sync_before_change):
    """8 sampled steps of an LL handle at R = 2 in two graph launches of 4, on a torch side stream ("stream") or the legacy
    stream ("legacy"); change(core) between them (after a synchronisation if sync_before_change).  Returns the arenas."""
    import contextlib
    from distributed_sac_b200.core import Replay
    spec = _spec("LL")
    core = _core(spec, 0, replicas=2, seed=7, p=0.1)
    rb = Replay(core, capacity=4096, where="device", seed=3)
    stream = torch.cuda.Stream() if mode == "stream" else None
    with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
        rb.fill_synthetic(4096, seed=9)
        core.prepare(rb)
        core.step_sampled(rb, 4)
        if sync_before_change:
            torch.cuda.synchronize()
        if change is not None:
            change(core)
        core.step_sampled(rb, 4)
        torch.cuda.synchronize()
        out = [core.export_arena(w, r) for w in (PARAMS, ADAM_M, ADAM_V) for r in range(2)]
    rb.close()
    core.close()
    return out


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("mode", ["stream", "legacy"])
def test_rate_set_between_graph_launches(cuda, mode):
    change = lambda core: core.set_critic_dropout(0.5, replica=1)          # noqa: E731
    ordered = _prepared_run(mode, change, sync_before_change=True)
    assert _same(_prepared_run(mode, change, sync_before_change=False), ordered)
    unchanged = _prepared_run(mode, None, sync_before_change=False)
    assert _same(ordered[0::2], unchanged[0::2])              # replica 0 keeps its rate
    assert not _same(ordered[1::2], unchanged[1::2])          # replica 1 changed from the second launch on

    def refused(core):
        for bad in (float("nan"), -0.1, 1.0, 2.0):
            with pytest.raises(RuntimeError, match="dropout"):
                core.set_critic_dropout(bad, replica=1)
        with pytest.raises(RuntimeError, match="replica"):
            core.set_critic_dropout(0.2, replica=2)
        assert core.get_critic_dropout(1) == 0.1
    assert _same(_prepared_run(mode, refused, sync_before_change=False), unchanged)


def test_plain_handle_gives_state_error(cuda):
    spec = _spec("LL")
    core = _core(spec, 0, dropout=False)
    before = core.export_arena(PARAMS)
    with pytest.raises(RuntimeError, match="critic_dropout"):
        core.set_critic_dropout(0.1)
    with pytest.raises(RuntimeError, match="critic_dropout"):
        core.get_critic_dropout()
    with pytest.raises(RuntimeError):
        core.debug("mQ.0")
    torch.cuda.synchronize()
    assert torch.equal(core.export_arena(PARAMS), before)
    core.close()


# ---- 8: the plan ------------------------------------------------------------------------------------------------------------------
def test_plan_equals_layer_norm_plan(cuda):
    spec = _spec("VS")
    drop, ln = _core(spec, 0, p=0.1), _core(spec, 0, dropout=False)
    assert drop.launches_per_step == ln.launches_per_step
    labels = plan_labels(drop)
    assert labels == plan_labels(ln)
    assert not any(l.startswith("chain") for l in labels)
    drop.close()
    ln.close()


# ---- 9: composition ------------------------------------------------------------------------------------------------------------------
def test_critic_only_step_draws_no_actor_pass_masks(cuda):
    spec, p = _spec("LL"), 0.1
    core = _core(spec, 0, p=p)
    core.set_update_intervals(2, 1)              # the first step (critic count 1) is critic-only
    before = {w: core.get_named(w) for w in (PARAMS, ADAM_M, ADAM_V)}
    b, e1, e2 = _inputs(spec, False, 1, 0)
    core.step(*b, e1, e2)
    after = {w: core.get_named(w) for w in (PARAMS, ADAM_M, ADAM_V)}
    for w in (PARAMS, ADAM_M, ADAM_V):
        for k in before[w]:
            if k.startswith("actor.") or k == "log_alpha":
                assert torch.equal(before[w][k], after[w][k]), (w, k)
    for l in range(len(spec.critic_hidden)):
        assert (_masks(core, spec, "P", l) == 0).all(), l            # never drawn: the zeroed buffer
        assert (_masks(core, spec, "Q", l) == 1).float().mean() > 0.5
    core.step(*b, e1, e2)                          # step 2 runs the actor pass
    for l, H in enumerate(spec.critic_hidden):
        got = _masks(core, spec, "P", l).numpy() == 1
        for net in (0, 1):
            assert np.array_equal(got[net], pr.drop_masks(0, 0, 2, "pi", l, net, spec.batch, H, p))
    core.close()


def test_grad_clip_norm_includes_dropout_grads(cuda):
    spec, p, seed = _spec("VS"), 0.1, 4
    core = _core(spec, 0, seed=seed, p=p, grad_clip=True)
    port = dq.DroqPortLearner(spec, _ln_params(spec, 8), p, seed)
    b = sp.synthetic_batch(spec, seed=21)
    e1, e2 = _eps(spec, torch.Generator().manual_seed(2))
    ref = capture_grads(port)
    kink_checked_step(core, port, spec, b, e1, e2)
    check_grads(core, ref, "grad_clip")
    norms = core.read_grad_norms(1)[0, 0]
    crit = torch.sqrt(sum((v.double() ** 2).sum() for k, v in ref.items() if k.startswith(("q1.", "q2."))))
    assert abs(float(norms[0]) - float(crit)) <= 1e-5 * float(crit), (float(norms[0]), float(crit))
    core.close()


def test_reset_then_steps_match_oracle(cuda):
    spec, p, seed = _spec("VS"), 0.1, 12
    fresh, core = _core(spec, 0, seed=seed, p=p), _core(spec, 0, seed=seed, p=p)
    for i in range(2):
        b, e1, e2 = _inputs(spec, False, 1, i)
        core.step(*b, e1, e2)
    core.reset(seed)
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(core.export_arena(w), fresh.export_arena(w)), w
    assert core.get_critic_dropout() == p                 # a reset keeps the rate
    shapes = lnp.init_params(spec)
    port = dq.DroqPortLearner(spec, {k: v.reshape(shapes[k].shape) for k, v in core.get_named(PARAMS).items()}, p, seed,
                              step=2)
    gen = torch.Generator().manual_seed(5)
    for i in range(2):
        b = sp.synthetic_batch(spec, seed=40 + i)
        e1, e2 = _eps(spec, gen)
        ref = capture_grads(port)
        kink_checked_step(core, port, spec, b, e1, e2)
        check_grads(core, ref, f"after reset, step {i}")
    core.close()
    fresh.close()


def _per_ring(core, spec, n=4096, seed=5):
    from distributed_sac_b200.core import Replay
    rb = Replay(core, n, "device", seed=1, prioritized=dict(alpha=0.6, beta=0.0, eps=1e-6), trajectories=True)
    rows = sp.synthetic_batch(spec, seed=seed, batch=n)
    rb.push(*[x.numpy() for x in rows], stream=np.arange(n) % 16)       # linked, horizon 1
    return rb, rows


def test_sampled_prioritized_linked_step_equals_step(cuda):
    """beta = 0 (every weight 1) and horizon 1: a sampled step equals b200sac_step on the rows it drew, bit for bit (same
    seed, so the same noise and the same masks); a 3-step graph equals three 1-step graphs."""
    spec, p = _spec("LL"), 0.1
    sampled, direct = _core(spec, 0, seed=2, p=p), _core(spec, 0, seed=2, p=p)
    rb, rows = _per_ring(sampled, spec)
    for _ in range(3):
        sampled.step_sampled(rb, 1)
        idx = sampled.debug("idx").long()
        assert torch.equal(sampled.debug("isw"), torch.ones(spec.batch))
        direct.step(*[x[idx].unsqueeze(0) for x in rows])
        assert torch.equal(sampled.debug("mQ.0"), direct.debug("mQ.0"))
    _arenas_equal(sampled, direct, what="sampled vs step")
    assert torch.equal(sampled.read_losses(3), direct.read_losses(3))
    # multi-step graphs: new masks every step
    one, many = _core(spec, 0, seed=6, p=p), _core(spec, 0, seed=6, p=p)
    r1, _ = _per_ring(one, spec)
    r3, _ = _per_ring(many, spec)
    for _ in range(3):
        one.step_sampled(r1, 1)
    many.step_sampled(r3, 3)
    _arenas_equal(one, many, what="3-step graph")
    for l, H in enumerate(spec.critic_hidden):
        got = _masks(many, spec, "Q", l).numpy() == 1
        assert np.array_equal(got[0], pr.drop_masks(6, 0, 3, "cur", l, 0, spec.batch, H, p))
    for x in (rb, r1, r3, sampled, direct, one, many):
        x.close()


# ---- 10: learners ----------------------------------------------------------------------------------------------------------------
MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


@pytest.mark.parametrize("family", ["LL", "VS", "MS"])
def test_learner_updates_and_checkpoints(cuda, tmp_path, monkeypatch, family):
    from distributed_sac_b200 import learner as L
    monkeypatch.chdir(tmp_path)                     # the checkpoint goes under saved_models/ of the working directory
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(MS_CFG if family == "MS" else LEARNER_CFGS[family]))
    kw = dict(write_mode=False, replay_where="device", critic_layer_norm=True, critic_dropout=0.01)

    def make(tag, **extra):
        srv = redis_stub.StrictRedis(host=str(tmp_path) + tag)
        if family == "MS":
            return L.MTSACLearner(None, ["t0", "t1", "t2"], str(p), server=srv, **kw, **extra)
        return (L.LunarLanderLearner if family == "LL" else L.VSACLearner)(str(p), server=srv, **kw, **extra)
    lr = make("a")
    assert lr.core.get_critic_dropout() == 0.01
    lr.memory.ring.fill_synthetic(4096, seed=1)
    for _ in range(3):
        out = lr.update()
        assert all(np.isfinite(x) for x in out[:2])
    path = lr.save_checkpoint(1)
    lr2 = make("b", checkpoint_path=path)
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(lr.core.export_arena(w), lr2.core.export_arena(w)), w
    assert tuple(lr.core.get_steps())[:3] == tuple(lr2.core.get_steps())[:3]
    assert lr2.core.get_critic_dropout() == 0.01
    lr2.core.set_critic_dropout(0.3)
    lr2.load_checkpoint(path)                       # loading applies the learner's rate again
    assert lr2.core.get_critic_dropout() == 0.01
    if family == "MS":
        sd = lr._module_state_dict("q1")
        assert "Q_function_1.2.weight" in sd and "Q_function_1.4.weight" in sd       # Linear 0, LayerNorm 0, Linear 1
    lr.memory.stop()
    lr2.memory.stop()
