"""GPU: layer-normalized critics (b200sac_cfg.critic_ln; include/b200sac.h "Layer-normalized critics").

  1  the step against the LayerNorm autograd oracle (oracle/critic_ln_port.py) with the CUDA ReLU masks forced, at the
     LL, VS and MS shapes of the envelope tests, precision 0 and 1, every gradient (dg, dc included) checked;
  2  the normalization launches alone: h == relu(LN(z)) in fp64 numpy over the device's own z, g and c;
  3  create: Linear tensors bit-equal to the plain handle's, g = 1, c = 0, targets = locals;
  4  determinism: two handles bit for bit; replica r of R = 3 equals an R = 1 handle bit for bit;
  5  the plan: never the layer-chained one, 5 * Lc launches more than the per-layer plan, labelled;
  6  critic-only steps; 7 gradient clipping; 8 resets; 9 Polyak; 10 ReDo refused; 11 learners; 12 a sampled step from a
     prioritized, linked device ring.
"""
import json

import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import redis_stub
from distributed_sac_b200 import names
import sac_port as sp
from _golden import core_config
from _harness import (LEARNER_CFGS, _eps, _inputs, capture_grads, check_grads, cuda, kink_checked_step, plan_labels,
                      run_checked)

pytestmark = pytest.mark.gpu

SHAPES = {      # the envelope tests' sizes
    "LL": dict(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=64),
    "VS": dict(state_dim=39, act_dim=4, actor_hidden=[96, 96, 96], critic_hidden=[96, 80, 96], batch=128),
    "MS": dict(state_dim=39, act_dim=4, actor_hidden=[96, 96, 96], critic_hidden=[96, 96, 96], batch=160, num_tasks=10,
               weighted_loss=True),
}
PARAMS, ADAM_M, ADAM_V, GRADS = 0, 1, 2, 3


def _spec(shape):
    return sp.SacSpec(**SHAPES[shape])


def _core(spec, precision=0, replicas=1, seed=0, **kw):
    from distributed_sac_b200.core import SacCore
    return SacCore(core_config(spec, replicas=replicas, precision=precision, critic_layer_norm=True, **kw), 0, seed=seed)


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


def _batch(spec, R, i):
    b, e1, e2 = _inputs(spec, False, R, i)
    return b, e1, e2


# ---- 1: parity --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("shape", ["LL", "VS", "MS"])
def test_step_matches_layer_norm_oracle(cuda, shape, precision):
    spec = _spec(shape)
    core = _core(spec, precision)
    port = lnp.LnPortLearner(spec, _ln_params(spec, 7))
    gen = torch.Generator().manual_seed(3)
    for i in range(3):
        b = sp.synthetic_batch(spec, seed=300 + i)
        e1, e2 = _eps(spec, gen)
        ref = capture_grads(port)
        with lnp._layer_norm_mlp():
            kink_checked_step(core, port, spec, b, e1, e2, want_intermediates=True)
        check_grads(core, ref, f"{shape} p{precision} step {i}")
    with lnp._layer_norm_mlp():
        flips, worst = run_checked(core, spec, port, 2, 11, f"{shape} p{precision}")
    print(f"[critic_ln] {shape} precision {precision}: {flips} kink flips, worst row deviation {worst:.2e}")
    core.close()


# ---- 2: the normalization launches alone --------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
def test_normalization_matches_fp64(cuda, precision):
    spec = _spec("VS")
    core = _core(spec, precision)
    core.set_named(_ln_params(spec, 5), PARAMS)
    b, e1, e2 = _batch(spec, 1, 0)
    core.step(*b, e1, e2)
    named = core.get_named(PARAMS)
    B = spec.batch
    # hQ / hT were normalized with the parameters before the step's updates; hP with the updated critics
    before = _ln_params(spec, 5)
    for kind, src in (("Q", before), ("T", before), ("P", named)):
        net_of = (lambda n: f"q{n + 1}_target") if kind == "T" else (lambda n: f"q{n + 1}")
        for l, H in enumerate(spec.critic_hidden):
            z = core.debug(f"z{kind}.{l}").reshape(2, B, H).double().numpy()
            h = core.debug(f"h{kind}.{l}").reshape(2, B, H).double().numpy()
            for n in range(2):
                ref, _, _ = lnp.ln_forward(z[n], src[f"{net_of(n)}.{l}.ln.weight"].reshape(-1).double().numpy(),
                                           src[f"{net_of(n)}.{l}.ln.bias"].reshape(-1).double().numpy())
                err = np.abs(h[n] - ref) / np.maximum(np.abs(ref), 1.0)
                assert err.max() <= 1e-6, (kind, l, n, float(err.max()))
    core.close()


# ---- 3: create -----------------------------------------------------------------------------------------------------------
def test_create_linear_tensors_bit_equal_plain_handle(cuda):
    from distributed_sac_b200.core import SacCore
    spec = _spec("VS")
    ln = _core(spec, seed=9)
    plain = SacCore(core_config(spec, precision=0), 0, seed=9)
    a, p = ln.get_named(PARAMS), plain.get_named(PARAMS)
    for k, v in p.items():
        assert torch.equal(a[k], v), k
    for k, v in a.items():
        if ".ln.weight" in k:
            assert torch.equal(v, torch.ones_like(v)), k
        elif ".ln.bias" in k:
            assert torch.equal(v, torch.zeros_like(v)), k
        if "_target." in k:
            assert torch.equal(v, a[k.replace("_target", "")]), k
    ln.close()
    plain.close()


# ---- 4: determinism ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1])
def test_runs_repeat_and_replicas_are_independent(cuda, precision):
    spec = _spec("LL")
    R = 3
    cores = [_core(spec, precision, replicas=R, seed=4), _core(spec, precision, replicas=R, seed=4),
             _core(spec, precision, replicas=1, seed=4)]
    for i in range(4):
        b, e1, e2 = _batch(spec, R, i)
        cores[0].step(*b, e1, e2)
        cores[1].step(*b, e1, e2)
        cores[2].step(*[t[:1] for t in b], e1[:1], e2[:1])
    for which in (PARAMS, ADAM_M, ADAM_V, GRADS):
        for r in range(R):
            assert torch.equal(cores[0].export_arena(which, r), cores[1].export_arena(which, r)), (which, r)
        assert torch.equal(cores[0].export_arena(which, 0), cores[2].export_arena(which, 0)), which
    for c in cores:
        c.close()


# ---- 5: the plan ------------------------------------------------------------------------------------------------------------
def test_plan_is_per_layer_with_five_launches_per_hidden_layer(cuda):
    from distributed_sac_b200.core import SacCore
    spec = _spec("LL")
    Lc = len(spec.critic_hidden)
    ln = _core(spec, 0)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("B200SAC_FUSE", "0")
        plain = SacCore(core_config(spec, precision=0), 0, seed=0)
    assert ln.launches_per_step == plain.launches_per_step + 5 * Lc
    labels = plan_labels(ln)
    assert not any(l.startswith("chain") for l in labels)
    want = [f"ln_fwd{{{p} {l}}}" for p in ("critic", "target", "actor pass") for l in range(Lc)]
    want += [f"ln_bwd{{{p} {l}}}" for p in ("critic", "actor pass") for l in range(Lc)]
    for w in want:
        assert labels.count(w) == 1, (w, labels)
    ln.close()
    plain.close()


# ---- 6: critic-only steps ---------------------------------------------------------------------------------------------
def test_critic_only_step_leaves_actor_and_matches_oracle_critics(cuda):
    from _golden import check_forced, cuda_relu_masks, rel_l2, sync_core_to_port
    spec = _spec("LL")
    core = _core(spec, 0)
    core.set_update_intervals(2, 1)              # the first step (critic count 1) is critic-only
    port = lnp.LnPortLearner(spec, _ln_params(spec, 3))
    sync_core_to_port(core, port)
    before = {w: core.get_named(w) for w in (PARAMS, ADAM_M, ADAM_V)}
    b = sp.synthetic_batch(spec, seed=5)
    e1, e2 = _eps(spec, torch.Generator().manual_seed(1))
    core.step(*b, e1, e2)
    after = {w: core.get_named(w) for w in (PARAMS, ADAM_M, ADAM_V)}
    for w in (PARAMS, ADAM_M, ADAM_V):
        for k in before[w]:
            if k.startswith("actor.") or k == "log_alpha":
                assert torch.equal(before[w][k], after[w][k]), (w, k)
    assert tuple(core.get_steps())[:3] == (1, 0, 0)
    # the critic half of the oracle's step, with the CUDA masks of the passes the critic update ran
    forced = {k: v for k, v in cuda_relu_masks(core, spec).items() if ":pi:" not in k and k not in ("route:pi", "tanh:cur")}
    with lnp._layer_norm_mlp(), sp.ReluTape(forced) as tape:
        port.update_SAC(*b, e1, e2)
    check_forced(tape, forced)
    ref = port.params()
    for k, v in ref.items():
        if k.startswith("q"):
            assert rel_l2(after[PARAMS][k], v) <= 1e-4, k
    core.close()


# ---- 7: gradient clipping --------------------------------------------------------------------------------------------------
def test_grad_clip_norm_includes_layer_norm_grads(cuda):
    spec = _spec("VS")
    core = _core(spec, 0, grad_clip=True)
    port = lnp.LnPortLearner(spec, _ln_params(spec, 8))
    b = sp.synthetic_batch(spec, seed=21)
    e1, e2 = _eps(spec, torch.Generator().manual_seed(2))
    ref = capture_grads(port)
    with lnp._layer_norm_mlp():
        kink_checked_step(core, port, spec, b, e1, e2)
    check_grads(core, ref, "grad_clip")
    norms = core.read_grad_norms(1)[0, 0]
    crit = torch.sqrt(sum((v.double() ** 2).sum() for k, v in ref.items() if k.startswith(("q1.", "q2."))))
    assert abs(float(norms[0]) - float(crit)) <= 1e-5 * float(crit), (float(norms[0]), float(crit))
    core.close()


# ---- 8: resets ---------------------------------------------------------------------------------------------------------------
def test_reset_layer_norm_tensors(cuda):
    spec = _spec("VS")
    fresh = _core(spec, 0, seed=12)
    core = _core(spec, 0, seed=12)
    for i in range(2):
        b, e1, e2 = _batch(spec, 1, i)
        core.step(*b, e1, e2)
    core.reset(12)
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(core.export_arena(w), fresh.export_arena(w)), w
    # depth d touches the LayerNorm of the Linear layers at depth <= d (counted from the head)
    for i in range(2):
        b, e1, e2 = _batch(spec, 1, i + 5)
        core.step(*b, e1, e2)
    Lc = len(spec.critic_hidden)
    for d in range(1, Lc + 2):
        before = core.get_named(PARAMS)
        core.reset(99, critic=d, shrink=0.5)
        after = core.get_named(PARAMS)
        for k in before:
            if ".ln." not in k:
                continue
            layer = int(k.split(".")[1])
            touched = Lc + 1 - layer <= d
            changed = not torch.equal(before[k], after[k])
            if touched and k.endswith("ln.weight"):
                ref = (0.5 * before[k].double() + 0.5 * 1.0).float()
                assert torch.equal(after[k], ref), k
            if not touched:
                assert not changed, (d, k)
    core.close()
    fresh.close()


# ---- 9: Polyak ---------------------------------------------------------------------------------------------------------------
def test_soft_update_moves_layer_norm_targets(cuda):
    spec = _spec("LL")
    core = _core(spec, 0)
    p = _ln_params(spec, 2)
    for k in list(p):
        if "_target." in k:
            p[k] = p[k] + 0.1
    core.set_named(p, PARAMS)
    tau = 0.25
    core.soft_update(tau)
    got = core.get_named(PARAMS)
    for k in p:
        if "_target." in k and ".ln." in k:
            loc = p[k.replace("_target", "")]
            ref = (tau * loc + (1.0 - tau) * p[k]).float()
            assert torch.allclose(got[k].reshape(-1), ref, rtol=0, atol=1e-6), k
    core.set_named(p, PARAMS)
    core.soft_update(tau, critic=2)
    got = core.get_named(PARAMS)
    for k in p:
        if k.startswith("q1_target.") and ".ln." in k:
            assert torch.equal(got[k].reshape(-1), p[k]), k
        if k.startswith("q2_target.") and ".ln." in k:
            assert not torch.equal(got[k].reshape(-1), p[k]), k
    core.close()


# ---- 10: ReDo is refused ---------------------------------------------------------------------------------------------------
def test_redo_refused(cuda):
    from distributed_sac_b200 import _lib
    spec = _spec("LL")
    core = _core(spec, 0)
    before = core.export_arena(PARAMS)
    s = torch.randn(8, spec.obs_dim)
    a = torch.rand(8, spec.act_dim)
    with pytest.raises(RuntimeError, match="critic_ln"):
        core.redo(1, s, a, actor=0.0, critic=0.0)
    torch.cuda.synchronize()
    assert torch.equal(core.export_arena(PARAMS), before)
    core.close()


# ---- 11: learners ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["device", "host"])
def test_learner_updates_and_checkpoints(cuda, tmp_path, where):
    from distributed_sac_b200 import learner as L
    p = tmp_path / "LL.json"
    p.write_text(json.dumps(LEARNER_CFGS["LL"]))
    kw = dict(write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + where), replay_where=where,
              critic_layer_norm=True)
    lr = L.LunarLanderLearner(str(p), **kw)
    B = lr.batch_size
    rng = np.random.default_rng(0)
    n = 4 * B
    lr.memory.add_many(rng.standard_normal((n, 8)).astype(np.float32), rng.uniform(-1, 1, (n, 2)).astype(np.float32),
                       rng.standard_normal(n).astype(np.float32), rng.standard_normal((n, 8)).astype(np.float32),
                       np.zeros(n, np.float32))
    for _ in range(3):
        out = lr.update()
        assert all(np.isfinite(x) for x in out[:2])
    sd = lr.local_critic_1.state_dict()
    assert "layer_norms.0.weight" in sd and "layer_norms.1.bias" in sd
    assert set(lr.get_parameters()) == {"actor"}
    assert set(lr.get_parameters()["actor"]) == set(names.actor_key_map("LL", 3))
    path = lr.save_checkpoint(1)
    lr2 = L.LunarLanderLearner(str(p), **dict(kw, server=redis_stub.StrictRedis(host=str(tmp_path) + where + "2")),
                               checkpoint_path=path)
    for w in (PARAMS, ADAM_M, ADAM_V):
        assert torch.equal(lr.core.export_arena(w), lr2.core.export_arena(w)), w
    assert tuple(lr.core.get_steps())[:3] == tuple(lr2.core.get_steps())[:3]
    # the state_dict keys load into the torch module with LayerNorm (test_critic_ln_host.py)
    from test_critic_ln_host import LnCritic
    m = LnCritic(8 + 2, [256, 256])
    m.load_state_dict({k: v.reshape(m.state_dict()[k].shape) for k, v in sd.items()}, strict=True)
    lr.memory.stop()
    lr2.memory.stop()


# ---- 12: a sampled step from a prioritized, linked device ring -----------------------------------------------------------
def test_sampled_prioritized_linked_step(cuda):
    from distributed_sac_b200.core import Replay
    spec = _spec("LL")
    core = _core(spec, 0)
    ring = Replay(core, 8 * spec.batch, "device", seed=3, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6), trajectories=True)
    ring.fill_synthetic(8 * spec.batch, seed=4)
    core.step_sampled(ring, 2)
    torch.cuda.synchronize()
    L = core.read_losses(2)
    assert torch.isfinite(L[:, 0, :2]).all(), L
    for l in range(len(spec.critic_hidden)):
        assert torch.isfinite(core.debug(f"zQ.{l}")).all()
    ring.close()
    core.close()
