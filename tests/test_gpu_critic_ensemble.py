"""GPU: critic ensembles (b200sac_cfg.critic_ensemble; include/b200sac.h "Critic ensembles").

  1  E = 2, m = 2, MIN equals the twin per-layer plan bit for bit (every arena and the losses), with LayerNorm, DroQ,
     gradient clipping, update intervals and three replicas;
  2  create: actor, q1, q2, their targets and log_alpha equal a twin handle of the same seed;
  3  the step against the autograd oracle (oracle/redq_port.py) over ten steps at exact fp32, and "tsub" against
     oracle/redq_ref.py;
  4  per-replica settings and their stream order; 5 critic-only steps, resets, copy_replica, soft_update_critic(k),
     critic_values; 6 the plan and every refusal.
"""
import contextlib

import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import redq_port as rq
import redq_ref
import sac_port as sp
from _golden import REL, core_config, rel_l2
import redis_stub
from _harness import LEARNER_CFGS, _inputs, cuda, plan_labels
from distributed_sac_b200 import _lib

pytestmark = pytest.mark.gpu

SEED = 77
SMALL = sp.ll_spec(batch=128, actor_hidden=[64, 64], critic_hidden=[64, 64])
ARENAS = (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V)


def _new(spec, unfused=True, replicas=1, precision=0, **kw):
    from distributed_sac_b200.core import SacCore
    with pytest.MonkeyPatch.context() as mp:
        if unfused:
            mp.setenv("B200SAC_FUSE", "0")
        return SacCore(core_config(spec, replicas=replicas, precision=precision, **kw), 0, seed=SEED)


def _run(core, spec, R, n, setup=None):
    for i in range(n):
        (s, a, r, s2, d), e1, e2 = _inputs(spec, False, R, i)
        core.step(s, a, r, s2, d, e1, e2)
    torch.cuda.synchronize()
    return core.read_losses(n)


def _bits(t):
    return t.numpy().view(np.uint32)


TWIN_CASES = {
    "LL": (sp.ll_spec(), 0, {}),
    "VS-fp32": (sp.vs_spec(batch=256), 0, {}),
    "VS-tf32": (sp.vs_spec(batch=256), 1, {}),
    "MS": (sp.ms_spec(), 1, {}),
    "LL-ln": (sp.ll_spec(), 0, dict(critic_layer_norm=True)),
    "LL-droq": (sp.ll_spec(), 0, dict(critic_layer_norm=True, critic_dropout=True)),
    "VS-ln-clip": (sp.vs_spec(batch=256), 1, dict(critic_layer_norm=True, grad_clip=True)),
}


@pytest.mark.parametrize("case", list(TWIN_CASES))
def test_twin_identity(cuda, case):
    spec, prec, kw = TWIN_CASES[case]
    R = 3
    twin = _new(spec, replicas=R, precision=prec, **kw)
    ens = _new(spec, replicas=R, precision=prec, critic_ensemble=2, **kw)
    ens.set_ensemble(2, "min")
    for c in (twin, ens):
        if kw.get("critic_dropout"):
            c.set_critic_dropout(0.1)
        if kw.get("grad_clip"):
            c.set_grad_clip(critic=1.0, actor=1.0)
        c.set_update_intervals(2, 2, replica=1)
    assert twin.launches_per_step == ens.launches_per_step
    lt, le = _run(twin, spec, R, 4), _run(ens, spec, R, 4)
    assert np.array_equal(_bits(lt), _bits(le))
    for r in range(R):
        for w in ARENAS:
            assert np.array_equal(_bits(twin.export_arena(w, r)), _bits(ens.export_arena(w, r))), (r, w)
        for name in ("y", "q1", "q2", "qmin", "dq_pi", "d_action", "hQ.0", "hP.1", "hT.1"):
            assert np.array_equal(_bits(twin.debug(name, r)), _bits(ens.debug(name, r))), name
        assert ens.debug("tsub", r).tolist() == [1.0, 1.0]
    twin.close(); ens.close()


@pytest.mark.parametrize("E", [3, 10])
def test_create_keeps_the_twin_prefix(cuda, E):
    twin, ens = _new(sp.ll_spec()), _new(sp.ll_spec(), critic_ensemble=E)
    a, b = twin.get_named(), ens.get_named()
    for name, t in a.items():
        assert torch.equal(t, b[name]), name
    for k in range(3, E + 1):                 # the extra critics are drawn, distinct, with their targets equal
        assert not torch.equal(b[f"q{k}.0.weight"], b["q1.0.weight"])
        assert torch.equal(b[f"q{k}.0.weight"], b[f"q{k}_target.0.weight"])
    assert ens.get_ensemble(0) == (2, "mean")
    twin.close(); ens.close()


def _port(core, spec, E, m, actor, r, steps):
    """The oracle at replica r's current device state: parameters, targets, Adam moments and step counts."""
    P, M, V = (core.get_named(w, r) for w in (_lib.PARAMS, _lib.ADAM_M, _lib.ADAM_V))
    names = list(P)
    shape = {k: (-1,) if ".ln." in k else sp.param_shape(spec, k) for k in names}
    port = rq.RedqPortLearner(spec, {k: P[k].reshape(shape[k]) for k in names}, E, m, actor, seed=SEED, replica=r,
                              step=steps)
    trainable = [k for k in names if "_target" not in k]
    port.load_adam({"m": {k: M[k].reshape(shape[k]) for k in trainable}, "v": {k: V[k].reshape(shape[k]) for k in trainable},
                    "step": (steps, steps, steps)})
    return port


def _check_close(core, port, r, what):
    """Every gradient the step computed, every parameter and target tensor within the repository's bar (relative L2 1e-4;
    plus 1e-7 per element for the parameters: an fp32 ulp at the 1e-3 scale of freshly trained biases), log_alpha to
    1e-6."""
    dev, grads = core.get_named(_lib.PARAMS, r), core.get_named(_lib.GRADS, r)
    for k, v in port.params().items():
        if k in port.grads and k != "log_alpha":      # (the temperature step keeps no gradient in the arena)
            g, ref = grads[k].reshape(v.shape).double(), port.grads[k].double()
            assert rel_l2(g, ref) <= REL, f"{what}: gradient of {k} off by {rel_l2(g, ref):.1e}"
        d = dev[k].reshape(v.shape).double()
        v = v.double()
        if k == "log_alpha":
            assert (d - v).abs().max().item() <= 1e-6, what
        else:
            err = (d - v).norm().item()
            assert err <= REL * v.norm().item() + 1e-7 * v.numel() ** 0.5, f"{what}: {k} off by {err:.1e}"


# Exact fp32 only: at precision 1 the 3xTF32 GEMMs move a pre-activation across a ReLU kink now and then, and the oracle
# then differs by that unit's whole contribution (the twin tests force the device's ReLU masks into the oracle for this).
# The ensemble kernels are the same at both precisions, and test_twin_identity pins precision 1 to the twin plan.
SPECS = {"LL": SMALL, "VS": sp.vs_spec(batch=128, actor_hidden=[64, 64], critic_hidden=[64, 48]),
         "MS": sp.ms_spec(batch=160, actor_hidden=[64, 64], critic_hidden=[64, 64])}


def _masks(core, spec, E, r):
    """{(k, tag, layer): bool [B][H]}: the keep masks of the replica's last step."""
    out = {}
    for letter, tag in (("Q", "cur"), ("T", "next"), ("P", "pi")):
        for l, H in enumerate(spec.critic_hidden):
            m = core.debug(f"m{letter}.{l}", r).reshape(E, spec.batch, H) == 1
            out.update({(k, tag, l): m[k] for k in range(E)})
    return out


def _parity(spec_name, E, m, actor, ln=False, p=None):
    """Ten steps, each checked against the oracle started from the device's state before it (the first step fills
    Adam's moments, where a zero gradient's sign is arbitrary); the subset of every step and replica against redq_ref.
    DroQ: the oracle takes the device's masks of the step."""
    spec = SPECS[spec_name]
    R = 2
    core = _new(spec, replicas=R, critic_ensemble=E, critic_layer_norm=ln, critic_dropout=p is not None)
    core.set_ensemble(m, actor)
    if p is not None:
        core.set_critic_dropout(p)
    for i in range(10):
        (s, a, rw, s2, d), e1, e2 = _inputs(spec, False, R, i)
        ports = [_port(core, spec, E, m, actor, r, i) for r in range(R)] if i > 0 else None
        core.step(s, a, rw, s2, d, e1, e2)
        torch.cuda.synchronize()
        for r in range(R):
            tsub = core.debug("tsub", r).numpy().astype(bool)
            assert np.array_equal(tsub, redq_ref.subset(SEED, r, i + 1, E, m)), (i, r)
            if ports:
                ctx = rq.ensemble_dropout(_masks(core, spec, E, r), p) if p is not None else (
                    lnp._layer_norm_mlp() if ln else contextlib.nullcontext())
                with ctx:
                    ports[r].update_SAC(s[r], a[r], rw[r], s2[r], d[r], e1[r], e2[r])
                _check_close(core, ports[r], r, f"step {i + 1}, replica {r}")
    if p is not None:
        keep = torch.stack([v.float().mean() for v in _masks(core, spec, E, 0).values()]).mean().item()
        assert 0.97 < keep < 1.0
    core.close()


# Exact fp32 only: at precision 1 the 3xTF32 GEMMs move a pre-activation across a ReLU kink now and then, and the oracle
# then differs by that unit's whole contribution (the twin tests force the device's ReLU masks into the oracle for this).
# The ensemble kernels are the same at both precisions, and test_twin_identity pins precision 1 to the twin plan.
@pytest.mark.parametrize("spec_name", ["LL", "VS", "MS"])
@pytest.mark.parametrize("E,m,actor", [(3, 1, "mean"), (3, 3, "min"), (10, 2, "mean"), (10, 2, "min"), (10, 10, "mean"),
                                       (10, 1, "min")])
def test_oracle_parity(cuda, spec_name, E, m, actor):
    _parity(spec_name, E, m, actor)


@pytest.mark.parametrize("spec_name", ["LL", "VS"])
@pytest.mark.parametrize("actor", ["mean", "min"])
def test_oracle_parity_rlpd_layer_norm(cuda, spec_name, actor):
    _parity(spec_name, 10, 2, actor, ln=True)


@pytest.mark.parametrize("spec_name", ["LL", "VS"])
def test_oracle_parity_droq_with_the_device_masks(cuda, spec_name):
    _parity(spec_name, 10, 2, "mean", ln=True, p=0.01)


def test_critic_values_of_a_layer_norm_ensemble(cuda):
    spec, E = SMALL, 10
    core = _new(spec, critic_ensemble=E, critic_layer_norm=True, critic_dropout=True)
    core.set_critic_dropout(0.5)                 # eval mode: no dropout whatever the rate
    _run(core, spec, 1, 3)
    g = torch.Generator().manual_seed(4)
    obs, act = torch.randn(200, spec.obs_dim, generator=g), torch.randn(200, spec.act_dim, generator=g)
    named = core.get_named()
    for target in (False, True):
        q = core.critic_values(obs, act, target=target).cpu()
        for k in range(E):
            net = f"q{k + 1}" + ("_target" if target else "")
            ref = lnp.mlp({n: v.reshape(-1) if ".ln." in n else v for n, v in named.items()}, net,
                          torch.cat([obs, act], -1)).squeeze(-1)
            assert torch.allclose(q[k], ref, rtol=1e-4, atol=1e-5), (target, k)
    core.close()


def _push_rows(rb, spec, n, seed, stream=None, done_every=None):
    """n rows pushed into replica 0 of rb; returns them as [n][w] tensors (slot i = row i)."""
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(n, spec.obs_dim, generator=g)
    a = torch.rand(n, spec.act_dim, generator=g) * 2 - 1
    r = torch.randn(n, 1, generator=g)
    s2 = torch.randn(n, spec.obs_dim, generator=g)
    d = (torch.rand(n, 1, generator=g) < 0.1).float()
    if done_every is not None:                   # consecutive rows chained: s2 of row i is s of row i + 1, episodes end with d = 1
        s2[:-1] = s[1:]
        d = ((torch.arange(n) % done_every) == done_every - 1).float().reshape(n, 1)
    rb.push(*[x.numpy() for x in (s, a, r, s2, d)], stream=stream)
    return s, a, r, s2, d


def test_prior_ring_steps_equal_b200sac_step(cuda):
    from distributed_sac_b200.core import Replay
    spec, E = SMALL, 10
    sampled, direct = _new(spec, critic_ensemble=E), _new(spec, critic_ensemble=E)
    on, pri = Replay(sampled, 8 * spec.batch, "device", seed=1), Replay(sampled, 8 * spec.batch, "device", seed=2)
    rows_on, rows_pr = _push_rows(on, spec, 8 * spec.batch, 3), _push_rows(pri, spec, 8 * spec.batch, 4)
    on.attach_prior(pri)
    on.set_prior_rows(spec.batch // 2)
    for _ in range(4):
        sampled.step_sampled(on, 1)
        idx = sampled.debug("idx").long()           # online k as k, prior k as -1 - k
        is_p = idx < 0
        assert is_p.sum().item() == spec.batch // 2
        rows = [torch.where(is_p.unsqueeze(1), xp[(-1 - idx).clamp(min=0)], xo[idx.clamp(min=0)])
                for xo, xp in zip(rows_on, rows_pr)]
        direct.step(*[x.unsqueeze(0) for x in rows])
    torch.cuda.synchronize()
    for w in ARENAS:
        assert torch.equal(sampled.export_arena(w), direct.export_arena(w)), w
    assert torch.equal(sampled.read_losses(4), direct.read_losses(4))
    on.close(); pri.close(); sampled.close(); direct.close()


def test_nstep_ring_steps_equal_b200sac_step(cuda):
    """Horizon 3 on episodes that end with d = 1: every row folds 3 rewards (disc = gamma^3) or stops at d = 1, where the
    discount does not enter.  b200sac_step with gamma = gamma^3 on the folded rows takes the same steps."""
    from distributed_sac_b200.core import Replay
    spec, E = SMALL, 10
    sampled, direct = _new(spec, critic_ensemble=E), _new(spec, critic_ensemble=E)
    n = 8 * spec.batch
    rb = Replay(sampled, n, "device", seed=1, trajectories=True)
    _push_rows(rb, spec, n, 5, stream=np.zeros(n, np.int64), done_every=16)      # (n % 16 == 0: no episode left open)
    rb.set_nstep(3)
    for i in range(4):
        sampled.step_sampled(rb, 1)
        torch.cuda.synchronize()
        idx = sampled.debug("idx").numpy().astype(np.int64)
        s, a, R, s2, d, disc, m = rb.fold(idx)
        assert np.array_equal(sampled.debug("r").numpy(), R.reshape(-1))
        full = d.reshape(-1) == 0
        assert full.any() and len(set(disc.reshape(-1)[full].tolist())) == 1
        if i == 0:
            direct.set_hparams(0, gamma=float(disc.reshape(-1)[full][0]))
        direct.step(*[torch.as_tensor(x).reshape(1, spec.batch, -1) for x in (s, a, R, s2, d)])
    torch.cuda.synchronize()
    for w in ARENAS:
        assert torch.equal(sampled.export_arena(w), direct.export_arena(w)), w
    rb.close(); sampled.close(); direct.close()


def test_per_replica_settings_and_stream_order(cuda):
    spec, E, R = SMALL, 5, 3
    core = _new(spec, replicas=R, critic_ensemble=E)
    core.set_ensemble(1, "min", replica=0)
    core.set_ensemble(5, "mean", replica=2)
    assert [core.get_ensemble(r) for r in range(R)] == [(1, "min"), (2, "mean"), (5, "mean")]
    _run(core, spec, R, 1)
    assert [int(core.debug("tsub", r).sum().item()) for r in range(R)] == [1, 2, 5]
    # a setting written on a side stream between launches of steps applies to the later ones only
    side = torch.cuda.Stream()
    (s, a, rw, s2, d), e1, e2 = _inputs(spec, False, R, 7)
    core.step(s, a, rw, s2, d, e1, e2)
    ev = torch.cuda.Event()
    ev.record()
    with torch.cuda.stream(side):
        side.wait_event(ev)
        core.set_ensemble(3, "mean", replica=1)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert int(core.debug("tsub", 1).sum().item()) == 2
    core.step(s, a, rw, s2, d, e1, e2)
    torch.cuda.synchronize()
    assert int(core.debug("tsub", 1).sum().item()) == 3
    core.close()


@pytest.mark.parametrize("where", ["current", "side"])
def test_prepared_graphs_pick_up_set_ensemble_in_stream_order(cuda, where):
    """Graph launches of b200sac_prepare's graphs, set_ensemble enqueued between them (on the step's stream, or on a side
    stream ordered by events): the step enqueued before the call keeps the old (m, reduction), the later ones take the
    new, exactly as a handle that synchronises and sets in between."""
    from distributed_sac_b200.core import Replay
    spec, E = SMALL, 4
    cores, rings = [], []
    for _ in range(2):
        c = _new(spec, critic_ensemble=E)
        rb = Replay(c, 8 * spec.batch, "device", seed=1)
        rb.fill_synthetic(8 * spec.batch, seed=2)
        c.prepare(rb)
        cores.append(c); rings.append(rb)
    async_core, ref = cores
    async_core.step_sampled(rings[0], 2)
    if where == "side":
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            async_core.set_ensemble(4, "min")
        torch.cuda.current_stream().wait_stream(side)
    else:
        async_core.set_ensemble(4, "min")
    async_core.step_sampled(rings[0], 2)
    torch.cuda.synchronize()
    assert async_core.debug("tsub").sum().item() == 4
    ref.step_sampled(rings[1], 2)
    torch.cuda.synchronize()
    assert ref.debug("tsub").sum().item() == 2
    ref.set_ensemble(4, "min")
    ref.step_sampled(rings[1], 2)
    torch.cuda.synchronize()
    for w in ARENAS:
        assert torch.equal(async_core.export_arena(w), ref.export_arena(w)), w
    assert torch.equal(async_core.read_losses(4), ref.read_losses(4))
    for x in rings + cores:
        x.close()


def test_critic_only_steps_clip_norms_and_copy_replica(cuda):
    spec, E, R = SMALL, 6, 2
    core = _new(spec, replicas=R, critic_ensemble=E, grad_clip=True)
    core.set_update_intervals(2, 1)
    before = core.get_named(_lib.PARAMS, 0)
    _run(core, spec, R, 1)                       # critic count 1: a critic-only step
    after = core.get_named(_lib.PARAMS, 0)
    assert torch.equal(before["actor.0.weight"], after["actor.0.weight"])
    for k in range(1, E + 1):
        assert not torch.equal(before[f"q{k}.0.weight"], after[f"q{k}.0.weight"])
    g = core.export_arena(_lib.GRADS, 0).double()
    tab = core.table
    lo, hi = tab["q1.0.weight"][0], tab["log_alpha"][0]
    norm = core.read_grad_norms(1)[0, 0, 0].item()
    assert abs(norm - g[lo:hi].norm().item()) <= 1e-5 * norm
    core.copy_replica(0, 1)
    torch.cuda.synchronize()
    assert torch.equal(core.export_arena(_lib.PARAMS, 0), core.export_arena(_lib.PARAMS, 1))
    core.close()


def test_reset_soft_update_and_critic_values(cuda):
    spec, E = SMALL, 7
    core = _new(spec, critic_ensemble=E)
    created = core.get_named()
    _run(core, spec, 1, 3)
    core.reset(SEED, critic=99)
    torch.cuda.synchronize()
    now = core.get_named()
    for k in range(1, E + 1):
        for n in (f"q{k}.0.weight", f"q{k}.2.bias", f"q{k}_target.1.weight"):
            assert torch.equal(now[n], created[n]), n
    _run(core, spec, 1, 2)
    for k in range(1, E + 1):
        core.soft_update(1.0, critic=k)
        torch.cuda.synchronize()
        named = core.get_named()
        assert torch.equal(named[f"q{k}.1.weight"], named[f"q{k}_target.1.weight"])
        if k < E:
            assert not torch.equal(named[f"q{k + 1}.1.weight"], named[f"q{k + 1}_target.1.weight"])
    with pytest.raises(RuntimeError):
        core.soft_update(1.0, critic=E + 1)
    # critic values against the oracle's networks, in any chunking
    g = torch.Generator().manual_seed(3)
    obs, act = torch.randn(300, spec.obs_dim, generator=g), torch.randn(300, spec.act_dim, generator=g)
    q = core.critic_values(obs, act).cpu()
    assert q.shape == (E, 300)
    named = core.get_named()
    p = {k: named[k] for k in named}
    for k in range(E):
        ref = sp.mlp(p, f"q{k + 1}", torch.cat([obs, act], -1)).squeeze(-1)
        assert torch.allclose(q[k], ref, rtol=1e-4, atol=1e-4)
    part = core.critic_values(obs[100:137], act[100:137]).cpu()
    assert torch.equal(part, q[:, 100:137])
    qt = core.critic_values(obs, act, target=True).cpu()
    assert qt.shape == (E, 300)
    core.close()


def test_plan_and_refusals(cuda):
    from distributed_sac_b200.core import Replay
    for spec in (sp.ll_spec(), sp.vs_spec(batch=256)):
        twin = _new(spec)
        ens = _new(spec, critic_ensemble=3)
        assert ens.launches_per_step == twin.launches_per_step
        assert plan_labels(ens) == plan_labels(twin)
        twin.close(); ens.close()
    # E = 10 keeps the twin plan's launches while a grouped launch holds at most GS_MAXG = 24 problems (LL: no split-K at
    # batch 256); at batch 1024 the ten critics' 4-way split weight gradients (40 problems) take two launches per layer
    for spec, more in ((sp.ll_spec(), False), (sp.vs_spec(batch=1024), True)):
        twin, big = _new(spec, precision=0), _new(spec, precision=0, critic_ensemble=10)
        if more:
            assert big.launches_per_step > twin.launches_per_step
        else:
            assert big.launches_per_step == twin.launches_per_step
            assert plan_labels(big) == plan_labels(twin)
        twin.close(); big.close()
    twin = _new(SMALL)
    with pytest.raises(RuntimeError, match="critic_ensemble"):
        twin.set_ensemble(2)
    with pytest.raises(RuntimeError, match="critic_ensemble"):
        twin.get_ensemble()
    ens = _new(SMALL, critic_ensemble=4)
    for m, mode in ((0, "mean"), (5, "min")):
        with pytest.raises(RuntimeError, match="subset"):
            ens.set_ensemble(m, mode)
    with pytest.raises(ValueError):
        ens.set_ensemble(2, "median")
    assert _lib.load().b200sac_set_ensemble(ens._h, 0, 2, 2, None) == -1
    assert ens.get_ensemble() == (2, "mean")
    obs = torch.zeros(4, SMALL.obs_dim)
    with pytest.raises(RuntimeError, match="ReDo"):
        ens.redo(1, obs, torch.zeros(4, SMALL.act_dim))
    with pytest.raises(RuntimeError, match="prioritized"):
        Replay(ens, 4 * SMALL.batch, "device", seed=1, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6))
    with pytest.raises(RuntimeError, match="tsub"):
        twin.debug("tsub")
    twin.close(); ens.close()


# ---- learners --------------------------------------------------------------------------------------------------------------
MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


@pytest.mark.parametrize("family", ["LL", "MS"])
def test_learner_ensemble_and_checkpoints(cuda, tmp_path, monkeypatch, family):
    import json
    from distributed_sac_b200 import learner as L
    monkeypatch.chdir(tmp_path)
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(MS_CFG if family == "MS" else LEARNER_CFGS[family]))

    def make(tag, **kw):
        kw = dict(dict(write_mode=False, replay_where="device"), **kw)
        srv = redis_stub.StrictRedis(host=str(tmp_path) + tag)
        if family == "MS":
            return L.MTSACLearner(None, ["t0", "t1", "t2"], str(p), server=srv, **kw)
        return L.LunarLanderLearner(str(p), server=srv, **kw)
    lr = make("a", critic_ensemble=10, target_subset=3, actor_q="min")
    assert lr.core.get_ensemble() == (3, "min")
    lr.set_ensemble(target_subset=2)
    assert lr.core.get_ensemble() == (2, "min")
    lr.memory.ring.fill_synthetic(4096, seed=1)
    for _ in range(3):
        out = lr.update()
        assert all(np.isfinite(x) for x in out[:2])
    assert lr.core.debug("tsub").sum().item() == 2
    obs = torch.zeros(5, lr.core.cfg.obs_dim)
    assert lr.q_values(obs, torch.zeros(5, lr.core.cfg.act_dim)).shape == (10, 5)
    if family == "LL":
        lr.soft_update(lr.local_critic_10, lr.target_critic_10, 1.0)
        named = lr.core.get_named()
        assert torch.equal(named["q10.0.weight"], named["q10_target.0.weight"])
        assert not torch.equal(named["q9.0.weight"], named["q9_target.0.weight"])
    path = lr.save_checkpoint(1)
    ck = torch.load(path, weights_only=False)
    if family == "LL":
        assert {f"local_critic_{k}" for k in range(1, 11)} <= set(ck) and "target_critic_10" in ck
    else:
        assert "Q_function_10.0.weight" in ck["local_critic"] and "Q_function_10.0.weight" in ck["target_critic"]
    n_critic_tensors = sum(len(lr._key_map(f"q{k}")) for k in range(1, 11))
    assert len(ck["critic_optimizer"]["state"]) == n_critic_tensors
    lr2 = make("b", critic_ensemble=10, checkpoint_path=path)
    for w in ARENAS:
        assert torch.equal(lr.core.export_arena(w), lr2.core.export_arena(w)), w
    assert tuple(lr.core.get_steps())[:3] == tuple(lr2.core.get_steps())[:3]
    five, twin = make("c", critic_ensemble=5), make("d")
    for other in (five, twin):                       # another ensemble size, or the twins, refuse the checkpoint
        with pytest.raises(ValueError, match="critics"):
            other.load_checkpoint(path)
    with pytest.raises(ValueError, match="critics"):
        lr2.load_checkpoint(twin.save_checkpoint(2))
    for x in (lr, lr2, five, twin):
        x.memory.stop()
