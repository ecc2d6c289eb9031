"""CPU: critic ensembles (b200sac_cfg.critic_ensemble; REDQ, RLPD) without a GPU -- the layout (names, offsets,
contiguity, the twin prefix, arena sizes), the refusals, the C signatures, the subset restatement and the oracle against
sac_port at E = 2."""
import ctypes as C

import numpy as np
import pytest
import torch

import redq_port as rq
import redq_ref
import sac_port as sp
from distributed_sac_b200 import _lib
from distributed_sac_b200.core import CoreConfig, layout

LL = dict(state_dim=8, act_dim=2, actor_hidden=[256, 256], critic_hidden=[256, 256], batch=256)
VS = dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 300, 200], batch=1024)


def _layout(**kw):
    return layout(CoreConfig(**kw))


@pytest.mark.parametrize("shape", [LL, VS], ids=["LL", "VS"])
@pytest.mark.parametrize("ln", [False, True])
def test_layout_appends_critics_and_keeps_the_twin_prefix(shape, ln):
    twin, arena2, train2 = _layout(critic_layer_norm=ln, **shape)
    per_net = twin["q2.0.weight"][0] - twin["q1.0.weight"][0]
    for E in range(2, 11):
        tab, arena, train = _layout(critic_ensemble=E, critic_layer_norm=ln, **shape)
        names = list(tab)
        for name, d in twin.items():          # actor, q1, q2, their targets and log_alpha keep their descriptors ...
            if not name.startswith(("q1_target", "q2_target", "log_alpha")):
                assert tab[name] == d, name
        extra = (E - 2) * per_net
        assert train == train2 + extra and arena == arena2 + 2 * extra
        delta = tab["q1_target.0.weight"][0] - tab["q1.0.weight"][0]
        for k in range(1, E + 1):
            q = f"q{k}"
            assert tab[f"{q}.0.weight"][0] == tab["q1.0.weight"][0] + (k - 1) * per_net
            assert names.index(f"{q}.0.weight") < names.index("log_alpha") < names.index(f"{q}_target.0.weight")
            for name in (n for n in tab if n.startswith(q + ".")):
                t = tab[name.replace(q + ".", q + "_target.", 1)]
                assert t[0] == tab[name][0] + delta and tab[name][3] == 1 and t[3] == 0 and tab[name][4] == 0
        assert f"q{E + 1}.0.weight" not in tab
        # ... and q1 .. qE are one contiguous block right after the actor
        assert tab["log_alpha"][0] == tab["q1.0.weight"][0] + E * per_net


@pytest.mark.parametrize("bad", [1, -1, 11, 64])
def test_layout_refuses_ensemble_sizes(bad):
    with pytest.raises(RuntimeError, match="critic_ensemble"):
        _layout(critic_ensemble=bad, **LL)


def test_layout_refuses_care_and_pcgrad():
    with pytest.raises(RuntimeError, match="critic_ensemble"):
        _layout(critic_ensemble=3, pcgrad=True, num_tasks=2, **LL)
    c = CoreConfig(critic_ensemble=3, **LL).to_c()
    c.care, c.num_tasks = 1, 2
    lib = _lib.load()
    n = C.c_int32(0)
    assert lib.b200sac_layout(C.byref(c), None, 0, C.byref(n), None, None) == -1      # B200SAC_ERR_INVALID


def test_c_signatures():
    lib = _lib.load()
    assert lib.b200sac_set_ensemble.argtypes == [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    assert lib.b200sac_get_ensemble.argtypes == [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    fields = [f for f, _ in _lib.Cfg._fields_]
    assert fields[fields.index("pcgrad") + 1] == "critic_ensemble"


def test_subset_restatement():
    seed = 0x1234_5678_9ABC_DEF0
    for E in range(2, 11):
        for m in range(1, E + 1):
            for step in (1, 2, (1 << 32) + 3):
                for rep in (0, 3):
                    s = redq_ref.subset(seed, rep, step, E, m)
                    assert s.sum() == m
                    if m < E:
                        w = redq_ref.words(seed, rep, step, E)
                        # every chosen (w, k) precedes every unchosen one
                        assert max((int(w[k]), k) for k in range(E) if s[k]) < min((int(w[k]), k) for k in range(E) if not s[k])
        assert redq_ref.subset(seed, 0, 5, E, E).all()
    # the counter's fourth word selects the group of four, the key the replica and the step the draw
    w = redq_ref.words(seed, 1, 9, 10)
    assert len(w) == 10 and not np.array_equal(w, redq_ref.words(seed, 2, 9, 10))
    assert not np.array_equal(w, redq_ref.words(seed, 1, 10, 10))
    draws = {tuple(redq_ref.subset(seed, 0, k, 10, 2)) for k in range(1, 200)}
    assert len(draws) > 30


def test_oracle_twin_equals_sac_port():
    spec = sp.ll_spec(batch=64, actor_hidden=[32, 32], critic_hidden=[32, 32])
    p = sp.init_params(spec, seed=3)
    ref = sp.PortLearner(spec, p)
    ens = rq.RedqPortLearner(spec, p, E=2, m=2, actor="min", seed=5)
    g = torch.Generator().manual_seed(0)
    for i in range(3):
        s, a, r, s2, d = sp.synthetic_batch(spec, seed=40 + i)
        e1, e2 = (torch.randn(spec.batch, spec.act_dim, generator=g) for _ in range(2))
        lo_ref = ref.update_SAC(s, a, r, s2, d, e1, e2)
        lo = ens.update_SAC(s, a, r, s2, d, e1, e2)
        for k in ("critic_loss", "actor_loss", "alpha_loss", "entropy"):
            assert lo[k] == lo_ref[k], k
    for k, v in ref.params().items():
        assert torch.equal(v, ens.params()[k]), k


def test_oracle_takes_the_subset_min():
    spec = sp.ll_spec(batch=16, actor_hidden=[8], critic_hidden=[8])
    E = 5
    p = rq.init_params(spec, E, seed=1)
    port = rq.RedqPortLearner(spec, p, E=E, m=2, actor="mean", seed=9)
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=2)
    e1 = torch.zeros(spec.batch, spec.act_dim)
    out = port.update_SAC(s, a, r, s2, d, e1, e1)
    S = redq_ref.subset(9, 0, 1, E, 2)
    assert np.array_equal(port.last_subset, S) and S.sum() == 2
    assert out["q"].shape == (E, spec.batch, 1)


# ---- learner checks, before any handle is built ----------------------------------------------------------------------------
MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


def _make(tmp_path, monkeypatch, family, **kw):
    import json
    from _harness import LEARNER_CFGS
    from distributed_sac_b200 import learner as L
    import distributed_sac_b200.core as core

    def no_handle(*a, **k):
        raise AssertionError("a handle was built")
    monkeypatch.setattr(L, "SacCore", no_handle)
    monkeypatch.setattr(core, "SacCore", no_handle)
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(MS_CFG if family == "MS" else LEARNER_CFGS[family]))
    if family == "MS":
        return L.MTSACLearner(None, ["t0", "t1", "t2"], str(p), write_mode=False, **kw)
    return (L.LunarLanderLearner if family == "LL" else L.VSACLearner)(str(p), write_mode=False, **kw)


@pytest.mark.parametrize("kw,match", [
    (dict(critic_ensemble=1), r"\[2, 10\]"),
    (dict(critic_ensemble=11), r"\[2, 10\]"),
    (dict(critic_ensemble=True), r"\[2, 10\]"),
    (dict(critic_ensemble=3.0), r"\[2, 10\]"),
    (dict(critic_ensemble=5, target_subset=0), "target_subset"),
    (dict(critic_ensemble=5, target_subset=6), "target_subset"),
    (dict(critic_ensemble=5, actor_q="median"), "actor_q"),
    (dict(critic_ensemble=5, redo_interval=10), "redo"),
    (dict(critic_ensemble=5, redo=dict(actor=0.0, critic=0.0), redo_interval=10), "redo"),
    (dict(critic_ensemble=5, replay_where="device", prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6)), "prioritized"),
])
@pytest.mark.parametrize("family", ["LL", "VS", "MS"])
def test_learner_refuses_bad_ensembles_before_building(tmp_path, monkeypatch, family, kw, match):
    with pytest.raises(ValueError, match=match):
        _make(tmp_path, monkeypatch, family, **kw)


@pytest.mark.parametrize("kw", [dict(pcgrad=True), dict(cagrad=0.5)])
def test_mtsac_learner_refuses_ensembles_with_gradient_surgery(tmp_path, monkeypatch, kw):
    with pytest.raises(ValueError, match="critic_ensemble"):
        _make(tmp_path, monkeypatch, "MS", critic_ensemble=4, **kw)


def test_care_learner_refuses_ensembles(tmp_path, monkeypatch):
    from distributed_sac_b200 import learner as L
    monkeypatch.setattr(L, "SacCore", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a handle was built")))
    monkeypatch.setattr(L.CARELearner, "_set_dims", lambda self: setattr(self, "num_tasks", 10))
    p = tmp_path / "care.json"
    p.write_text("{}")
    with pytest.raises(ValueError, match="CARE"):
        L.CARELearner([], [], str(p), write_mode=False, critic_ensemble=4)


def test_key_maps_of_every_critic():
    from distributed_sac_b200 import names
    for k in (3, 10):
        m = names.critic_key_map("MS", 3, k, target=True, layer_norm=True)
        assert m[f"Q_function_{k}.0.weight"] == f"q{k}_target.0.weight"
        assert m[f"Q_function_{k}.1.weight"] == f"q{k}_target.0.ln.weight"
        assert names.critic_key_map("LL", 3, k)["first_layer.weight"] == f"q{k}.0.weight"
