"""CPU: dropout Q-functions (b200sac_cfg.critic_dropout, DroQ) without a GPU -- the Philox reference against known-answer
vectors, the refusals and the layout, the C signatures, the learner argument checks, the DroQ oracle against the
LayerNorm oracle and fp64 autograd, and the MS state_dict keys."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import critic_ln_port as lnp
import droq_port as dq
import philox_ref as pr
import sac_port as sp
from distributed_sac_b200 import _lib, names
from distributed_sac_b200.core import CoreConfig, layout

SHAPES = {
    "LL": dict(state_dim=8, act_dim=2, actor_hidden=[256, 256], critic_hidden=[256, 256], batch=256),
    "VS": dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 300, 200], batch=1024),
    "MS": dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 400, 400], batch=1280,
               num_tasks=10, weighted_loss=True),
}


# ---- Philox4x32-10: Random123's known-answer vectors (key[0] = the seed's low 32 bits) ----------------------------------
@pytest.mark.parametrize("seed,counter,want", [
    (0, (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    (0xFFFFFFFFFFFFFFFF, (0xFFFFFFFF,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    (0x299f31d0a4093822, (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(seed, counter, want):
    assert tuple(int(x) for x in pr.philox(seed, *counter)) == want


def test_mask_draw_follows_the_documented_layout():
    seed, rep, step, p, B, H = 0x1234_5678_9ABC_DEF0, 2, (1 << 32) + 7, 0.3, 5, 13
    m = pr.drop_masks(seed, rep, step, "pi", 3, 1, B, H, p)
    key = (seed ^ (0xE7037ED1A0B428DB * 3)) & (2 ** 64 - 1)
    tag = (2 * 8 + 3) * 2 + 1
    t = math.floor(p * 2 ** 32)
    for b in range(B):
        for j in range(H):
            w = pr.philox(key, 7, 1, b, (tag << 24) | (j // 4))[j % 4]
            assert bool(m[b, j]) == (int(w) >= t), (b, j)
    assert pr.drop_masks(seed, rep, step, 0, 0, 0, B, H, 0.0).all()
    assert pr.scale(0.0) == np.float32(1.0) and pr.scale(0.5) == np.float32(2.0)


def test_masks_differ_per_coordinate():
    base = dict(seed=3, replica=0, step=1, pass_=0, layer=0, net=0, B=64, H=96, p=0.5)
    ref = pr.drop_masks(**base)
    for k, v in (("replica", 1), ("step", 2), ("pass_", 1), ("layer", 1), ("net", 1), ("seed", 4)):
        assert (pr.drop_masks(**dict(base, **{k: v})) != ref).any(), k
    assert abs(ref.mean() - 0.5) < 5 * 0.5 / math.sqrt(ref.size)


# ---- refusals, layout and signatures -----------------------------------------------------------------------------------
def _layout_rc(c):
    n = C.c_int32(0)
    return _lib.load().b200sac_layout(C.byref(c), None, 0, C.byref(n), None, None)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_layout_equals_layer_norm_layout(shape):
    ln = layout(CoreConfig(**SHAPES[shape], critic_layer_norm=True))
    dr = layout(CoreConfig(**SHAPES[shape], critic_layer_norm=True, critic_dropout=True))
    assert dr == ln


@pytest.mark.parametrize("ln,drop", [(0, 1), (1, 2), (1, -1), (0, 2)])
def test_layout_and_create_refuse_bad_cfgs(ln, drop):
    c = CoreConfig(**SHAPES["LL"]).to_c()
    c.critic_ln, c.critic_dropout = ln, drop
    assert _layout_rc(c) == -1                                  # B200SAC_ERR_INVALID
    assert "critic_dropout" in _lib.load().b200sac_last_error().decode()
    # create checks the cfg before it touches a device
    h = C.c_void_p()
    assert _lib.load().b200sac_create(C.byref(c), 0, 0, C.byref(h)) == -1
    assert not h.value


@pytest.mark.parametrize("kw", [dict(care=True, num_tasks=10, batch=260), dict(pcgrad=True, num_tasks=10, batch=260)])
def test_care_and_pcgrad_refused_through_layer_norm(kw):
    with pytest.raises(RuntimeError, match="critic_ln"):
        layout(CoreConfig(**dict(SHAPES["LL"], **kw), critic_layer_norm=True, critic_dropout=True))


def test_ctypes_struct_and_signatures_match_header():
    import os
    hdr = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "b200sac.h")).read()
    body = hdr[hdr.index("typedef struct b200sac_cfg {"):hdr.index("} b200sac_cfg;")]
    fields = [f for f, _ in _lib.Cfg._fields_]
    assert fields[-2:] == ["critic_ln", "critic_dropout"]
    assert body.rstrip().splitlines()[-3].split()[1] == "critic_dropout;"
    assert _lib.Cfg.critic_dropout.offset == _lib.Cfg.critic_ln.offset + 4
    assert "int b200sac_set_critic_dropout(b200sac_t* h, int32_t replica, double p, void* stream);" in hdr
    assert "int b200sac_get_critic_dropout(b200sac_t* h, int32_t replica, double* p);" in hdr
    assert _lib.SYMBOLS["b200sac_set_critic_dropout"] == (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_void_p])
    assert _lib.SYMBOLS["b200sac_get_critic_dropout"] == (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_double)])
    lib = _lib.load()
    assert lib.b200sac_set_critic_dropout(None, 0, 0.1, None) == -1
    assert lib.b200sac_get_critic_dropout(None, 0, None) == -1


# ---- learner checks, before any handle is built ----------------------------------------------------------------------------
MS_CFG = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 60, "gamma": 0.99, "tau": 0.005,
          "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": 3,
          "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-1.0, 1.0], "actor_hidden_dim": [64, 64]},
          "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}


def _cfg_file(tmp_path, family):
    from _harness import LEARNER_CFGS
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(MS_CFG if family == "MS" else LEARNER_CFGS[family]))
    return str(p)


def _no_handles(monkeypatch):
    from distributed_sac_b200 import learner as L
    import distributed_sac_b200.core as core

    def no_handle(*a, **k):
        raise AssertionError("a handle was built")
    monkeypatch.setattr(L, "SacCore", no_handle)
    monkeypatch.setattr(core, "SacCore", no_handle)
    return L


@pytest.mark.parametrize("kw,match", [
    (dict(critic_dropout=0.01), "critic_layer_norm"),
    (dict(critic_dropout=-0.1, critic_layer_norm=True), r"\[0, 1\)"),
    (dict(critic_dropout=1.0, critic_layer_norm=True), r"\[0, 1\)"),
    (dict(critic_dropout=float("nan"), critic_layer_norm=True), r"\[0, 1\)"),
    (dict(critic_dropout=True, critic_layer_norm=True), r"\[0, 1\)"),
])
@pytest.mark.parametrize("family", ["LL", "VS"])
def test_learner_refuses_bad_dropout_before_building(tmp_path, monkeypatch, kw, match, family):
    L = _no_handles(monkeypatch)
    cls = L.LunarLanderLearner if family == "LL" else L.VSACLearner
    with pytest.raises(ValueError, match=match):
        cls(_cfg_file(tmp_path, family), write_mode=False, **kw)


def test_mtsac_learner_refuses_bad_dropout_before_building(tmp_path, monkeypatch):
    L = _no_handles(monkeypatch)
    with pytest.raises(ValueError, match=r"\[0, 1\)"):
        L.MTSACLearner(None, ["t0", "t1", "t2"], _cfg_file(tmp_path, "MS"), write_mode=False, critic_layer_norm=True,
                       critic_dropout=1.5)


@pytest.mark.parametrize("ln", [False, True])
def test_care_learner_refuses_dropout_before_building(tmp_path, monkeypatch, ln):
    from distributed_sac_b200 import learner as L
    monkeypatch.setattr(L, "SacCore", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a handle was built")))
    monkeypatch.setattr(L.CARELearner, "_set_dims", lambda self: setattr(self, "num_tasks", 10))
    p = tmp_path / "care.json"
    p.write_text("{}")
    with pytest.raises(ValueError, match="critic_layer_norm"):
        L.CARELearner([], [], str(p), write_mode=False, critic_layer_norm=ln, critic_dropout=0.01)


# ---- the DroQ oracle ---------------------------------------------------------------------------------------------------------
SMALL = dict(state_dim=8, act_dim=2, actor_hidden=[32, 32], critic_hidden=[24, 40], batch=16)


def test_droq_port_at_zero_equals_layer_norm_port():
    spec = sp.SacSpec(**SMALL)
    params = lnp.init_params(spec, seed=4)
    a, b = lnp.LnPortLearner(spec, params), dq.DroqPortLearner(spec, params, 0.0, seed=9)
    gen = torch.Generator().manual_seed(1)
    for i in range(3):
        batch = sp.synthetic_batch(spec, seed=20 + i)
        e1, e2 = torch.randn(16, 2, generator=gen), torch.randn(16, 2, generator=gen)
        oa, ob = a.update_SAC(*batch, e1, e2), b.update_SAC(*batch, e1, e2)
        assert oa == ob
    for k, v in a.params().items():
        assert torch.equal(v, b.params()[k]), k
    assert b.step == 3


def test_droq_port_drops_the_philox_masks():
    spec = sp.SacSpec(**SMALL)
    params = lnp.init_params(spec, seed=4)
    port = dq.DroqPortLearner(spec, params, 0.5, seed=9, step=4)
    seen, droq_mlp = {}, dq.mlp

    def spy(params, net, x, tag=None):
        if net.startswith("q"):
            seen[(net, tag)] = dict(dq._masks)
        return droq_mlp(params, net, x, tag)
    gen = torch.Generator().manual_seed(1)
    batch = sp.synthetic_batch(spec, seed=3)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(dq, "mlp", spy)
        port.update_SAC(*batch, torch.randn(16, 2, generator=gen), torch.randn(16, 2, generator=gen))
    assert {t for _, t in seen} == {"cur", "next", "pi"}
    m = seen[("q2", "pi")][(1, "pi", 1)]
    want = pr.drop_masks(9, 0, 5, 2, 1, 1, 16, 40, 0.5)
    assert torch.equal(m, torch.from_numpy(want).float() * 2.0)


@pytest.mark.parametrize("rows,H,p", [(37, 96, 0.1), (16, 300, 0.5), (9, 1, 0.3), (5, 64, 0.01)])
def test_droq_backward_matches_fp64_autograd(rows, H, p):
    g = torch.Generator().manual_seed(rows * 1000 + H)
    z = torch.randn(rows, H, generator=g, dtype=torch.float64)
    w = 1.0 + 0.2 * torch.randn(H, generator=g, dtype=torch.float64)
    b = 0.1 * torch.randn(H, generator=g, dtype=torch.float64)
    up = torch.randn(rows, H, generator=g, dtype=torch.float64)
    m = torch.from_numpy(pr.drop_masks(5, 0, 1, 0, 0, 0, rows, H, p))
    s = float(pr.scale(p))
    zt, wt, bt = (t.clone().requires_grad_(True) for t in (z, w, b))
    h = torch.relu(F.layer_norm(zt * (m.double() * s), (H,), wt, bt, eps=lnp.EPS))
    (h * up).sum().backward()
    dy = up.numpy() * (h.detach().numpy() > 0)
    dz, dg, dc = dq.drop_backward(dy, z.numpy(), w.numpy(), m.numpy(), s)
    scale = lambda t: max(1.0, float(np.abs(t).max()))
    np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-9, atol=1e-9 * scale(zt.grad.numpy()))
    np.testing.assert_allclose(dg, wt.grad.numpy(), rtol=1e-10, atol=1e-10 * scale(dg))
    np.testing.assert_allclose(dc, bt.grad.numpy(), rtol=1e-10, atol=1e-10 * scale(dc))
    assert (dz[~m.numpy()] == 0).all()
    # the fp32 DroQ mlp's critic gradients agree with the same graph in fp64
    spec = sp.SacSpec(**dict(SMALL, critic_hidden=[H], batch=rows))
    params = {k: v.double() for k, v in lnp.init_params(spec, seed=2).items()}
    x = torch.randn(rows, spec.obs_dim + spec.act_dim, generator=g, dtype=torch.float64)
    masks = dq.step_masks(spec, 5, 1, p)
    grads = {}
    for dt in (torch.float32, torch.float64):
        pp = {k: v.to(dt).requires_grad_(k.startswith("q1.")) for k, v in params.items()}
        with dq._droq_mlp({k: (mm.to(dt) * torch.tensor(pr.scale(p), dtype=torch.float32).to(dt)) for k, mm in masks.items()}):
            sp.mlp(pp, "q1", x.to(dt), "cur").sum().backward()
        grads[dt] = {k: v.grad.double() for k, v in pp.items() if v.grad is not None}
    for k, v in grads[torch.float64].items():
        assert float((grads[torch.float32][k] - v).norm()) <= 1e-5 * max(float(v.norm()), 1e-6), k


# ---- the MS key map loads strictly into nn.Sequential(Linear, Dropout, LayerNorm, ReLU, ...) -----------------------------------
class DroqTwinCritic(nn.Module):
    def __init__(self, inp, hidden, p=0.01):
        super().__init__()
        for w in (1, 2):
            layers, a = [], inp
            for h in hidden:
                layers += [nn.Linear(a, h), nn.Dropout(p), nn.LayerNorm(h, eps=1e-5), nn.ReLU()]
                a = h
            setattr(self, f"Q_function_{w}", nn.Sequential(*layers, nn.Linear(a, 1)))


def test_ms_state_dict_loads_strict_into_droq_sequential():
    table, _, _ = layout(CoreConfig(**SHAPES["MS"], critic_layer_norm=True, critic_dropout=True))
    can = {k: torch.randn(r, c) if c > 1 else torch.randn(r) for k, (off, r, c, t, o, p) in table.items()}
    hid = SHAPES["MS"]["critic_hidden"]
    Lc = len(hid)
    m = DroqTwinCritic(SHAPES["MS"]["state_dim"] + SHAPES["MS"]["num_tasks"] + SHAPES["MS"]["act_dim"], list(hid))
    sd = {}
    for which in (1, 2):
        km = names.critic_key_map("MS", Lc + 1, which, layer_norm=True, dropout=True)
        sd.update({ref: can[c] for ref, c in km.items()})
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.Q_function_1[2].bias.data, can["q1.0.ln.bias"])
    assert torch.equal(m.Q_function_2[4 * Lc].weight.data.reshape(-1), can[f"q2.{Lc}.weight"].reshape(-1))
    # LL / VS keys do not change: the dropout has no parameters
    for fam in ("LL", "VS"):
        assert names.critic_key_map(fam, 3, 1, layer_norm=True, dropout=True) == names.critic_key_map(fam, 3, 1, layer_norm=True)
    with pytest.raises(ValueError):
        names.critic_key_map("MS", 3, 1, dropout=True)
