"""CPU: layer-normalized critics (b200sac_cfg.critic_ln) without a GPU -- the layout table, the refusals, the learner
argument checks, the numpy LayerNorm backward the kernels implement, and the reference-format state_dict keys."""
import ctypes as C
import json

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import critic_ln_port as lnp
from distributed_sac_b200 import _lib, names
from distributed_sac_b200.core import CoreConfig, layout

SHAPES = {
    "LL": dict(state_dim=8, act_dim=2, actor_hidden=[256, 256], critic_hidden=[256, 256], batch=256),
    "VS": dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 300, 200], batch=1024),
    "MS": dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 400, 400], batch=1280,
               num_tasks=10, weighted_loss=True),
}


def _layout_list(cfg):
    lib = _lib.load()
    c = cfg.to_c()
    n, arena, train = C.c_int32(0), C.c_int64(0), C.c_int64(0)
    _lib.check(lib.b200sac_layout(C.byref(c), None, 0, C.byref(n), C.byref(arena), C.byref(train)))
    descs = (_lib.TensorDesc * n.value)()
    _lib.check(lib.b200sac_layout(C.byref(c), descs, n.value, C.byref(n), C.byref(arena), C.byref(train)))
    return [(d.name.decode(), d.offset, d.rows, d.cols, d.trainable, d.opt, d.pitch) for d in descs]


@pytest.mark.parametrize("shape", list(SHAPES))
def test_layout_keeps_every_other_tensor_and_places_layer_norm(shape):
    plain = _layout_list(CoreConfig(**SHAPES[shape]))
    ln = _layout_list(CoreConfig(**SHAPES[shape], critic_layer_norm=True))
    Lc = len(SHAPES[shape]["critic_hidden"])
    # every non-LayerNorm tensor keeps its name, shape, pitch, optimizer and order
    assert [(n, r, c, t, o, p) for n, _, r, c, t, o, p in ln if ".ln." not in n] == \
        [(n, r, c, t, o, p) for n, _, r, c, t, o, p in plain]
    by = {d[0]: d for d in ln}
    names_in_order = [d[0] for d in ln]
    for net in ("q1", "q2", "q1_target", "q2_target"):
        target = net.endswith("_target")
        for l, H in enumerate(SHAPES[shape]["critic_hidden"]):
            i = names_in_order.index(f"{net}.{l}.bias")
            assert names_in_order[i + 1:i + 3] == [f"{net}.{l}.ln.weight", f"{net}.{l}.ln.bias"]
            for kind in ("weight", "bias"):
                _, off, r, c, t, o, _ = by[f"{net}.{l}.ln.{kind}"]
                assert (r, c) == (H, 1)
                assert (t, o) == ((0, -1) if target else (1, 0))
        assert f"{net}.{Lc}.ln.weight" not in by            # the head has none
    # targets at + target_delta with the same relative layout, and q1 / q2 contiguous
    delta = by["q1_target.0.weight"][1] - by["q1.0.weight"][1]
    for n, off, *_ in ln:
        if n.startswith(("q1.", "q2.")):
            assert by[n.replace("q1.", "q1_target.").replace("q2.", "q2_target.")][1] == off + delta, n
    q = [d for d in ln if d[0].startswith(("q1.", "q2."))]
    for a, b in zip(q, q[1:]):
        assert b[1] == (a[1] + a[2] * a[6] + 3) // 4 * 4, (a[0], b[0])


@pytest.mark.parametrize("kw", [dict(care=True, num_tasks=10, batch=260), dict(pcgrad=True, num_tasks=10, batch=260)])
def test_layout_refuses_unsupported_combinations(kw):
    cfg = CoreConfig(**dict(SHAPES["LL"], **kw), critic_layer_norm=True)
    with pytest.raises(RuntimeError, match="critic_ln"):
        layout(cfg)
    layout(CoreConfig(**dict(SHAPES["LL"], **kw)))           # the same cfg without critic_ln is fine


def test_layout_refuses_bad_value():
    c = CoreConfig(**SHAPES["LL"]).to_c()
    c.critic_ln = 2
    n = C.c_int32(0)
    assert _lib.load().b200sac_layout(C.byref(c), None, 0, C.byref(n), None, None) == -1


def _cfg_file(tmp_path, family):
    from _harness import LEARNER_CFGS
    p = tmp_path / f"{family}.json"
    p.write_text(json.dumps(LEARNER_CFGS[family]))
    return str(p)


@pytest.mark.parametrize("kw", [dict(redo_interval=10), dict(redo_interval=5, redo=dict(actor=0.0, critic=0.1))])
def test_learner_refuses_redo_with_layer_norm_before_building(tmp_path, monkeypatch, kw):
    from distributed_sac_b200 import learner as L
    import distributed_sac_b200.core as core

    def no_handle(*a, **k):
        raise AssertionError("a handle was built")
    monkeypatch.setattr(L, "SacCore", no_handle)
    monkeypatch.setattr(core, "SacCore", no_handle)
    with pytest.raises(ValueError, match="critic_layer_norm"):
        L.LunarLanderLearner(_cfg_file(tmp_path, "LL"), write_mode=False, critic_layer_norm=True, **kw)


def test_care_learner_refuses_layer_norm_before_building(tmp_path, monkeypatch):
    from distributed_sac_b200 import learner as L
    monkeypatch.setattr(L, "SacCore", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a handle was built")))
    monkeypatch.setattr(L.CARELearner, "_set_dims", lambda self: setattr(self, "num_tasks", 10))
    p = tmp_path / "care.json"
    p.write_text("{}")
    with pytest.raises(ValueError, match="critic_layer_norm"):
        L.CARELearner([], [], str(p), write_mode=False, critic_layer_norm=True)


def test_dormant_fraction_refused():
    from distributed_sac_b200 import learner as L
    lr = L.LunarLanderLearner.__new__(L.LunarLanderLearner)
    lr.critic_layer_norm = True
    with pytest.raises(ValueError, match="critic_layer_norm"):
        lr.dormant_fraction(0.0)
    with pytest.raises(ValueError, match="critic_layer_norm"):
        lr._recycle(0, {})


# ---- the LayerNorm backward the kernels implement, against autograd in fp64 -----------------------------------------------
@pytest.mark.parametrize("rows,H,kind", [(37, 96, "random"), (5, 64, "constant"), (9, 1, "random"), (16, 300, "random")])
def test_numpy_layer_norm_backward_matches_autograd(rows, H, kind):
    g = torch.Generator().manual_seed(rows * 1000 + H)
    z = torch.randn(rows, H, generator=g, dtype=torch.float64)
    if kind == "constant":                     # var ~ 0: rstd ~ 1 / sqrt(eps)
        z = 3.0 + 1e-7 * z
    w = 1.0 + 0.2 * torch.randn(H, generator=g, dtype=torch.float64)
    b = 0.1 * torch.randn(H, generator=g, dtype=torch.float64)
    up = torch.randn(rows, H, generator=g, dtype=torch.float64)
    zt, wt, bt = (t.clone().requires_grad_(True) for t in (z, w, b))
    h = torch.relu(F.layer_norm(zt, (H,), wt, bt, eps=lnp.EPS))
    (h * up).sum().backward()
    h_np, _, _ = lnp.ln_forward(z.numpy(), w.numpy(), b.numpy())
    np.testing.assert_allclose(h_np, h.detach().numpy(), rtol=1e-12, atol=1e-12)
    dy = up.numpy() * (h_np > 0)               # the ReLU-masked gradient the kernel reads
    dz, dg, dc = lnp.ln_backward(dy, z.numpy(), w.numpy())
    scale = lambda t: max(1.0, float(np.abs(t).max()))
    np.testing.assert_allclose(dz, zt.grad.numpy(), rtol=1e-9, atol=1e-9 * scale(zt.grad.numpy()))
    np.testing.assert_allclose(dg, wt.grad.numpy(), rtol=1e-10, atol=1e-10 * scale(dg))
    np.testing.assert_allclose(dc, bt.grad.numpy(), rtol=1e-10, atol=1e-10 * scale(dc))


# ---- reference-format state dicts load into torch modules with LayerNorm ---------------------------------------------------
class LnCritic(nn.Module):
    """The LL / VS reference Critic (first_layer, layer_module) with a LayerNorm after every hidden Linear."""

    def __init__(self, inp, hidden):
        super().__init__()
        self.first_layer = nn.Linear(inp, hidden[0])
        self.layer_module = nn.ModuleList([nn.Linear(a, b) for a, b in zip(hidden, hidden[1:] + [1])])
        self.layer_norms = nn.ModuleList([nn.LayerNorm(h, eps=1e-5) for h in hidden])


class LnTwinCritic(nn.Module):
    """The MS reference's twin Critic with nn.Sequential(Linear, LayerNorm, ReLU, ..., Linear) Q-functions."""

    def __init__(self, inp, hidden):
        super().__init__()
        for w in (1, 2):
            layers, a = [], inp
            for h in hidden:
                layers += [nn.Linear(a, h), nn.LayerNorm(h, eps=1e-5), nn.ReLU()]
                a = h
            setattr(self, f"Q_function_{w}", nn.Sequential(*layers, nn.Linear(a, 1)))


def _canonical(shape):
    """A canonical tensor per layout entry, shaped as the library exports it."""
    table, _, _ = layout(CoreConfig(**SHAPES[shape], critic_layer_norm=True))
    return {k: torch.randn(r, c) if c > 1 else torch.randn(r) for k, (off, r, c, t, o, p) in table.items()}


@pytest.mark.parametrize("shape", ["LL", "VS"])
def test_ll_vs_state_dicts_load_strict(shape):
    can = _canonical(shape)
    hid = SHAPES[shape]["critic_hidden"]
    inp = SHAPES[shape]["state_dim"] + SHAPES[shape]["act_dim"]
    for which in (1, 2):
        for target in (False, True):
            km = names.critic_key_map(shape, len(hid) + 1, which, target=target, layer_norm=True)
            m = LnCritic(inp, list(hid))
            m.load_state_dict({ref: can[c] for ref, c in km.items()}, strict=True)
            assert torch.equal(m.layer_norms[0].weight.data, can[f"q{which}{'_target' if target else ''}.0.ln.weight"])
    # without layer_norm the map is exactly the plain one
    assert names.critic_key_map(shape, len(hid) + 1, 1) == \
        {k: v for k, v in names.critic_key_map(shape, len(hid) + 1, 1, layer_norm=True).items() if ".ln." not in v}


def test_ms_state_dict_loads_strict_into_sequential():
    can = _canonical("MS")
    hid = SHAPES["MS"]["critic_hidden"]
    inp = SHAPES["MS"]["state_dim"] + SHAPES["MS"]["num_tasks"] + SHAPES["MS"]["act_dim"]
    m = LnTwinCritic(inp, list(hid))
    assert isinstance(m.Q_function_1, nn.Sequential)
    sd = {}
    for which in (1, 2):
        km = names.critic_key_map("MS", len(hid) + 1, which, layer_norm=True)
        sd.update({ref: can[c] for ref, c in km.items()})
    m.load_state_dict(sd, strict=True)
    Lc = len(hid)
    assert torch.equal(m.Q_function_2[3 * Lc].weight.data.reshape(-1), can[f"q2.{Lc}.weight"].reshape(-1))
    assert torch.equal(m.Q_function_1[1].bias.data, can["q1.0.ln.bias"])
    # canonical layout order: the critic optimizer's parameter order
    order = list(names.critic_key_map("MS", Lc + 1, 1, layer_norm=True).values())
    table, _, _ = layout(CoreConfig(**SHAPES["MS"], critic_layer_norm=True))
    q1 = sorted((v[0], k) for k, v in table.items() if k.startswith("q1."))
    assert order == [k for _, k in q1]
