"""CPU: the CAGrad solve the device implements (cagrad_ref.solve) against autograd + torch.optim.SGD (cagrad_ref.literal),
SLSQP's optimum of the same dual, its scale invariance, the mirror-image closed form, and cagrad_update's Adam input
against the literal CAGrad combination of the per-task mean gradients."""
import math

import numpy as np
import pytest
import scipy.optimize
import torch

import cagrad_ref as cr
from _cagrad import gram_sets
import pcgrad_ref as pr
import sac_port as sp


SETS = gram_sets()
IDS = [f"T{T}-{kind}-c{c}" for T, kind, c, _ in SETS]


@pytest.mark.parametrize("T,kind,c,G", SETS, ids=IDS)
def test_solve_matches_literal(T, kind, c, G):
    a, b = cr.solve(G, c), cr.literal(G, c)
    assert a["ibest"] == b["ibest"]
    for k in ("lam", "best", "first", "scale"):
        assert abs(a[k] - b[k]) <= 1e-12 * max(1.0, abs(b[k])), k
    assert np.max(np.abs(a["p"] - b["p"])) <= 1e-12
    assert np.max(np.abs(a["w"] - b["w"])) <= 1e-12 * np.abs(b["w"]).max()


@pytest.mark.parametrize("T,kind,c,G", SETS, ids=IDS)
def test_best_between_slsqp_and_uniform(T, kind, c, G):
    rec = cr.solve(G, c)
    A = G / rec["scale"] ** 2
    u = np.full(T, 1.0 / T)
    assert rec["first"] == pytest.approx(cr.objective(A, c, u), rel=1e-12)
    assert rec["best"] <= rec["first"]
    assert rec["best"] == pytest.approx(cr.objective(A, c, rec["p"]), rel=1e-12)
    opt = scipy.optimize.minimize(lambda p: cr.objective(A, c, p), u, method="SLSQP", bounds=[(0.0, 1.0)] * T,
                                  constraints=[{"type": "eq", "fun": lambda p: p.sum() - 1.0}],
                                  options={"ftol": 1e-12, "maxiter": 500})
    assert opt.success
    assert opt.fun <= rec["best"] + 1e-9 * abs(rec["best"])


@pytest.mark.parametrize("k", [1e-6, 1e-3, 1.0, 1e3, 1e6])
def test_scale_invariance(k):
    for T, kind, c, G in SETS[::3]:
        a, b = cr.solve(G, c), cr.solve(k * k * G, c)
        assert a["ibest"] == b["ibest"], (T, kind)
        assert np.allclose(a["p"], b["p"], rtol=0, atol=1e-12), (T, kind)
        assert np.allclose(a["w"], b["w"], rtol=1e-12, atol=0), (T, kind)
        assert b["scale"] == pytest.approx(k * a["scale"], rel=1e-12)


@pytest.mark.parametrize("h", [0.7, 0.0, -0.4, -1.0])
def test_mirror_image_tasks(h):
    """G_00 = G_11: the gradient of F vanishes at uniform weights, so p* = (1/2, 1/2) exactly and lambda has a closed form."""
    g = 2.5
    G = np.array([[g, h * g], [h * g, g]])
    c = 0.5
    rec = cr.solve(G, c)
    assert np.array_equal(rec["p"], np.array([0.5, 0.5])) and rec["ibest"] == 0
    abar = (1.0 + h) / 2.0
    lam = c * math.sqrt(abar + 1e-4) / (math.sqrt(abar + 1e-4) + 1e-4)
    assert rec["lam"] == pytest.approx(lam, rel=1e-14)
    assert np.allclose(rec["w"], (1.0 + lam) / (1.0 + c * c), rtol=1e-14)


def test_degenerate():
    for G in (np.zeros((3, 3)), np.array([[1.0, np.nan], [np.nan, 1.0]]), np.array([[np.inf, 0.0], [0.0, 1.0]])):
        rec = cr.solve(G, 0.5)
        assert rec["ibest"] == -2 and np.array_equal(rec["w32"], np.ones(G.shape[0], np.float32))
        assert np.isnan(rec["p"]).all() and math.isnan(rec["lam"])


def test_cagrad_update_adam_input():
    """The gradient cagrad_update hands each Adam is the literal CAGrad direction (g0 + lambda gw) / (1 + c^2) on the
    flattened per-task mean gradients G_t = T g_t (g0 their mean, gw = sum_t p*_t G_t), up to w's fp32 rounding."""
    T, c = 3, 0.5
    spec = sp.SacSpec(state_dim=6, act_dim=2, actor_hidden=[24, 20], critic_hidden=[20, 24], batch=60, num_tasks=T,
                      weighted_loss=True)
    params = sp.init_params(spec, seed=5)
    batch = pr.block_batch(spec, seed=21)
    g = torch.Generator().manual_seed(6)
    e1, e2 = torch.randn(spec.batch, spec.act_dim, generator=g), torch.randn(spec.batch, spec.act_dim, generator=g)
    port = sp.PortLearner(spec, params)
    seen = {}

    def capture(which):       # no update: the actor pass reads `params` like task_grads below
        return lambda *a, **k: seen.update({which: {n: port.p[n].grad.clone() for n in pr.opt_names(spec, which)}})
    port.opt_critic.step, port.opt_actor.step = capture(0), capture(1)
    recs = cr.cagrad_update(port, *batch, e1, e2, c)
    for which in (0, 1):
        names = pr.opt_names(spec, which)
        per = pr.flat(pr.task_grads(spec, params, batch, e1, e2, which), names)
        mean_grads = T * per
        rec = recs[which][2]
        assert rec["ibest"] >= 0
        g0 = mean_grads.mean(0)
        gw = rec["p"] @ mean_grads
        direction = (g0 + rec["lam"] * gw) / (1.0 + c * c)
        got = np.concatenate([seen[which][n].double().reshape(-1).numpy() for n in names])
        assert np.linalg.norm(got - direction) <= 1e-5 * np.linalg.norm(direction), which
        assert np.allclose(recs[which][0], per @ per.T, rtol=1e-10, atol=1e-12 * np.abs(recs[which][0]).max())
