"""CPU: the fp32 restatement of the policy head (tests/_policy_head.py), which the GPU tests hold the kernels to bit for bit,
against the reference's formula (sac_port.policy_sample): in fp64 within the error bounds that follow from each point's
conditioning, in every regime the GPU tests build; in the oracle's own fp32 at well-conditioned points; and NaN where
torch.clamp propagates it."""
import zlib

import numpy as np
import pytest
import torch

import sac_port as sp
from _policy_head import BOUNDS, bounds, reference64, restate_dout, restate_point, row_sum

F32 = np.float32


def _points(regime, n, A, rng):
    """(mu, raw, eps) [n][A] of one regime of the raw log-std (or, "sat", of mu)."""
    mu = rng.normal(0, 1.5, (n, A)).astype(F32)
    raw = rng.normal(-0.5, 1.0, (n, A)).astype(F32)
    eps = rng.normal(0, 1, (n, A)).astype(F32)
    if regime == "high":
        raw = rng.uniform(2, 40, (n, A)).astype(F32)
        raw[raw <= 2] = 40
    elif regime == "low":
        raw = rng.uniform(-60, -20, (n, A)).astype(F32)
        raw[raw >= -20] = -60
    elif regime in BOUNDS:
        raw[:] = BOUNDS[regime]
    elif regime == "sat":
        mu = rng.uniform(-30, 30, (n, A)).astype(F32)
    elif regime in ("+inf", "-inf"):
        raw[:] = float(regime[0] + "inf")
    return mu, raw, eps


def _head_terms(mu, raw, eps, k, rng):
    B = mu.shape[0]
    p = restate_point(mu, raw, eps, k)
    da = rng.normal(0, 0.3, mu.shape).astype(F32)
    alpha = np.exp(rng.normal(-0.5, 0.5, B)).astype(F32)
    c = F32(1.0 / B)
    glp = c * alpha
    sv = np.stack([p[n] for n in ("std", "diff", "t", "act", "jac", "eps", "mask", "logp_j")], -1)
    dmu, dls = restate_dout(sv, da, alpha[:, None], c, k)
    return p, da, glp, dmu, dls


@pytest.mark.parametrize("k", [1.0, 1.5, 0.4])
@pytest.mark.parametrize("regime", ["nominal", "high", "low", *BOUNDS, "sat", "+inf", "-inf"])
def test_restatement_within_the_conditioning_bounds_of_the_fp64_reference(regime, k):
    rng = np.random.default_rng(zlib.crc32(f"{regime} {k}".encode()))
    mu, raw, eps = _points(regime, 512, 3, rng)
    p, da, glp, dmu, dls = _head_terms(mu, raw, eps, k, rng)
    act64, logp64, ls64, dmu64, dls64 = reference64(mu, raw, eps, da, glp, k)
    b_act, b_lp, b_mu, b_ls = bounds(p, mu, da, glp, k)
    assert (np.abs(p["act"] - act64) <= 2 * b_act + 1e-6 * np.abs(act64)).all()
    assert (np.abs(row_sum(p["logp_j"]) - logp64) <= 2 * b_lp.sum(-1) + 1e-6 * np.abs(logp64)).all()
    assert (np.abs(p["logstd"] - ls64) <= 8 * 2.0 ** -24 * np.abs(ls64) + 1e-7).all()
    assert (np.abs(dmu - dmu64) <= 2 * b_mu).all(), float((np.abs(dmu - dmu64) / b_mu).max())
    assert (np.abs(dls - dls64) <= 2 * b_ls).all(), float((np.abs(dls - dls64) / np.maximum(b_ls, 1e-300)).max())
    inside = (raw >= -20) & (raw <= 2)
    assert ((dls == 0) == ~inside).all() and ((dls64 == 0) == ~inside).all()
    benign = (1 - p["t"].astype(np.float64) ** 2 > 0.1) & inside
    if regime == "nominal":                    # where the point is benign, the bounds are tight enough to mean something
        assert benign.mean() > 0.5
        scale = np.abs(dmu64) + glp[:, None]
        assert (b_mu[benign] < 1e-4 * scale[benign]).all() and (b_act[benign] < 2e-6 * k).all()
        assert (b_ls[benign] < 1e-4 * (np.abs(dls64) + glp[:, None])[benign]).all()


def test_restatement_matches_the_fp32_oracle_at_well_conditioned_points():
    rng = np.random.default_rng(3)
    mu, raw, eps = _points("nominal", 256, 4, rng)
    mu = np.clip(mu, -1.5, 1.5)
    for k in (1.0, 1.5):
        p, da, glp, dmu, dls = _head_terms(mu, raw, eps, k, rng)
        spec = sp.SacSpec(act_dim=4, action_scale=k)
        head = torch.from_numpy(np.concatenate([mu, raw], -1)).requires_grad_(True)
        act, logp, _ = sp.policy_sample(spec, {}, head, torch.from_numpy(eps))
        ((torch.from_numpy(da) * act).sum() + (torch.from_numpy(glp) * logp[:, 0]).sum()).backward()
        g = head.grad.numpy()
        np.testing.assert_allclose(p["act"], act.detach().numpy(), rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(row_sum(p["logp_j"]), logp[:, 0].detach().numpy(), rtol=1e-5, atol=1e-5)
        scale = np.abs(g).mean()
        np.testing.assert_allclose(dmu, g[:, :4], rtol=1e-4, atol=1e-5 * scale)
        np.testing.assert_allclose(dls, g[:, 4:], rtol=1e-4, atol=1e-5 * scale)


def test_nan_log_std_propagates_like_torch_clamp():
    rng = np.random.default_rng(5)
    mu, raw, eps = _points("nominal", 16, 3, rng)
    raw[:, 1] = np.nan
    p, da, glp, dmu, dls = _head_terms(mu, raw, eps, 1.5, rng)
    act64, logp64, _, dmu64, dls64 = reference64(mu, raw, eps, da, glp, 1.5)
    for got, ref in ((p["act"], act64), (row_sum(p["logp_j"]), logp64), (dmu, dmu64), (dls, dls64)):
        assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.isnan(p["act"][:, 1]).all() and np.isfinite(p["act"][:, [0, 2]]).all() and np.isnan(logp64).all()
    assert p["mask"][:, 1].sum() == 0 and (dls[:, 1] == 0).all()      # torch.clamp's backward: no gradient at NaN
