"""GPU: the two on-device random-number consumers against their distributions (SURVEY.md 8(a) a16 + the production noise).

* Parameter init (b200sac_create): nn.init.xavier_uniform_(gain 1) weights / zero biases for every nn.Linear
  (LunarLander_Distributed_SAC/src/model.py:33-36, MT10_Distributed_MTSAC/src/utils.py:30-33), torch.randn for the CARE
  mixture-of-encoders weights AND biases (MT10_Distributed_CARE/src/state_encoder.py:146-153), targets = hard copies.
* The reparameterisation noise the policy head draws in-kernel when no eps is injected (Philox4x32-10 + Box-Muller) --
  what every production step uses (Normal.rsample, model.py:55).
The checks are distributional (Kolmogorov-Smirnov, moments, independence); exact streams differ from torch's by design."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from _harness import cuda

pytestmark = pytest.mark.gpu


def _check_xavier(name, w):
    out_f, in_f = w.shape
    bound = math.sqrt(6.0 / (in_f + out_f))
    x = w.double().flatten().numpy()
    n = x.size
    assert np.abs(x).max() <= bound * (1 + 1e-6), (name, np.abs(x).max(), bound)
    sd = bound / math.sqrt(3.0)
    assert abs(x.mean()) <= 5 * sd / math.sqrt(n), (name, "mean", x.mean())
    assert abs(x.var() / sd ** 2 - 1) <= 6 * math.sqrt(0.8 / n) + 1e-3, (name, "var", x.var(), sd ** 2)      # Var(s^2)/sigma^4 = 0.8/n for a uniform
    if n >= 512:
        p = stats.kstest(x / bound, stats.uniform(loc=-1, scale=2).cdf).pvalue
        assert p > 1e-4, (name, "KS vs U(-bound, bound)", p)
        r = np.corrcoef(x[:-1], x[1:])[0, 1]                                                            # neighbours are independent draws
        assert abs(r) <= 5 / math.sqrt(n), (name, "lag-1 correlation", r)


def test_parameter_init_distributions(cuda):
    from distributed_sac_b200.core import CoreConfig, SacCore
    core = SacCore(CoreConfig(replicas=2), 0, seed=1234)           # LunarLander shape
    p0, p1 = core.get_named(replica=0), core.get_named(replica=1)
    n_w = 0
    for k, v in p0.items():
        if k.endswith(".weight"):
            _check_xavier(k, v)
            n_w += 1
            if "_target" not in k:
                assert not torch.equal(v, p1[k]), f"replicas share {k}"                # replica r is seeded seed + r
        elif k.endswith(".bias"):
            assert float(v.abs().max()) == 0.0, (k, "bias must start at zero")
    assert n_w == 15 and float(p0["log_alpha"]) == 0.0
    for q in ("q1", "q2"):                                          # Learner.run() hard-copies local -> target before training
        for i in range(3):
            assert torch.equal(p0[f"{q}.{i}.weight"], p0[f"{q}_target.{i}.weight"])
    assert not torch.equal(p0["q1.1.weight"], p0["q2.1.weight"])    # the twin critics are independent draws
    other = SacCore(CoreConfig(), 0, seed=99).get_named()
    assert not torch.equal(other["actor.1.weight"], p0["actor.1.weight"])
    again = SacCore(CoreConfig(replicas=2), 0, seed=1234).get_named()
    assert all(torch.equal(again[k], p0[k]) for k in p0)            # same seed, same parameters
    core.close()


def test_care_mixture_init_is_standard_normal(cuda):
    from distributed_sac_b200.core import CoreConfig, SacCore
    core = SacCore(CoreConfig(state_dim=39, act_dim=4, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=40, num_tasks=10,
                              care=True, precision=1), 0, seed=7)
    p = core.get_named()
    for k in ("cse.mix.0.W", "cse.mix.1.W", "cse.mix.0.b", "cse.mix.1.b"):
        x = p[k].double().flatten().numpy()
        n = x.size
        assert abs(x.mean()) <= 5 / math.sqrt(n), (k, x.mean())
        assert abs(x.var() - 1) <= 6 * math.sqrt(2.0 / n), (k, x.var())
        if n >= 512:
            assert stats.kstest(x, "norm").pvalue > 1e-4, (k, "KS vs N(0,1)")
    assert p["cse.mix.0.W"].shape == (6, 39, 50)                    # the reference's (K, in, out) layout on export
    for k, v in p.items():
        if (".trunk." in k or ".ctx." in k) and k.endswith(".weight") and k.startswith("cse."):
            _check_xavier(k, v)
        if k.startswith("tse."):
            assert torch.equal(v, p["cse" + k[3:]])                 # target encoder = hard copy
    core.close()


def test_in_kernel_policy_noise_is_standard_normal(cuda):
    """The eps the policy head drew in production mode (eps_next = eps_cur = NULL), read back from what it saved per
    (row, action): N(0,1) marginals, independent across steps / rows / actions / the two rsample() calls, different per
    replica, reproducible per seed."""
    from distributed_sac_b200.core import CoreConfig, Replay, SacCore

    def draw(seed, steps, replicas=1):
        core = SacCore(CoreConfig(replicas=replicas), 0, seed=seed)
        ring = Replay(core, 4096, "device", seed=1)
        ring.fill_synthetic(4096, seed=2)
        out = []
        for _ in range(steps):
            core.step_sampled(ring, 1)
            out.append(torch.stack([core.debug("psave", r).reshape(2 * 256, 2, 8)[:, :, 5] for r in range(replicas)]))
        ring.close(); core.close()
        return torch.stack(out).double().numpy()                    # [steps][replicas][2B][A]

    e = draw(5, 40)
    x = e.reshape(-1)
    n = x.size                                                     # 40 * 512 * 2 = 40 960 draws
    assert abs(x.mean()) <= 5 / math.sqrt(n), x.mean()
    assert abs(x.var() - 1) <= 6 * math.sqrt(2.0 / n), x.var()
    assert abs(stats.kurtosis(x)) <= 6 * math.sqrt(24.0 / n), stats.kurtosis(x)
    assert stats.kstest(x, "norm").pvalue > 1e-4
    assert np.abs(x).max() < 6.5                                   # Box-Muller on (0,1]: finite, tails present
    assert (np.abs(x) > 3).mean() > 0.0015
    lim = 5 / math.sqrt(e[0].size)
    for t in range(1, e.shape[0]):                                 # a step never reuses another step's noise
        assert abs(np.corrcoef(e[t].reshape(-1), e[t - 1].reshape(-1))[0, 1]) <= lim
    flat = e[:, 0]                                                 # [steps][2B][A]
    assert abs(np.corrcoef(flat[:, :, 0].reshape(-1), flat[:, :, 1].reshape(-1))[0, 1]) <= 5 / math.sqrt(flat[:, :, 0].size)   # actions
    assert abs(np.corrcoef(flat[:, :256].reshape(-1), flat[:, 256:].reshape(-1))[0, 1]) <= 5 / math.sqrt(flat[:, :256].size)   # next / current halves
    assert len(np.unique(np.round(x, 7))) > 0.99 * n               # no repeated blocks
    again = draw(5, 3)
    assert np.array_equal(again, e[:3])                             # same seed -> same noise
    two = draw(5, 3, replicas=2)
    assert not np.array_equal(two[:, 0], two[:, 1])                 # replicas draw their own streams
    assert abs(np.corrcoef(two[:, 0].reshape(-1), two[:, 1].reshape(-1))[0, 1]) <= 5 / math.sqrt(two[:, 0].size)
