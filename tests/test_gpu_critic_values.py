"""GPU: critic inference (b200sac_critic_values; include/b200sac.h).

  1  q1 / q2 and their targets against the oracle MLP (oracle/refresh_ref.py) at the parity bar, at the LL, VS and MS
     shapes, precision 0 and 1, plain, critic_ln and critic_dropout critics, for n in {1, 7, batch, chunk + 1,
     3 chunk + 5} from host and device memory; eval mode: a dropout rate of 0.5 gives the values of 0 bit for bit;
  2  replica 1 of an R = 3 handle against the oracle and bit for bit against an R = 1 handle with the same parameters;
  3  every row's values bit-identical whatever n is and wherever the row sits;
  4  steps with critic_values calls between them end bit-identical to the same steps without them, and the plan does
     not change.
"""
import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import refresh_ref as rr
import sac_port as sp
from _golden import core_config
from _harness import plan_labels

pytestmark = pytest.mark.gpu

PARAMS = 0
SPECS = {"LL": sp.ll_spec, "VS": sp.vs_spec, "MS": sp.ms_spec}
BAR = 1e-4


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_sac_b200 import _lib
    _lib.load()
    return torch.device("cuda", 0)


def _core(spec, precision=0, replicas=1, mode="plain", seed=0):
    from distributed_sac_b200.core import SacCore
    kw = dict(critic_layer_norm=mode != "plain", critic_dropout=mode == "droq")
    return SacCore(core_config(spec, replicas=replicas, precision=precision, **kw), 0, seed=seed)


def _params(spec, seed, ln=False):
    """Xavier weights, small random biases, targets moved off the locals, LayerNorm weights near 1."""
    p = (lnp if ln else sp).init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in p:
        if k.endswith(".ln.weight"):
            p[k] = 1.0 + 0.1 * torch.randn(p[k].shape, generator=g)
        elif k.endswith(".bias"):
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
        elif "_target." in k:
            p[k] = p[k] + 0.02 * torch.randn(p[k].shape, generator=g)
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


def _rows(spec, n, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(n, spec.state_dim, generator=g)
    if spec.num_tasks:
        s = torch.cat([s, torch.nn.functional.one_hot(torch.randint(0, spec.num_tasks, (n,), generator=g), spec.num_tasks)
                       .float()], 1)
    return s, torch.rand(n, spec.act_dim, generator=g) * 2 - 1


def _check(got, ref, what):
    got, ref = np.asarray(got), np.asarray(ref)
    err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= BAR, f"{what}: max error {err:.3g} over the parity bar"


@pytest.mark.parametrize("mode", ["plain", "ln", "droq"])
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("shape", ["LL", "VS", "MS"])
def test_matches_the_oracle(cuda, shape, precision, mode):
    spec = SPECS[shape]()
    core = _core(spec, precision, mode=mode)
    p = _params(spec, 3, ln=mode != "plain")
    core.set_named(p, PARAMS)
    chunk = core.critic_values_chunk()
    assert chunk % 32 == 0 and 32 <= chunk <= 65536
    big_s, big_a = _rows(spec, 3 * chunk + 5, 7)
    refs = {t: rr.critic_values(p, big_s, big_a, t) for t in (False, True)}
    for k, n in enumerate((1, 7, spec.batch, chunk + 1, 3 * chunk + 5)):
        s, a = big_s[:n], big_a[:n]
        if k % 2:
            s, a = s.cuda(), a.cuda()
        for target in (False, True):
            q1, q2 = core.critic_values(s, a, target=target)
            assert q1.device == s.device and q1.shape == (n,)
            _check(q1.cpu(), refs[target][0][:n], f"{shape} p{precision} {mode} n={n} target={target} q1")
            _check(q2.cpu(), refs[target][1][:n], f"{shape} p{precision} {mode} n={n} target={target} q2")
    if mode == "droq":          # eval mode: no dropout at any rate
        s, a = big_s[:chunk + 1], big_a[:chunk + 1]
        q0 = core.critic_values(s, a)
        core.set_critic_dropout(0.5)
        q5 = core.critic_values(s, a)
        assert all(torch.equal(x, y) for x, y in zip(q0, q5))


def test_replica_of_a_three_replica_handle(cuda):
    spec = sp.ll_spec()
    three, one = _core(spec, replicas=3), _core(spec)
    ps = [_params(spec, 10 + r) for r in range(3)]
    for r in range(3):
        three.set_named(ps[r], PARAMS, replica=r)
    one.set_named(ps[1], PARAMS)
    s, a = _rows(spec, 1000, 4)
    for target in (False, True):
        got = three.critic_values(s, a, target=target, replica=1)
        ref = rr.critic_values(ps[1], s, a, target)
        _check(got[0], ref[0], "replica 1 q1")
        _check(got[1], ref[1], "replica 1 q2")
        assert all(torch.equal(x, y) for x, y in zip(got, one.critic_values(s, a, target=target)))
        assert not torch.equal(got[0], three.critic_values(s, a, target=target, replica=0)[0])


@pytest.mark.parametrize("mode", ["plain", "ln"])
def test_rows_do_not_depend_on_the_call(cuda, mode):
    spec = sp.vs_spec()
    core = _core(spec, mode=mode)
    core.set_named(_params(spec, 5, ln=mode != "plain"), PARAMS)
    chunk = core.critic_values_chunk()
    s, a = _rows(spec, 2 * chunk + 3, 8)
    full = core.critic_values(s, a)
    for lo, hi in ((0, 1), (5, 12), (chunk - 2, chunk + 3), (2 * chunk, 2 * chunk + 3)):
        part = core.critic_values(s[lo:hi], a[lo:hi])
        assert all(torch.equal(x, y[lo:hi]) for x, y in zip(part, full)), (lo, hi)
    perm = torch.randperm(len(s), generator=torch.Generator().manual_seed(0))
    shuffled = core.critic_values(s[perm], a[perm])
    assert all(torch.equal(x, y[perm]) for x, y in zip(shuffled, full))


@pytest.mark.parametrize("mode", ["plain", "droq"])
def test_steps_do_not_see_the_calls(cuda, mode):
    spec = sp.SacSpec(state_dim=8, act_dim=2, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=64)
    a, b = _core(spec, mode=mode, seed=4), _core(spec, mode=mode, seed=4)
    if mode == "droq":
        a.set_critic_dropout(0.2)
        b.set_critic_dropout(0.2)
    launches = a.launches_per_step
    s, act = _rows(spec, 300, 9)
    for i in range(6):
        batch = [t.unsqueeze(0).cuda() for t in sp.synthetic_batch(spec, seed=50 + i)]
        a.critic_values(s, act, target=bool(i % 2))
        a.step(*batch)
        b.step(*batch)
    assert torch.equal(a.read_losses(6), b.read_losses(6))
    for w in (0, 1, 2):
        assert torch.equal(a.export_arena(w), b.export_arena(w))
    from distributed_sac_b200 import _lib
    import ctypes as C
    n = C.c_int32(0)
    _lib.check(a.lib.b200sac_launches_per_step(a._h, C.byref(n)))
    assert n.value == launches
    assert plan_labels(a) == plan_labels(b)
