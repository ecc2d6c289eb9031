"""The tanh-Gaussian policy head (policy_point / policy_dout_point, sac_kernels.cuh) at the edges of its domain, on every site
that evaluates it: the layer-chained head and policy backward (chain_kernel), policy_head_kernel with the in-kernel
policy backward of head_bwd_kernel (fp32, with and without row slices, and at precision 1), policy_dout_kernel, both CARE
variants, and b200sac_act in its four modes.

Edge heads (tests/_policy_head.py) overwrite only the head layer, so the hidden layers stay as _params makes them.  Each
action column is put in one regime -- the head as it is, raw log-std clamped high or low, exactly at a clamp bound or the
float beyond it, mu saturating tanh, raw +-inf -- and the columns rotate through the regimes over a few steps, at action
scales 1 and 1.5.

1. Bit for bit against the fp32 restatement, from the head output the step computed (debug "head"), the noise it used
   and the d(action) it read: all eight saved values, the actions, the log-probabilities and d(mu | log_std).  The only
   difference allowed is an element whose fp64 transcendental lies next to an fp32 rounding midpoint (counted; none are
   expected).
2. Against the reference's formula in fp64 (sac_port.policy_sample in autograd) within bounds that follow from each
   point's conditioning, and d(log_std) exactly 0 iff the raw log-std is outside [-20, 2] (+-inf included; the bounds
   themselves keep their gradient, as torch.clamp's backward does).  This catches a wrong sign or a misplaced action scale
   that the restatement, copied from the kernel, would share.
3. Whole steps against the autograd oracle at three replicas with one well-conditioned regime each (clamped high, the
   clamp bounds, saturated tanh with the CUDA tanh forced), and the parameters of fully clamped columns unchanged bit for
   bit after a first step from zero Adam moments.  Clamped low is left to 1 and 2: there d(mu) is the difference of two
   terms of size c alpha |eps| / std, 10^6-10^8 times the result, so the oracle's own fp32 value is rounding noise.
4. A NaN raw log-std: the step's losses, actions, log-probabilities and parameters are NaN exactly where the oracle's are,
   and act returns NaN in that column (torch.clamp propagates NaN).
"""
import dataclasses

import numpy as np
import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import CareCase, check_forced, check_port_state, cuda_relu_masks, sync_core_to_port
from _harness import (CARE_ROW_OUTPUTS, LAYER_CASES, LL, PARAMS, ROW_OUTPUTS, _core, _params, _tasks, check_active,
                      check_losses, check_rows, cuda)
from _policy_head import BOUNDS, OUTSIDE, REGIMES, SAVE, bounds, edge_head, reference64, restate_dout, restate_point, \
    rotation, row_sum

gpu = pytest.mark.gpu
F32 = np.float32

# id -> (SacSpec fields or CARE fixture, care, precision)
SITES = {
    "chained": (LL, False, 0),                             # chain_kernel<FWD> head, chain_kernel<BWD> policy backward
    "layer_fp32": (LAYER_CASES["odd67"], False, 0),        # policy_head_kernel, head_bwd_kernel in policy mode
    "pdout257": (LAYER_CASES["pdout257"], False, 0),       # policy_dout_kernel
    "split517": (LAYER_CASES["split517"], False, 0),       # head_bwd_kernel in policy mode with row slices
    "in45_tc": (LAYER_CASES["in45"], False, 1),            # precision 1
    "care_m": ("care_small_s4", True, 1),
    "care_o": ("care_o_small_s4", True, 1),
}
MODES = ("eps", "det", "mu", "fresh")          # injected noise, k tanh(mu), k mu, fresh Philox noise


def site_spec(name, k):
    fields, care, precision = SITES[name]
    spec = CareCase(fields).spec if care else sp.SacSpec(**fields)
    return dataclasses.replace(spec, action_scale=k), care, precision


def _head_names(spec):
    La = len(spec.actor_hidden)
    return f"actor.{La}.weight", f"actor.{La}.bias"


def _act(core, obs, mode, eps):
    return core.act(obs, stochastic=mode in ("eps", "fresh"), eps=eps, no_tanh=(mode == "mu"))


def _bits_equal(got, want):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    return (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))


# ---------------------------------------------------------------------------------------------------------------------
# the device runs of tests 1 and 2: one per site and action scale, shared by both tests
# ---------------------------------------------------------------------------------------------------------------------
_RUNS = {}


def site_run(name, k):
    """Every rotation of the edge regimes as one step of a handle (head, psave, actions, log-probs, d(action), d_head)
    and act calls in every mode at n = 7 and the largest n the handle accepts (head, psave, actions, log-probs)."""
    if (name, k) in _RUNS:
        return _RUNS[(name, k)]
    spec, care, precision = site_spec(name, k)
    B, A, La = spec.batch, spec.act_dim, len(spec.actor_hidden)
    mod = cp if care else sp
    core = _core(spec, care, precision)
    p = _params(spec, 7, care)
    wn, bn = _head_names(spec)
    batch = mod.synthetic_batch(spec, seed=21)
    gen = torch.Generator().manual_seed(22)
    e1, e2 = torch.randn(B, A, generator=gen), torch.randn(B, A, generator=gen)
    core.set_named(p, PARAMS)
    core.step(*batch, e1, e2)
    h = core.debug(f"hA.{La - 1}").reshape(2 * B, -1).numpy()        # what the head sees (the head does not change it)
    alpha = np.exp(p["log_alpha"].numpy().astype(np.float64)).astype(F32)[_tasks(spec, batch[0])]
    run = dict(spec=spec, alpha=alpha, c=F32(1.0 / B / (B if spec.weighted_loss else 1)), steps=[], acts=[])
    obs = batch[0] if care else torch.cat([batch[0], batch[3]])
    nmax = B if care else 2 * B
    for i in range(-(-len(REGIMES) // A)):
        regs = rotation(A, i)
        W, b = edge_head(p[wn], p[bn], h, regs)
        core.set_named({**p, wn: W, bn: b}, PARAMS)
        core.step(*batch, e1, e2)
        d = lambda n: core.debug(n).numpy()
        run["steps"].append(dict(regs=regs, head=d("head").reshape(2 * B, 2 * A), psave=d("psave").reshape(2 * B, A, 8),
                                 a=np.concatenate([d("a_next"), d("a_cur")]).reshape(2 * B, A),
                                 logp=np.concatenate([d("logp_next"), d("logp_cur")]), da=d("d_action").reshape(B, A),
                                 d_head=d("d_head").reshape(B, 2 * A)))
        for n in (7, nmax):
            for mode in MODES:
                eps = torch.randn(n, A, generator=gen) if mode == "eps" else None
                a = _act(core, obs[:n], mode, eps).numpy()
                run["acts"].append(dict(regs=regs, mode=mode, n=n, a=a, head=d("head")[:n * 2 * A].reshape(n, 2 * A),
                                        psave=d("psave")[:n * A * 8].reshape(n, A, 8),
                                        logp=np.concatenate([d("logp_next"), d("logp_cur")])[:n]))
    core.close()
    _RUNS[(name, k)] = run
    return run


# ---------------------------------------------------------------------------------------------------------------------
# 1: bit for bit against the fp32 restatement
# ---------------------------------------------------------------------------------------------------------------------
class Exact:
    def __init__(self, what):
        self.what, self.bad, self.near, self.n = what, [], 0, 0

    def __call__(self, tag, got, want, near):
        ok = _bits_equal(got, want)
        self.n += ok.size
        self.near += int((~ok & near).sum())
        miss = ~ok & ~near
        if miss.any():
            i = tuple(int(x) for x in np.argwhere(miss)[0])
            self.bad.append(f"{tag}: {int(miss.sum())} of {miss.size} differ, first {list(i)} got {np.asarray(got)[i]!r} "
                            f"want {np.asarray(want)[i]!r}")


def check_point(ex, tag, head, ps, k, a=None, logp=None, mode=None):
    """psave, actions and log-probs of rows whose head output was `head` against the restatement."""
    A = ps.shape[1]
    mu, raw = head[:, :A], head[:, A:]
    r = restate_point(mu, raw, ps[..., 5], k)
    near = r["near"]
    for i, n in enumerate(SAVE):
        ex(f"{tag} psave.{n}", ps[..., i], r[n], near)
    if a is not None:
        ex(f"{tag} action", a, F32(k) * mu if mode == "mu" else r["act"], near & (mode != "mu"))
    if logp is not None:
        ex(f"{tag} log-prob", logp, row_sum(r["logp_j"]), near.any(-1))
    return r


@gpu
@pytest.mark.parametrize("k", [1.0, 1.5])
@pytest.mark.parametrize("site", list(SITES))
def test_head_matches_fp32_restatement_bit_for_bit(cuda, site, k):
    run = site_run(site, k)
    B = run["spec"].batch
    ex = Exact(f"{site} k {k}")
    seen = dict(clamped=0, at_lo=0, at_hi=0, t_one=0, t_band=0, inf=0)
    for st in run["steps"]:
        tag = f"regimes {st['regs']}"
        r = check_point(ex, tag, st["head"], st["psave"], k, st["a"], st["logp"])
        dmu, dls = restate_dout(st["psave"][B:], st["da"], run["alpha"][:, None], run["c"], k)
        none = np.zeros(dmu.shape, bool)
        ex(f"{tag} d(mu)", st["d_head"][:, :dmu.shape[1]], dmu, none)
        ex(f"{tag} d(log_std)", st["d_head"][:, dmu.shape[1]:], dls, none)
        raw, t = st["head"][:, dmu.shape[1]:], r["t"]
        seen["clamped"] += int((r["mask"] == 0).sum())
        seen["at_lo"] += int((raw == BOUNDS["at_lo"]).sum())
        seen["at_hi"] += int((raw == BOUNDS["at_hi"]).sum())
        seen["t_one"] += int((np.abs(t) == 1).sum())
        seen["t_band"] += int(((1 - t * t > 0) & (1 - t * t < 1e-4)).sum())
        seen["inf"] += int(np.isinf(raw).sum())
    for ac in run["acts"]:
        check_point(ex, f"act {ac['mode']} n {ac['n']} regimes {ac['regs']}", ac["head"], ac["psave"], k, ac["a"],
                    ac["logp"], ac["mode"])
    assert not ex.bad, f"{ex.what}: " + "; ".join(ex.bad[:6])
    assert all(v > 0 for v in seen.values()), f"{ex.what}: a regime was not reached: {seen}"
    print(f"[exact] {ex.what}: {ex.n} values bit for bit, {ex.near} differ next to an fp32 rounding midpoint; {seen}")


# ---------------------------------------------------------------------------------------------------------------------
# 2: against the reference's formula in fp64
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("k", [1.0, 1.5])
@pytest.mark.parametrize("site", list(SITES))
def test_head_matches_fp64_reference_within_its_conditioning(cuda, site, k):
    run = site_run(site, k)
    spec = run["spec"]
    B, A = spec.batch, spec.act_dim
    glp = (run["c"] * run["alpha"]).astype(F32)
    bad = []

    def within(tag, got, ref, bound):
        dev = np.abs(np.asarray(got, np.float64) - ref)
        miss = ~(dev <= bound)
        if miss.any():
            i = tuple(int(x) for x in np.argwhere(miss)[0])
            bad.append(f"{tag}: {int(miss.sum())} of {miss.size} beyond the bound, first {list(i)} got {np.asarray(got)[i]!r} "
                       f"ref {ref[i]!r} bound {bound[i]:.3g}")

    records = [(f"step regimes {st['regs']}", st["head"], st["psave"], st["a"], st["logp"], st) for st in run["steps"]]
    records += [(f"act {ac['mode']} n {ac['n']} regimes {ac['regs']}", ac["head"], ac["psave"], ac["a"], ac["logp"], None)
                for ac in run["acts"] if ac["mode"] != "mu"]
    for tag, head, ps, a, logp, st in records:
        n = head.shape[0]
        mu, raw, eps = head[:, :A], head[:, A:], ps[..., 5]
        p = {name: ps[..., i] for i, name in enumerate(SAVE)}
        da, g = (st["da"], glp) if st is not None else (np.zeros((0, A), F32), glp[:0])
        rows = slice(B, 2 * B) if st is not None else slice(n, n)
        fwd = reference64(mu, raw, eps, np.zeros((n, A)), np.zeros(n), k)
        b_act, b_lp, _, _ = bounds(p, mu, np.zeros((n, A)), np.zeros(n), k)
        within(f"{tag} action", a, fwd[0], 2 * b_act + 1e-6 * np.abs(fwd[0]))
        within(f"{tag} log-prob", logp, fwd[1], 2 * b_lp.sum(-1) + 1e-6 * np.abs(fwd[1]))
        if st is None:
            continue
        sub = {name: v[rows] for name, v in p.items()}
        _, _, _, dmu64, dls64 = reference64(mu[rows], raw[rows], eps[rows], da, g, k)
        _, _, b_mu, b_ls = bounds(sub, mu[rows], da, g, k)
        within(f"{tag} d(mu)", st["d_head"][:, :A], dmu64, 2 * b_mu)
        within(f"{tag} d(log_std)", st["d_head"][:, A:], dls64, 2 * b_ls)
        inside = (raw[rows] >= -20) & (raw[rows] <= 2)
        zero = st["d_head"][:, A:] == 0
        if not np.array_equal(zero, ~inside):
            i = tuple(int(x) for x in np.argwhere(zero != ~inside)[0])
            bad.append(f"{tag}: d(log_std) at raw {raw[rows][i]!r} is {st['d_head'][:, A:][i]!r}: zero iff raw is outside "
                       f"[-20, 2]")
        assert np.array_equal(dls64 == 0, ~inside)
    assert not bad, f"{site} k {k}: " + "; ".join(bad[:6])


# ---------------------------------------------------------------------------------------------------------------------
# 3: whole steps against the autograd oracle, three replicas with one regime each
# ---------------------------------------------------------------------------------------------------------------------
STEP_REGIMES = ("high", "bounds", "sat")


def step_regimes(regime, A, i):
    """Column regimes of a replica in step i: the regime on the even columns, the head as it is on the odd ones; "bounds"
    puts every column at a clamp bound or the float beyond it, rotating with the step."""
    if regime == "bounds":
        return [list(BOUNDS)[(i * A + j) % len(BOUNDS)] for j in range(A)]
    return [regime if j % 2 == 0 else "nominal" for j in range(A)]


@gpu
@pytest.mark.parametrize("site", list(SITES))
def test_edge_step_matches_oracle(cuda, site):
    spec, care, precision = site_spec(site, 1.5)
    B, A, La, R = spec.batch, spec.act_dim, len(spec.actor_hidden), len(STEP_REGIMES)
    mod = cp if care else sp
    wn, bn = _head_names(spec)
    ports = [(cp.CarePortLearner if care else sp.PortLearner)(spec, _params(spec, 11 + 7 * r, care)) for r in range(R)]
    core = _core(spec, care, precision, R)
    gen = torch.Generator().manual_seed(5)
    for i in range(2):
        batches = [mod.synthetic_batch(spec, seed=100 * i + r) for r in range(R)]
        eps = [(torch.randn(B, A, generator=gen), torch.randn(B, A, generator=gen)) for _ in range(R)]
        inputs = [torch.stack([b[j] for b in batches]) for j in range(5)] + [torch.stack([e[j] for e in eps]) for j in (0, 1)]
        for r in range(R):
            sync_core_to_port(core, ports[r], r)
        core.step(*inputs)                                # the last hidden activations the head will see
        regs, head = [], []
        for r in range(R):
            h = core.debug(f"hA.{La - 1}", r).reshape(2 * B, -1).numpy()
            regs.append(step_regimes(STEP_REGIMES[r], A, i))
            W, b = edge_head(ports[r].p[wn].detach(), ports[r].p[bn].detach(), h, regs[r])
            ports[r].p[wn].data.copy_(W)
            ports[r].p[bn].data.copy_(b)
            head.append((W, b))
            sync_core_to_port(core, ports[r], r)
        core.step(*inputs)
        for r in range(R):
            what = f"{site} step {i} replica {r} ({regs[r]}): "
            forced = cuda_relu_masks(core, spec, r, care)
            with sp.ReluTape(forced) as tape:
                o = (ports[r].update if care else ports[r].update_SAC)(*batches[r], *eps[r], want_intermediates=True)
            check_forced(tape, forced, what)
            check_active(core, spec, r, what, care)
            check_losses(core, o, r, what)
            check_port_state(core, ports[r], replica=r)
            check_rows(core, spec, o, r, what, outputs=CARE_ROW_OUTPUTS if care else ROW_OUTPUTS)
            if i == 0:                                    # zero gradient from zero Adam moments: p' == p exactly
                got = core.get_named(PARAMS, r)
                for j in (j for j, g in enumerate(regs[r]) if g in OUTSIDE):
                    W, b = head[r]
                    assert torch.equal(got[bn][A + j], b[A + j]) and torch.equal(got[wn][A + j], W[A + j]), \
                        f"{what}the clamped column {j}'s log-std parameters moved"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: a NaN raw log-std propagates, as through torch.clamp
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("site", list(SITES))
def test_nan_log_std_propagates_like_the_oracle(cuda, site):
    spec, care, precision = site_spec(site, 1.5)
    B, A = spec.batch, spec.act_dim
    mod = cp if care else sp
    wn, bn = _head_names(spec)
    p = _params(spec, 7, care)
    p[bn] = p[bn].clone()
    p[bn][A] = float("nan")                               # action column 0's log-std
    port = (cp.CarePortLearner if care else sp.PortLearner)(spec, p)
    core = _core(spec, care, precision)
    sync_core_to_port(core, port)
    batch = mod.synthetic_batch(spec, seed=31)
    obs = batch[0]
    for mode in MODES:
        a = _act(core, obs, mode, torch.randn(B, A) if mode == "eps" else None)
        assert torch.isfinite(a[:, 1:]).all(), f"{site} act {mode}"
        if mode == "mu":                                  # k mu does not read the log-std
            assert torch.isfinite(a[:, 0]).all(), f"{site} act {mode}"
        else:
            assert torch.isnan(a[:, 0]).all(), f"{site} act {mode}: a NaN log-std gave finite actions {a[:4, 0].tolist()}"
    gen = torch.Generator().manual_seed(32)
    e1, e2 = torch.randn(B, A, generator=gen), torch.randn(B, A, generator=gen)
    core.step(*batch, e1, e2)
    o = (port.update if care else port.update_SAC)(*batch, e1, e2, want_intermediates=True)
    L = core.read_losses(1)[0, 0]
    for i, key in enumerate(("critic_loss", "actor_loss", "alpha_loss", "entropy")):
        assert bool(torch.isnan(L[i])) == (o[key] != o[key]), f"{site} {key}: {float(L[i])} vs oracle {o[key]}"
    for key in ("a_next", "a_cur", "logp_next", "logp_cur"):
        ref = o[key].reshape(B, -1)
        got = core.debug(key).reshape(ref.shape)
        assert torch.equal(torch.isnan(got), torch.isnan(ref)), f"{site} {key}: NaN pattern differs from the oracle's"
    got, ref = core.get_named(PARAMS), port.params()
    names = [k for k in ref if k in got]
    assert {k for k in ref if k.startswith(("actor.", "q1.", "q2."))} <= set(names)
    bad = [k for k in names if not torch.equal(torch.isnan(got[k]), torch.isnan(ref[k].reshape(got[k].shape)))]
    assert not bad, f"{site}: NaN pattern of {bad[:8]} differs from the oracle's"
    core.close()
