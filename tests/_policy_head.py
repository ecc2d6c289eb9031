"""The tanh-Gaussian policy head restated point by point, for the tests of policy_point / policy_dout_point
(sac_kernels.cuh): an fp32 restatement in the kernels' operation order, the reference's formula
(sac_port.policy_sample) in fp64 autograd, the error bounds that follow from the conditioning of each point, and the
edge heads that put the head's action columns at the clamp, its boundaries, saturated tanh and infinities."""
import math

import numpy as np
import torch

import sac_port as sp

F32 = np.float32
ULP = 2.0 ** -24                      # unit roundoff of fp32
LN_SQRT_2PI = F32(0.91893853320467274178)
SAVE = ("std", "diff", "t", "act", "jac", "eps", "mask", "logp_j")     # psave entries 0..7


def _r64(f, x):
    """f evaluated in fp64 and rounded once to fp32, like exp_f64r / tanh_f64r / log_f64r; and whether the fp64 value lies
    within two double ulps of an fp32 rounding midpoint (the device's and the host's libm may round such a value apart)."""
    with np.errstate(all="ignore"):
        v = f(x.astype(np.float64))
        r = v.astype(F32)
        nxt = np.nextafter(r, np.where(v > r.astype(np.float64), F32(np.inf), F32(-np.inf)))
        mid = (r.astype(np.float64) + nxt.astype(np.float64)) / 2
        near = np.isfinite(v) & np.isfinite(mid) & (np.abs(v - mid) <= 2 * np.spacing(np.abs(v)))
    return r, near


def restate_point(mu, raw, eps, k):
    """policy_point: {psave name: fp32 array} plus "logstd" and "near" (elements with a transcendental near a midpoint).
    Every +, -, *, / rounds once to fp32 (numpy float32 arithmetic; the library is built with -fmad=false)."""
    mu, raw, eps, k = (np.asarray(x, F32) for x in (mu, raw, eps, k))
    with np.errstate(all="ignore"):
        ls = np.where(raw < F32(-20), F32(-20), np.where(raw > F32(2), F32(2), raw))
        mask = ((raw >= F32(-20)) & (raw <= F32(2))).astype(F32)
        std, n1 = _r64(np.exp, ls)
        u = mu + std * eps
        t, n2 = _r64(np.tanh, u)
        act = k * t
        diff = u - mu
        var = std * std
        logstd, n3 = _r64(np.log, std)
        gauss = -(diff * diff) / (F32(2) * var) - logstd - LN_SQRT_2PI
        q = act / k
        jac = k * (F32(1) - q * q + F32(1e-6))
        lj, n4 = _r64(np.log, jac)
        logp_j = gauss - lj
    return dict(std=std, diff=diff, t=t, act=act, jac=jac, eps=eps, mask=mask, logp_j=logp_j, logstd=logstd,
                near=n1 | n2 | n3 | n4)


def restate_dout(sv, da, alpha, c_loss, k):
    """policy_dout_point from the saved values sv [..., 8] (psave layout): (dmu, dls)."""
    sv = np.asarray(sv, F32)
    std, diff, t, act, jac, eps, mask = (sv[..., i] for i in range(7))
    da, alpha, c_loss, k = (np.asarray(x, F32) for x in (da, alpha, c_loss, k))
    with np.errstate(all="ignore"):
        glp = c_loss * alpha
        var = std * std
        d_act = da + glp * (F32(2) * (act / k) / k) * k / jac
        g_u_t = d_act * k * (F32(1) - t * t)
        g_u = g_u_t + glp * (-diff / var)
        dmu = g_u + glp * (diff / var)
        dstd = g_u * eps + glp * ((diff * diff) / (var * std) - F32(1) / std)
        dls = np.where(mask != 0, dstd * std, F32(0))
    return dmu, dls


def row_sum(x):
    """Sum over the last axis in index order, in fp32 (the head's per-row log-prob)."""
    x = np.asarray(x, F32)
    tot = np.zeros(x.shape[:-1], F32)
    for j in range(x.shape[-1]):
        tot = tot + x[..., j]
    return tot


def reference64(mu, raw, eps, da, glp, k):
    """sac_port.policy_sample's formula in fp64 autograd at the head output [mu | raw] (an actor without layers), with the
    loss sum(da * action) + sum(glp_row * logp_row) whose gradient the step feeds the head.  Returns (action, logp per row,
    log_std, dmu, dls) as float64 numpy arrays."""
    A = mu.shape[-1]
    spec = sp.SacSpec(act_dim=A, action_scale=float(k))
    head = torch.from_numpy(np.concatenate([mu, raw], -1).astype(np.float64)).requires_grad_(True)
    act, logp, log_std = sp.policy_sample(spec, {}, head, torch.from_numpy(np.asarray(eps, np.float64)))
    loss = (torch.from_numpy(np.asarray(da, np.float64)) * act).sum() + (torch.from_numpy(np.asarray(glp, np.float64)) *
                                                                         logp[:, 0]).sum()
    loss.backward()
    g = head.grad.numpy()
    return act.detach().numpy(), logp[:, 0].detach().numpy(), log_std.detach().numpy(), g[:, :A], g[:, A:]


def bounds(p, mu, da, glp, k):
    """First-order error bounds of one fp32 evaluation against the fp64 value, per element, from the fp32 point p
    ({psave name: array}: restate_point's dict or the device's psave) and its mu: (act, logp_j, dmu, dls).  Each
    collects, in units of the fp32 unit roundoff, the magnitudes of the terms that are rounded, and the sensitivities of
    the result to the rounding of u, of tanh(u) and of the Jacobian term where tanh saturates."""
    e = ULP
    std, diff, t, act, jac, eps, mask = (np.asarray(p[n], np.float64) for n in SAVE[:7])
    glp = np.asarray(glp, np.float64)[..., None] * np.ones_like(std)
    da = np.asarray(da, np.float64)
    mu_abs = np.abs(np.asarray(mu, np.float64))
    with np.errstate(all="ignore"):
        var = std * std
        omt = 1.0 - t * t
        J = omt + 1e-6
        du = 3 * e * (mu_abs + np.abs(std * eps))                 # u = mu + std * eps: std, the product and the sum
        diff = np.maximum(np.abs(diff), np.abs(std * eps))        # u - mu as rounded can be 0 where std * eps is not
        dt = omt * du + 2 * e * np.abs(t)                         # tanh(u): through u, and its own rounding
        b_act = k * dt + 2 * e * np.abs(act)
        b_lp = ((diff * du + du * du) / var + 8 * e * (diff * diff / (2 * var) + 22 + np.abs(np.log(jac)))
                + 2 * np.abs(t) / J * (dt + 4 * e))
        d_act = da + glp * 2 * (act / k) / jac
        dd = glp * (2 / (k * J) + 4 * t * t / (k * J * J))        # d(d_act)/dt
        b_gut = (8 * e * np.abs(d_act * k * omt) + np.abs(d_act * k) * (2 * np.abs(t) * dt + 4 * e)
                 + k * omt * (dd * (dt + 4 * e) + 8 * e * np.abs(glp * 2 * t / jac)))
        big = glp * np.abs(diff) / var
        b_mu = b_gut + 16 * e * big
        g_u = np.abs(d_act * k * omt) + big
        b_ls = mask * (np.abs(eps) * std * (b_gut + 8 * e * big) + 2 * glp * np.abs(eps) / std * du
                       + 8 * e * (g_u * np.abs(eps) * std + glp * (diff * diff / var + 1)))
    return b_act, b_lp, b_mu, b_ls


# ---------------------------------------------------------------------------------------------------------------------
# edge heads
# ---------------------------------------------------------------------------------------------------------------------
LO, HI = F32(-20.0), F32(2.0)
BOUNDS = {"at_lo": LO, "at_hi": HI, "below_lo": np.nextafter(LO, F32(-np.inf)), "above_hi": np.nextafter(HI, F32(np.inf))}
# regimes of one action column: the head as _params makes it; raw log-std spread over [3, 39] (clamped high) or [-58, -22]
# (clamped low); raw exactly at a clamp bound or the float beyond it (weight row zero); mu spread over [-30, 30] (tanh
# saturated: 1 - t^2 loses its bits, and t == +-1 exactly); raw +-inf; raw NaN
REGIMES = ("nominal", "high", "low", *BOUNDS, "sat", "+inf", "-inf")
OUTSIDE = ("high", "low", "below_lo", "above_hi", "+inf", "-inf")          # raw outside [-20, 2] on every row


def _spread(w, h, lo, hi):
    """(w', b') with h @ w' + b' spread over [lo, hi]: w scaled and shifted."""
    z = h @ w.astype(np.float64)
    c, half = (z.max() + z.min()) / 2, max((z.max() - z.min()) / 2, 1e-3)
    s = (hi - lo) / 2 / half
    return (w * s).astype(F32), F32((lo + hi) / 2 - s * c)


def edge_head(W, b, h, regimes):
    """The head weight [2A][H] and bias [2A] with action column j put in regimes[j]; h: the last hidden activations
    [rows][H] the head will see.  Only the rows of the columns a regime touches change."""
    W, b = np.array(W, F32), np.array(b, F32)
    A = W.shape[0] // 2
    h = np.asarray(h, np.float64)
    for j, reg in enumerate(regimes):
        r = A + j
        if reg == "high":
            W[r], b[r] = _spread(W[r], h, 3.0, 39.0)
        elif reg == "low":
            W[r], b[r] = _spread(W[r], h, -58.0, -22.0)
        elif reg in BOUNDS or reg in ("+inf", "-inf", "nan"):
            W[r] = 0
            b[r] = BOUNDS[reg] if reg in BOUNDS else F32({"+inf": np.inf, "-inf": -np.inf, "nan": np.nan}[reg])
        elif reg == "sat":
            W[j], b[j] = _spread(W[j], h, -30.0, 30.0)
        else:
            assert reg == "nominal", reg
    return torch.from_numpy(W), torch.from_numpy(b)


def rotation(A, i):
    """The regimes of the A action columns in rotation i: consecutive entries of REGIMES, so that ceil(len / A)
    rotations put every regime on some column."""
    return [REGIMES[(i * A + j) % len(REGIMES)] for j in range(A)]
