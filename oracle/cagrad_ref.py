"""CAGrad reference (Liu et al., "Conflict-Averse Gradient Descent for Multi-task Learning", NeurIPS 2021) for the pcgrad
step plan's CAGrad mode (b200sac_set_cagrad).

Three pieces:
  solve           the restatement of include/b200sac.h's definition in the kernel's order of operations
                  (pcgrad_kernels.cuh, cagrad_solve): every sum over tasks in the kernel's fixed reduction tree, every
                  sum inside a task's value serial, no fused multiply-add;
  literal         the same dual solved with torch autograd and torch.optim.SGD (momentum 0.5) at fp64;
  cagrad_update   one whole step of a sac_port.PortLearner with CAGrad on the critic and actor optimizers.
"""
import math

import numpy as np
import torch

import pcgrad_ref as pr
import sac_port as sp

ITERS = 20


def _width(T):
    """The padded width n of the device's reduction tree: one warp's 32 lanes, two tasks per lane above T = 32."""
    return 32 if T <= 32 else 64


def _tree(v, op, pad):
    """op-reduction of v (length T) in the device's fixed tree (pcgrad_kernels.cuh, cag_tsum / cag_tmax): v padded with
    `pad` to n, for n = 64 first s_l = op(v_l, v_{l+32}), then s_l = op(s_l, s_{l xor o}) for o = 16, 8, 4, 2, 1;
    the result is lane 0's."""
    v = np.asarray(v, np.float64)
    n = _width(len(v))
    full = np.full(n, pad)
    full[:len(v)] = v
    s = op(full[:32], full[32:]) if n == 64 else full
    w = min(n, 32)
    o = w // 2
    while o >= 1:
        s = op(s, s[np.arange(w) ^ o])
        o //= 2
    return float(s[0])


def _tsum(v):
    return _tree(v, np.add, 0.0)


def _tmax(v):
    return _tree(v, np.fmax, -np.inf)


def _scale(G):
    T = G.shape[0]
    with np.errstate(invalid="ignore"):
        s = _tsum(np.sqrt(np.diag(G))) / T
    degenerate = not np.isfinite(G).all() or not s > 0 or math.isinf(s)
    return s, degenerate


def _degenerate(T, s):
    nan = float("nan")
    return dict(w=np.ones(T), w32=np.ones(T, np.float32), p=np.full(T, nan), lam=nan, best=nan, first=nan, scale=s,
                ibest=-2)


def _weights(T, c, lam, p):
    w = (1.0 + T * lam * p) / (1.0 + c * c)
    return w, w.astype(np.float32)


def solve(G, c):
    """The device's CAGrad weights from the Gram matrix G ([T][T], fp64) and c > 0.  Returns {w (fp64, before the fp32
    rounding), w32, p (p*), lam, best, first (F at iteration 0), scale (s), ibest}; ibest = -2 for a degenerate G."""
    G = np.asarray(G, np.float64)
    T = G.shape[0]
    s, degenerate = _scale(G)
    if degenerate:
        return _degenerate(T, s)
    A = G / (s * s)
    acc = np.zeros(T)
    for k in range(T):
        acc = acc + A[k, :]
    a = acc / T
    abar = _tsum(a) / T
    ce = c * math.sqrt(abar + 1e-4)
    lr, mu = 5.0 * c, 0.5

    def evaluate(x):
        """p = softmax(x), u = A p, q = p'Ap, pa = p.a, through the unnormalised e as the kernel does."""
        e = np.exp(x - _tmax(x))
        v = np.zeros(T)
        for k in range(T):
            v = v + A[k, :] * e[k]
        Z, Ev, Ea = _tsum(e), _tsum(e * v), _tsum(e * a)
        return e / Z, v / Z, Ev / (Z * Z), Ea / Z

    x, m, xb = np.zeros(T), np.zeros(T), np.zeros(T)
    best, first, ib = math.inf, 0.0, 0
    for it in range(ITERS + 1):
        p, u, q, pa = evaluate(x)
        r = math.sqrt(q + 1e-4)
        F = pa + ce * r
        if it == 0:
            first = F
        if F < best:
            best, ib, xb = F, it, x.copy()
        if it == ITERS:
            break
        ph = pa + ce * q / r
        d = p * ((a + ce * u / r) - ph)
        m = d if it == 0 else mu * m + d
        x = x - lr * m
    p, _, q, _ = evaluate(xb)
    lam = ce / (math.sqrt(q + 1e-4) + 1e-4)
    w, w32 = _weights(T, c, lam, p)
    return dict(w=w, w32=w32, p=p, lam=lam, best=best, first=first, scale=s, ibest=ib)


def objective(A, c, p):
    """F(p) = p.a + ce sqrt(p' A p + 1e-4) on the scaled Gram matrix A (a = A 1/T, ce = c sqrt(mean(a) + 1e-4))."""
    a = A.mean(1)
    ce = c * math.sqrt(a.mean() + 1e-4)
    return float(p @ a + ce * math.sqrt(p @ A @ p + 1e-4))


def literal(G, c):
    """The dual solved literally: p = softmax(x), F = p' A b + ce sqrt(p' A p + 1e-4) (b uniform), torch autograd and
    torch.optim.SGD(lr = 5c, momentum = 0.5) over 20 steps at fp64, the best of the 21 iterates kept."""
    G = np.asarray(G, np.float64)
    T = G.shape[0]
    s, degenerate = _scale(G)
    if degenerate:
        return _degenerate(T, s)
    A = torch.tensor(G / (s * s), dtype=torch.float64)
    b = torch.full((T,), 1.0 / T, dtype=torch.float64)
    ce = c * torch.sqrt(b @ A @ b + 1e-4)
    x = torch.zeros(T, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.SGD([x], lr=5.0 * c, momentum=0.5)
    best, first, ib, xb = math.inf, None, 0, x.detach().clone()
    for it in range(ITERS + 1):
        p = torch.softmax(x, 0)
        F = p @ A @ b + ce * torch.sqrt(p @ A @ p + 1e-4)
        if it == 0:
            first = float(F.detach())
        if float(F.detach()) < best:
            best, ib, xb = float(F.detach()), it, x.detach().clone()
        if it < ITERS:
            opt.zero_grad()
            F.backward()
            opt.step()
    p = torch.softmax(xb, 0)
    lam = float(ce / (torch.sqrt(p @ A @ p + 1e-4) + 1e-4))
    p = p.numpy()
    w, w32 = _weights(T, c, lam, p)
    return dict(w=w, w32=w32, p=p, lam=lam, best=best, first=first, scale=s, ibest=ib)


def cagrad_update(port, s, a, r, s2, d, eps_next, eps_cur, c):
    """One step of sac_port.update_SAC with CAGrad on the critic and actor optimizers: per-task gradients from autograd,
    their Gram matrix in fp64, solve(G, c) (c a number or a (critic, actor) pair; 0 = the plain sum, w = 1), Adam on
    sum_t w_t g_t with w rounded to fp32; the temperature and the Polyak update as update_SAC does them.  Runs under an
    installed sac_port.ReluTape like update_SAC.  Returns [(G, w32, solve record or None)] of both optimizers."""
    spec, p = port.spec, port.p
    cs = (c, c) if np.isscalar(c) else tuple(c)
    batch = (s, a, r, s2, d)
    rows = pr.task_of_rows(spec, s.shape[0])
    out, keep = [], {}
    for which, opt in ((0, port.opt_critic), (1, port.opt_actor)):
        opt.zero_grad()
        lrow = pr._row_losses(spec, p, *batch, eps_next, eps_cur, which, keep)
        names = pr.opt_names(spec, which)
        gs = []
        for t in range(spec.num_tasks):
            g = torch.autograd.grad(lrow[rows == t].sum(), [p[n] for n in names], retain_graph=True)
            gs.append({n: x.detach() for n, x in zip(names, g)})
        G = pr.gram(pr.flat(gs, names))
        rec = solve(G, cs[which]) if cs[which] > 0 else None
        w32 = rec["w32"] if rec is not None else np.ones(spec.num_tasks, np.float32)
        for n in names:
            tot = sum(float(w32[t]) * gs[t][n].double() for t in range(spec.num_tasks))
            p[n].grad = tot.float()
        opt.step()
        out.append((G, w32, rec))
    tid = sp.task_ids(spec, s)
    port.opt_alpha.zero_grad()
    la = p["log_alpha"][tid].unsqueeze(1)
    alpha_loss = -(la * (keep["logp"] - float(spec.act_dim))).mean()
    alpha_loss.backward()
    port.opt_alpha.step()
    with torch.no_grad():
        for q in ("q1", "q2"):
            for i, _ in enumerate(sp.layer_dims(spec, q)):
                for kind in ("weight", "bias"):
                    t_, l_ = p[f"{q}_target.{i}.{kind}"], p[f"{q}.{i}.{kind}"]
                    t_.copy_(spec.tau * l_ + (1.0 - spec.tau) * t_)
    return out
