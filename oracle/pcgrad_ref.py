"""PCGrad reference (Yu et al., "Gradient Surgery for Multi-Task Learning", NeurIPS 2020) for the pcgrad step plan.

Three pieces:
  task_grads      per-task gradients of one optimizer from sac_port's autograd step, the minibatch partitioned by
                  t(i) = i // (B / T): g_t = d/dtheta sum_{i: t(i) = t} l_i, so sum_t g_t is the ordinary step gradient;
  pcgrad_vector   the literal restatement of PCGrad on flattened gradients, in fp64, given the permutations (and optionally
                  the projection decisions to take);
  gram_solve      the Gram-form coefficients c^(i) and weights w_k = 1 - sum_i c^(i)_k that the device implements;
and pcgrad_update, one whole PCGrad step of a sac_port.PortLearner on given permutations.
"""
import numpy as np
import torch

import sac_port as sp


def task_of_rows(spec, B=None):
    B = B or spec.batch
    return torch.arange(B) // (B // spec.num_tasks)


def block_batch(spec, seed=1234):
    """sac_port.synthetic_batch with the rows sorted into task blocks (row i of task i // (B / T))."""
    s, a, r, s2, d = sp.synthetic_batch(spec, seed=seed)
    order = torch.argsort(sp.task_ids(spec, s), stable=True)
    return s[order], a[order], r[order], s2[order], d[order]


def _row_losses(spec, p, s, a, r, s2, d, eps_next, eps_cur, which, keep=None):
    """Per-row loss terms l_i of the critic (which = 0) or actor (which = 1) loss, as sac_port.update_SAC evaluates them
    (the 1/B mean and weighted_loss's extra 1/B included); their sum is the optimizer's loss.  keep (actor): receives the
    policy's log-prob and log-std under "logp" and "log_std"."""
    B = s.shape[0]
    tid = sp.task_ids(spec, s)
    alpha = p["log_alpha"].detach()[tid].exp().unsqueeze(1)
    div = float(B) if spec.weighted_loss else 1.0
    if which == 0:
        with torch.no_grad():
            a2, logp2, _ = sp.policy_sample(spec, p, s2, eps_next, "next")
            x2 = torch.cat([s2, a2], -1)
            qt = torch.min(sp.mlp(p, "q1_target", x2, "next"), sp.mlp(p, "q2_target", x2, "next"))
            y = spec.reward_scale * r + spec.gamma * (1 - d) * (qt - alpha * logp2)
        x = torch.cat([s, a], -1)
        q1, q2 = sp.mlp(p, "q1", x, "cur"), sp.mlp(p, "q2", x, "cur")
        return (((y - q1) ** 2) / B / div + ((y - q2) ** 2) / B / div).reshape(-1)
    a_cur, logp, log_std = sp.policy_sample(spec, p, s, eps_cur, "cur")
    if keep is not None:
        keep.update(logp=logp.detach(), log_std=log_std.detach())
    xa = torch.cat([s, a_cur], -1)
    qmin = sp.min_tagged(sp.mlp(p, "q1", xa, "pi"), sp.mlp(p, "q2", xa, "pi"), "route:pi")
    return (-(qmin - alpha * logp) / B / div).reshape(-1)


def opt_names(spec, which):
    return sp.param_names(spec, ("q1", "q2") if which == 0 else ("actor",), False)


def task_grads(spec, params, batch, eps_next, eps_cur, which):
    """[T] dicts {name: gradient of the rows of task t} of optimizer `which` (0 critic, 1 actor) at `params` (the actor's
    gradient is taken through the critics in `params`: pass the critics after the step's critic update)."""
    p = {k: torch.nn.Parameter(v.detach().clone().float()) for k, v in params.items()}
    lrow = _row_losses(spec, p, *batch, eps_next, eps_cur, which)
    rows = task_of_rows(spec, lrow.shape[0])
    names = opt_names(spec, which)
    out = []
    for t in range(spec.num_tasks):
        g = torch.autograd.grad(lrow[rows == t].sum(), [p[n] for n in names], retain_graph=True, allow_unused=True)
        out.append({n: (x if x is not None else torch.zeros_like(p[n])).detach() for n, x in zip(names, g)})
    return out


def flat(gs, names):
    """[T][n] fp64 matrix of per-task gradient dicts."""
    return np.stack([np.concatenate([g[n].double().reshape(-1).numpy() for n in names]) for g in gs])


def draw_perms(T, rng):
    return np.stack([rng.permutation(T) for _ in range(T)])


def pcgrad_vector(g, perms, decisions=None):
    """Literal PCGrad on the rows of g ([T][n], fp64): for each task i, g_i^PC = g_i; for j in perms[i]:
    if g_i^PC . g_j < 0 (or decisions[i][j], when given): g_i^PC -= (g_i^PC . g_j) / |g_j|^2 g_j.
    Returns (sum_i g_i^PC, [T][T] bool projections taken)."""
    g = np.asarray(g, np.float64)
    T = g.shape[0]
    taken = np.zeros((T, T), bool)
    total = np.zeros(g.shape[1])
    for i in range(T):
        gi = g[i].copy()
        for j in perms[i]:
            dot = gi @ g[j]
            proj = bool(decisions[i][j]) if decisions is not None else dot < 0
            if proj:
                gi -= dot / (g[j] @ g[j]) * g[j]
                taken[i, j] = True
        total += gi
    return total, taken


def gram(g):
    g = np.asarray(g, np.float64)
    return g @ g.T


def gram_solve(G, perms, on=True):
    """The device's Gram form: c^(i) [T][T], w [T] (fp64, before the fp32 rounding) and the projections taken, from the
    Gram matrix G and the permutations, in the kernel's order of operations."""
    T = G.shape[0]
    c = np.zeros((T, T))
    taken = np.zeros((T, T), bool)
    if on:
        for i in range(T):
            for j in perms[i]:
                s = 0.0
                for k in range(T):
                    s += c[i, k] * G[k, j]
                dot = G[i, j] - s
                if dot < 0:
                    c[i, j] += dot / G[j, j]
                    taken[i, j] = True
    w = np.empty(T)
    for k in range(T):
        s = 0.0
        for i in range(T):
            s += c[i, k]
        w[k] = 1.0 - s
    return c, w, taken


def combine_fp32(slices, w32):
    """The gradient Adam reads: fp32(w_0 g_0) + fp32(w_1 g_1) + ... in index order, every operation rounded to fp32."""
    acc = np.float32(w32[0]) * slices[0].astype(np.float32)
    for k in range(1, len(slices)):
        acc = (acc + np.float32(w32[k]) * slices[k].astype(np.float32)).astype(np.float32)
    return acc


def pcgrad_update(port, s, a, r, s2, d, eps_next, eps_cur, perms, on=(True, True)):
    """One step of sac_port.update_SAC with PCGrad on the critic and actor optimizers: per-task gradients from autograd,
    the Gram matrix in fp64, the Gram-form solve on the given permutations perms[o] ([T][T], e.g. the device's), Adam on
    sum_k w_k g_k with w rounded to fp32; the temperature and the Polyak update as update_SAC does them.  Runs under an
    installed sac_port.ReluTape like update_SAC.  Returns [(G, w32, taken)] of both optimizers."""
    spec, p = port.spec, port.p
    batch = (s, a, r, s2, d)
    rows = task_of_rows(spec, s.shape[0])
    out, keep = [], {}
    for which, opt in ((0, port.opt_critic), (1, port.opt_actor)):
        opt.zero_grad()
        lrow = _row_losses(spec, p, *batch, eps_next, eps_cur, which, keep)
        names = opt_names(spec, which)
        gs = []
        for t in range(spec.num_tasks):
            g = torch.autograd.grad(lrow[rows == t].sum(), [p[n] for n in names], retain_graph=True)
            gs.append({n: x.detach() for n, x in zip(names, g)})
        G = gram(flat(gs, names))
        _, w, taken = gram_solve(G, np.asarray(perms[which]), on[which])
        w32 = w.astype(np.float32)
        for n in names:
            tot = sum(float(w32[t]) * gs[t][n].double() for t in range(spec.num_tasks))
            p[n].grad = tot.float()
        opt.step()
        out.append((G, w32, taken))
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
