"""Gradient surgery (PCGrad, CAGrad) reference for the CARE learners: the counterparts of pcgrad_ref.task_grads /
pcgrad_update and cagrad_ref.cagrad_update on care_port.CarePortLearner.

  row_losses     per-row critic / actor loss terms exactly as CarePortLearner.update forms them (the 1/B mean,
                 weighted_loss's extra 1/B, the detaches of the actor pass); their sum is the optimizer's loss;
  task_grads     per-task gradients of one loss, the minibatch partitioned by t(i) = i // (B / T): the critic loss gives
                 the critic optimizer's names (cse.*, q1, q2) and, on CARE(O), the context encoder's cenc.*; the actor loss
                 the actor's names;
  surgery_update one whole step of a CarePortLearner with PCGrad (given permutations and switches) or CAGrad (given c) on
                 the critic and actor optimizers, the context encoder stepped on the plain sum of its task gradients.
Everything runs under an installed sac_port.ReluTape with update()'s tags, so _golden.cuda_relu_masks(..., care=True) can
force a device step's masks.
"""
import numpy as np
import torch

import cagrad_ref as cr
import care_port as cp
import pcgrad_ref as pr
import sac_port as sp


def opt_names(port, which):
    """Names of optimizer `which`: 0 critic (learner.py:150-153 order), 1 actor, 2 CARE(O) context encoder."""
    return (port.critic_names, port.actor_names, port.ctx_names)[which]


def loss_names(port, which):
    """Names the loss of optimizer `which` (0 critic, 1 actor) trains: the critic loss also trains the context encoder."""
    return port.critic_names + port.ctx_names if which == 0 else port.actor_names


def row_losses(port, s, a, r, s2, d, eps_next, eps_cur, which, keep=None):
    """Per-row loss terms l_i of the critic (which = 0) or actor (which = 1) loss at the port's current parameters, as
    CarePortLearner.update evaluates them.  keep (actor): receives the policy's log-prob under "logp"."""
    spec, p = port.spec, port.p
    B = s.shape[0]
    tid = torch.argmax(s[:, -spec.num_tasks:], dim=1)
    alpha = p["log_alpha"].detach()[tid].exp().unsqueeze(1)
    div = float(B) if spec.weighted_loss else 1.0
    z = cp.context_encode(spec, p, tid)
    if which == 0:
        with torch.no_grad():
            a2, logp2, _ = port._policy("ase", z, s2, eps_next, False, "next")
            qt1, qt2 = port._q("tse", "q1_target", "q2_target", z, s2, a2, tag="next")
            y = spec.reward_scale * r + spec.gamma * (1 - d) * (torch.min(qt1, qt2) - alpha * logp2)
        q1, q2 = port._q("cse", "q1", "q2", z, s, a, tag="cur")
        return (((y - q1) ** 2) / B / div + ((y - q2) ** 2) / B / div).reshape(-1)
    a_cur, logp, _ = port._policy("ase", z.detach(), s, eps_cur, True, "cur")
    if keep is not None:
        keep.update(logp=logp.detach())
    q1n, q2n = port._q("cse", "q1", "q2", z.detach(), s, a_cur, detach=True, tag="pi")
    qmin = sp.min_tagged(q1n, q2n, "route:pi")
    return (-(qmin - alpha * logp) / B / div).reshape(-1)


def task_grads(port, batch, eps_next, eps_cur, which, keep=None):
    """[T] dicts {name: gradient of the rows of task t} of loss `which` at the port's current parameters (for the actor,
    set the port's critic names to the critics after the step's critic update; `ase.*` stays the encoder before it)."""
    rows = pr.task_of_rows(port.spec, batch[0].shape[0])
    lrow = row_losses(port, *batch, eps_next, eps_cur, which, keep)
    names = loss_names(port, which)
    out = []
    for t in range(port.spec.num_tasks):
        g = torch.autograd.grad(lrow[rows == t].sum(), [port.p[n] for n in names], retain_graph=True, allow_unused=True)
        out.append({n: (x if x is not None else torch.zeros_like(port.p[n])).detach() for n, x in zip(names, g)})
    return out


def surgery_update(port, s, a, r, s2, d, eps_next, eps_cur, perms=None, on=(True, True), c=None):
    """One CarePortLearner.update with gradient surgery on the critic and actor optimizers: per-task gradients from
    autograd, their Gram matrix in fp64, then pcgrad_ref.gram_solve on perms[o] and the switches `on` (c None) or
    cagrad_ref.solve with c (a number or a (critic, actor) pair; 0 = the plain sum), Adam on sum_t fp32(w_t) g_t.  The
    context encoder's Adam reads the plain sum of its task gradients; the temperature, both Polyak rates and the encoder
    tie follow in update()'s order.  Returns [(G, w32, taken or the CAGrad record)] of both optimizers."""
    spec, p = port.spec, port.p
    batch = (s, a, r, s2, d)
    T = spec.num_tasks
    cs = None if c is None else ((c, c) if np.isscalar(c) else tuple(c))
    for opt in (port.opt_critic, port.opt_actor, port.opt_alpha) + ((port.opt_ctx,) if port.opt_ctx else ()):
        opt.zero_grad()
    out, keep, ctx_gs = [], {}, None
    for which, opt in ((0, port.opt_critic), (1, port.opt_actor)):
        gs = task_grads(port, batch, eps_next, eps_cur, which, keep)
        names = opt_names(port, which)
        G = pr.gram(pr.flat(gs, names))
        if cs is None:
            _, w, rec = pr.gram_solve(G, np.asarray(perms[which]), on[which])
            w32 = w.astype(np.float32)
        else:
            rec = cr.solve(G, cs[which]) if cs[which] > 0 else None
            w32 = rec["w32"] if rec is not None else np.ones(T, np.float32)
        for n in names:
            p[n].grad = sum(float(w32[t]) * gs[t][n].double() for t in range(T)).float()
        opt.step()
        if which == 0:
            ctx_gs = gs
        out.append((G, w32, rec))
    tid = torch.argmax(s[:, -T:], dim=1)
    la = p["log_alpha"][tid].unsqueeze(1)
    alpha_loss = -(la * (keep["logp"] + (-float(spec.act_dim)))).mean()
    alpha_loss.backward()
    port.opt_alpha.step()
    with torch.no_grad():
        ms = spec.mlp_spec()
        for q in ("q1", "q2"):
            for i, _ in enumerate(sp.layer_dims(ms, q)):
                for kind in ("weight", "bias"):
                    t_, l_ = p[f"{q}_target.{i}.{kind}"], p[f"{q}.{i}.{kind}"]
                    t_.copy_(spec.tau * l_ + (1.0 - spec.tau) * t_)
        for k in cp.encoder_names(spec, "cse"):
            t_, l_ = p["tse" + k[3:]], p[k]
            t_.copy_(spec.tau_se * l_ + (1.0 - spec.tau_se) * t_)
    if port.opt_ctx is not None:
        for n in port.ctx_names:
            p[n].grad = sum(ctx_gs[t][n].double() for t in range(T)).float()
        port.opt_ctx.step()
    with torch.no_grad():
        for k in cp.encoder_names(spec, "cse"):
            p["ase" + k[3:]].copy_(p[k])
    return out
