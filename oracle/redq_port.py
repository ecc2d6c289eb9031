"""CPU oracle for critic ensembles (b200sac_cfg.critic_ensemble; REDQ, RLPD) -- TEST INFRASTRUCTURE, NOT PRODUCT.

oracle/sac_port.py's step with E critics q1 .. qE and their targets (include/b200sac.h "Critic ensembles"):
  y      = rs r + gamma (1 - d)(min over the step's subset S of Qt_k - alpha logpi'), S from oracle/redq_ref.py;
  L_Q    = sum_k mean((y - Q_k)^2) (/ B with weighted_loss);
  actor  = mean((alpha logpi - Q)), Q = mean over the E critics ("mean") or torch.amin over them ("min"; amin_tagged lets
         a test force the device's routing, tag "amin:pi").
The critic Adam holds every tensor of q1 .. qE (LayerNorm weights included) and the Polyak update every target tensor.
Networks run through sac_port.mlp, so critic_ln_port._layer_norm_mlp() gives the LayerNorm critics, and
ensemble_dropout(masks, p) the DroQ critics with the masks of critic k keyed (k - 1, tag, layer); either way every critic
ReLU is tagged "<net>:<pass>:<layer>", so sac_port.ReluTape can force the device's masks.  At E = 2, m = 2 and "min" the step is sac_port's
(test_critic_ensemble_host.py checks it).
"""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

import critic_ln_port as lnp
import philox_ref as pr
import redq_ref
import sac_port as sp


def nets(E):
    return tuple(f"q{k + 1}" for k in range(E))


def param_names(spec, E, with_targets=True):
    names = sp.param_names(spec, ("actor",) + nets(E), False)
    if with_targets:
        names += sp.param_names(spec, tuple(f"{q}_target" for q in nets(E)), False)
    return names + ["log_alpha"]


def init_params(spec, E, seed=0, log_alpha=0.0):
    """sac_port.init_params, plus q3 .. qE drawn after it from the same generator; targets = locals."""
    p = sp.init_params(spec, seed=seed, log_alpha=log_alpha)
    g = torch.Generator().manual_seed(seed + 7919)
    for k in range(2, E):
        for i, (fin, fout) in enumerate(sp.layer_dims(spec, "q1")):
            bound = math.sqrt(6.0 / (fin + fout))
            p[f"q{k + 1}.{i}.weight"] = (torch.rand(fout, fin, generator=g) * 2 - 1) * bound
            p[f"q{k + 1}.{i}.bias"] = torch.zeros(fout)
            for kind in ("weight", "bias"):
                p[f"q{k + 1}_target.{i}.{kind}"] = p[f"q{k + 1}.{i}.{kind}"].clone()
    return p


@contextlib.contextmanager
def ensemble_dropout(masks, p):
    """sac_port.mlp with DroQ's x * (m * s) before every critic LayerNorm while it runs: masks = {(k - 1, tag, layer): bool
    [B][H]} for critic k and tag "cur" / "next" / "pi" (e.g. the device's own "mQ" / "mT" / "mP" of a step)."""
    s = torch.tensor(pr.scale(p), dtype=torch.float32)
    scaled = {key: m.float() * s for key, m in masks.items()}

    def mlp(params, net, x, tag=None):
        k = int(net.split("_")[0][1:]) - 1 if net != "actor" else None
        n = 0
        while f"{net}.{n}.weight" in params:
            n += 1
        for i in range(n):
            x = F.linear(x, params[f"{net}.{i}.weight"], params[f"{net}.{i}.bias"])
            if i < n - 1:
                g = params.get(f"{net}.{i}.ln.weight")
                if g is not None:
                    x = x * scaled[(k, tag, i)]
                    x = F.layer_norm(x, (x.shape[-1],), g, params[f"{net}.{i}.ln.bias"], eps=lnp.EPS)
                x = sp.relu_tagged(x, None if tag is None else f"{net}:{tag}:{i}")
        return x
    saved = sp.mlp
    sp.mlp = mlp
    try:
        yield
    finally:
        sp.mlp = saved


def amin_tagged(qn, tag):
    """torch.amin(qn, 0) of the actor's "min" reduction over the E critics' Q [E][B][1], under sac_port's test hook (the
    style of sac_port.min_tagged): which critics sit at the minimum routes the actor gradient, the step's discontinuity.
    The tape records z = Q_k - min [E][B] (z == 0 <=> critic k is at the minimum) and, if `forced` holds a boolean mask
    [E][B] for the tag, splits the row's gradient evenly over the critics the mask sets -- the library's rule, and
    torch.amin's own among exactly tied values.  A row's value is then the mean of its forced critics' Q, which differs
    from the minimum only where a forced critic is a near-tie (what check_forced asserts)."""
    tape = sp.ReluTape.current
    if tape is None or tag is None:
        return qn.amin(0)
    tape.z[tag] = (qn - qn.amin(0, keepdim=True)).detach().reshape(qn.shape[0], -1)
    m = tape.forced.get(tag)
    if m is None:
        return qn.amin(0)
    w = m.reshape(qn.shape).to(qn.dtype)
    return (qn * w).sum(0) / w.sum(0)


class RedqPortLearner(sp.PortLearner):
    """E critics; step k of its replica (k = 1 on the first step after create) takes the subset redq_ref.subset(seed,
    replica, k, E, m).  actor: "mean" or "min"."""

    def __init__(self, spec, params, E, m=2, actor="mean", seed=0, replica=0, step=0):
        self.spec, self.E = spec, int(E)
        self.m, self.actor, self.seed, self.replica, self.step = int(m), actor, int(seed), int(replica), int(step)
        self.p = {k: torch.nn.Parameter(v.detach().clone().float(), requires_grad=not ("_target" in k))
                  for k, v in params.items()}
        self.opt_actor = torch.optim.Adam([self.p[n] for n in sp.param_names(spec, ("actor",), False)], lr=spec.lr_actor)
        self.critic_names = [k for k in self.p if k.split(".")[0] in nets(self.E)]
        self.opt_critic = torch.optim.Adam([self.p[n] for n in self.critic_names], lr=spec.lr_critic)
        self.opt_alpha = torch.optim.Adam([self.p["log_alpha"]], lr=spec.lr_actor)
        self.last_subset = None

    def load_adam(self, st):
        """Adam state {"m": {name: t}, "v": {name: t}, "step": (critic, actor, alpha)} over q1 .. qE, the actor and log_alpha."""
        steps = dict(zip(("critic", "actor", "alpha"), st["step"]))
        for name in sp.param_names(self.spec, ("actor",), False) + self.critic_names + ["log_alpha"]:
            which = "alpha" if name == "log_alpha" else ("actor" if name.startswith("actor.") else "critic")
            opt = {"alpha": self.opt_alpha, "actor": self.opt_actor, "critic": self.opt_critic}[which]
            opt.state[self.p[name]] = {"step": torch.tensor(float(steps[which])),
                                       "exp_avg": torch.as_tensor(st["m"][name]).clone().float(),
                                       "exp_avg_sq": torch.as_tensor(st["v"][name]).clone().float()}

    def adam_state(self):
        """{"m", "v", "step"} as load_adam takes it, over the actor, q1 .. qE (LayerNorm tensors included) and log_alpha."""
        m, v = {}, {}
        steps = {"critic": 0, "actor": 0, "alpha": 0}
        for name in sp.param_names(self.spec, ("actor",), False) + self.critic_names + ["log_alpha"]:
            which = "alpha" if name == "log_alpha" else ("actor" if name.startswith("actor.") else "critic")
            st = self._opt_of(name).state.get(self.p[name], None)
            if not st:
                m[name], v[name] = torch.zeros_like(self.p[name].data), torch.zeros_like(self.p[name].data)
            else:
                m[name], v[name] = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
                steps[which] = int(st["step"])
        return {"m": m, "v": v, "step": (steps["critic"], steps["actor"], steps["alpha"])}

    def update_SAC(self, s, a, r, s2, d, eps_next, eps_cur, want_intermediates=False):
        """One step; want_intermediates: the per-row outputs as tests/_harness.check_rows reads them, q1 .. qE included
        (the actor-pass reduction as "qmin", d(actor loss)/d(action) summed over the critics as "d_action")."""
        spec, p, E = self.spec, self.p, self.E
        self.step += 1
        S = redq_ref.subset(self.seed, self.replica, self.step, E, self.m)
        self.last_subset = S
        tid = sp.task_ids(spec, s)
        alpha = p["log_alpha"].detach()[tid].exp().unsqueeze(1)
        for opt in (self.opt_critic, self.opt_actor, self.opt_alpha):
            opt.zero_grad()
        div = float(s.shape[0]) if spec.weighted_loss else 1.0
        with torch.no_grad():
            a2, logp2, _ = sp.policy_sample(spec, p, s2, eps_next, "next")
            x2 = torch.cat([s2, a2], -1)
            qts = [sp.mlp(p, f"{q}_target", x2, "next") for q in nets(E)]
            qt = torch.stack([qts[k] for k in range(E) if S[k]]).amin(0)
            y = spec.reward_scale * r + spec.gamma * (1 - d) * (qt - alpha * logp2)
        x = torch.cat([s, a], -1)
        qs = [sp.mlp(p, q, x, "cur") for q in nets(E)]
        q_loss = sum(torch.mean((y - q) ** 2) / div for q in qs)
        q_loss.backward()
        grad_of = lambda names: {n: self.p[n].grad.detach().clone() for n in names}      # noqa: E731
        self.grads = grad_of(self.critic_names)      # each optimizer's gradient, as Adam reads it
        self.opt_critic.step()

        keep = {} if want_intermediates else None
        a_cur, logp, log_std = sp.policy_sample(spec, p, s, eps_cur, "cur", keep)
        xa = torch.cat([s, a_cur], -1)
        if want_intermediates:
            xa.retain_grad()
        qn = torch.stack([sp.mlp(p, q, xa, "pi") for q in nets(E)])
        qred = qn.mean(0) if self.actor == "mean" else amin_tagged(qn, "amin:pi")
        pi_loss = torch.mean(-(qred - alpha * logp)) / div
        pi_loss.backward()
        self.grads.update(grad_of(sp.param_names(spec, ("actor",), False)))
        self.opt_actor.step()

        la = p["log_alpha"][tid].unsqueeze(1)
        alpha_loss = -(la * (logp.detach() - float(spec.act_dim))).mean()
        alpha_loss.backward()
        self.grads.update(grad_of(["log_alpha"]))
        self.opt_alpha.step()

        with torch.no_grad():
            for name in self.critic_names:
                q, rest = name.split(".", 1)
                t, l = p[f"{q}_target.{rest}"], p[name]
                t.copy_(spec.tau * l + (1.0 - spec.tau) * t)
        entropy = (0.5 * spec.act_dim * (1.0 + math.log(2 * math.pi)) + log_std.detach().sum(-1)).mean()
        out = {"critic_loss": q_loss.item(), "actor_loss": pi_loss.item(), "alpha_loss": alpha_loss.item(),
               "entropy": entropy.item(), "y": y, "q": torch.stack([q.detach() for q in qs])}
        if want_intermediates:
            out.update({f"q{k + 1}": q.detach() for k, q in enumerate(qs)})
            out.update(a_next=a2, logp_next=logp2, a_cur=a_cur.detach(), logp_cur=logp.detach(), qmin=qred.detach(),
                       d_action=xa.grad[:, spec.obs_dim:].clone(), d_head=keep["head"].grad.clone())
        return out
