"""CPU oracle for the SAC gradient step -- TEST INFRASTRUCTURE, NOT PRODUCT.

Clean-room plain-PyTorch (fp32, CPU, autograd) restatement of the reference's
learner hot path.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference leg may import this module; the product
package `distributed_sac_b200` never does.

Parity pin: this port is checked against the UNMODIFIED reference (imported
from /root/reference through oracle/ref_harness.py) by
tests/test_oracle_vs_reference.py in the build container, and against the
committed fixtures tests/golden/*.npz (generated from the real reference by
oracle/gen_golden.py) everywhere.  The reference itself has no tests or golden
vectors (SURVEY.md §4), and its arithmetic lives in an unpinned PyTorch, so the
pin is "this image's torch 2.11 CPU fp32 running the reference's own code".

Reference sites restated here (paths relative to /root/reference):
  step ordering ........ LunarLander_Distributed_SAC/src/learner.py:203-239,246-264
                         MT10_Distributed_MTSAC/src/learner.py:253-325,332-352
  tanh-Gaussian policy . LunarLander_Distributed_SAC/src/model.py:38-65
                         MT10_Distributed_MTSAC/src/model.py:35-56
  Q networks ........... LunarLander_Distributed_SAC/src/model.py:117-142
                         MT10_Distributed_MTSAC/src/model.py:151-196
  per-task alpha ....... MT10_Distributed_MTSAC/src/learner.py:213-233
  "weighted" loss ...... MT10_Distributed_MTSAC/src/model.py:100-114,184-194
                         (a (B,)x(B,1) broadcast: equals mean(loss)/B, SURVEY §0.6)
  Polyak ............... LunarLander_Distributed_SAC/src/learner.py:126-137
  Adam ................. torch.optim.Adam defaults (learner.py:115-124)

Canonical parameter names used across oracle/, tests/golden/ and the product:
  actor.{i}.weight|bias   i = 0..La   (i == La is the mu/log_std head, 2*act wide)
  q1.{i}.weight|bias, q2.{i}...       i = 0..Lc (i == Lc is the scalar head)
  q1_target.*, q2_target.*            same shapes
  log_alpha                           (T,)  T = max(num_tasks, 1)
"""
import math
from dataclasses import dataclass, field, asdict
from typing import List

import numpy as np
import torch
import torch.nn.functional as F


@dataclass
class SacSpec:
    state_dim: int = 8          # width of the raw state (without the task one-hot)
    act_dim: int = 2
    actor_hidden: List[int] = field(default_factory=lambda: [256, 256])
    critic_hidden: List[int] = field(default_factory=lambda: [256, 256])
    batch: int = 256
    num_tasks: int = 0          # 0 -> single-task SAC (scalar log_alpha); T>0 -> one-hot head
    weighted_loss: bool = False  # MTSAC "use_weighted_loss" (== extra 1/B)
    gamma: float = 0.99
    tau: float = 0.005
    reward_scale: float = 1.0
    lr_actor: float = 3e-4
    lr_critic: float = 3e-4
    action_scale: float = 1.0   # k = (hi - lo) / 2
    beta1: float = 0.9
    beta2: float = 0.999
    adam_eps: float = 1e-8

    @property
    def obs_dim(self):          # what the networks see ("mtobs" in the MT variants)
        return self.state_dim + self.num_tasks

    @property
    def n_alpha(self):
        return max(self.num_tasks, 1)

    def to_json(self):
        return asdict(self)


def ll_spec(**kw):
    return SacSpec(**kw)


def vs_spec(**kw):
    d = dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 400, 400], batch=1024)
    d.update(kw)
    return SacSpec(**d)


def ms_spec(**kw):
    d = dict(state_dim=39, act_dim=4, actor_hidden=[400, 400, 400], critic_hidden=[400, 400, 400], batch=1280,
             num_tasks=10, weighted_loss=True)
    d.update(kw)
    return SacSpec(**d)


def layer_dims(spec: SacSpec, net: str):
    if net == "actor":
        dims = [spec.obs_dim] + list(spec.actor_hidden) + [2 * spec.act_dim]
    else:
        dims = [spec.obs_dim + spec.act_dim] + list(spec.critic_hidden) + [1]
    return list(zip(dims[:-1], dims[1:]))


NETS = ("actor", "q1", "q2", "q1_target", "q2_target")
TRAINABLE_NETS = ("actor", "q1", "q2")


def param_names(spec: SacSpec, nets=NETS, with_alpha=True):
    names = []
    for net in nets:
        for i, _ in enumerate(layer_dims(spec, net)):
            names += [f"{net}.{i}.weight", f"{net}.{i}.bias"]
    if with_alpha:
        names.append("log_alpha")
    return names


def param_shape(spec: SacSpec, name: str):
    if name == "log_alpha":
        return (spec.n_alpha,)
    net, i, kind = name.split(".")
    fin, fout = layer_dims(spec, net)[int(i)]
    return (fout, fin) if kind == "weight" else (fout,)


def init_params(spec: SacSpec, seed=0, log_alpha=0.0):
    """Xavier-uniform(gain 1) weights, zero biases (LL/model.py:33-36, MS/utils.py:30-33);
    targets start as copies of the locals (LL/learner.py:287-288)."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for net in TRAINABLE_NETS:
        for i, (fin, fout) in enumerate(layer_dims(spec, net)):
            bound = math.sqrt(6.0 / (fin + fout))
            p[f"{net}.{i}.weight"] = (torch.rand(fout, fin, generator=g) * 2 - 1) * bound
            p[f"{net}.{i}.bias"] = torch.zeros(fout)
    for q in ("q1", "q2"):
        for i, _ in enumerate(layer_dims(spec, q)):
            for kind in ("weight", "bias"):
                p[f"{q}_target.{i}.{kind}"] = p[f"{q}.{i}.{kind}"].clone()
    p["log_alpha"] = torch.full((spec.n_alpha,), float(log_alpha))
    return p


def synthetic_batch(spec: SacSpec, seed=1234, batch=None):
    """SURVEY §8(d) synthetic transitions: s,s'~N(0,1), a~U(-1,1), r~N(0,1), d~Bern(0.01);
    MT: task id = i mod T appended as one-hot to s and s' (same id)."""
    B = batch or spec.batch
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(B, spec.state_dim, generator=g)
    a = torch.rand(B, spec.act_dim, generator=g) * 2 - 1
    r = torch.randn(B, 1, generator=g)
    s2 = torch.randn(B, spec.state_dim, generator=g)
    d = (torch.rand(B, 1, generator=g) < 0.01).float()
    if spec.num_tasks > 0:
        tid = torch.arange(B) % spec.num_tasks
        tid = tid[torch.randperm(B, generator=g)]
        oh = F.one_hot(tid, spec.num_tasks).float()
        s = torch.cat([s, oh], 1)
        s2 = torch.cat([s2, oh], 1)
    return s, a, r, s2, d


class ReluTape:
    """Test hook for the ReLU-kink analysis (tests/test_gpu_parity.py).  While installed (`with ReluTape(...)`), every
    ReLU of the port records its pre-activation under a tag "<net>:<pass>:<layer>" and, if `forced` holds a boolean mask
    for that tag, gates with THAT mask instead of z > 0 (forward z * mask, backward grad * mask).  Two correct fp32
    evaluations of the same step can put a pre-activation within rounding of zero on different sides of the ReLU; with
    the masks of the implementation under test forced into the oracle, everything else must agree to 1e-4, and every
    forced bit that differs from the oracle's own must sit on such a numerically-zero pre-activation."""
    current = None

    def __init__(self, forced=None):
        self.forced = forced or {}
        self.z = {}

    def __enter__(self):
        ReluTape.current = self
        return self

    def __exit__(self, *exc):
        ReluTape.current = None


def relu_tagged(z, tag):
    tape = ReluTape.current
    if tape is None or tag is None:
        return torch.relu(z)
    tape.z[tag] = z.detach()
    m = tape.forced.get(tag)
    return torch.relu(z) if m is None else z * m.to(z.dtype)


def min_tagged(a, b, tag):
    """torch.min(a, b) of the actor loss (LL/learner.py:222-223) under the same test hook: the routing of the gradient (which
    twin is the smaller one) is the step's other discontinuity.  The tape records z = b - a (z > 0 <=> `a` is taken) and, if
    `forced` holds a boolean mask for the tag, takes `a` exactly where the mask says so."""
    tape = ReluTape.current
    if tape is None or tag is None:
        return torch.min(a, b)
    tape.z[tag] = (b - a).detach()
    m = tape.forced.get(tag)
    return torch.min(a, b) if m is None else torch.where(m.reshape(a.shape), a, b)


class _GivenTanh(torch.autograd.Function):
    """tanh whose VALUE is given (the implementation under test's own tanh(u), within a few ulp of torch's) and whose
    derivative is 1 - t^2 of that given value: what autograd does with torch.tanh's saved output, for a prescribed output."""

    @staticmethod
    def forward(ctx, u, t_given):
        ctx.save_for_backward(t_given)
        return t_given.clone()

    @staticmethod
    def backward(ctx, g):
        (t,) = ctx.saved_tensors
        return g * (1 - t * t), None


def tanh_tagged(u, tag):
    """torch.tanh(u) of the policy head (LL/model.py:50-60) under the test hook.  log(1 - tanh(u)^2 + 1e-6) and its gradient
    are ill-conditioned where tanh saturates: one ulp of tanh(u) moves 1 - t^2 by a large relative amount (DESIGN.md 3), so
    two correct evaluations whose pre-activations differ in the last bits (3xTF32 GEMMs vs fp32 FFMA) can differ by percents
    in the gradient of such a row.  The tape records torch's own t under `tag`; if `forced` holds a float tensor for the tag
    the port continues with THAT t (value and 1 - t^2 derivative) -- the test then asserts that the two t agree to the
    parity tolerance, and everything downstream must agree without any allowance."""
    tape = ReluTape.current
    t = torch.tanh(u)
    if tape is None or tag is None:
        return t
    tape.z[tag] = t.detach()
    given = tape.forced.get(tag)
    return t if given is None else _GivenTanh.apply(u, given.reshape(u.shape).to(u.dtype))


def mlp(params, net, x, tag=None):
    n = len([k for k in params if k.startswith(net + ".") and k.endswith(".weight")])
    for i in range(n):
        x = F.linear(x, params[f"{net}.{i}.weight"], params[f"{net}.{i}.bias"])
        if i < n - 1:
            x = relu_tagged(x, None if tag is None else f"{net}:{tag}:{i}")
    return x


def policy_sample(spec, params, obs, eps, tag=None, keep=None):
    """LL/model.py:38-65. Returns action, log_prob (B,1), log_std (B,act).  keep (a dict): receives the head output
    [mu | raw log_std] under "head", with its gradient retained."""
    A = spec.act_dim
    out = mlp(params, "actor", obs, tag)
    if keep is not None and out.requires_grad:
        out.retain_grad()
        keep["head"] = out
    mu = out[:, :A]
    log_std = torch.clamp(out[:, A:], -20, 2)
    std = torch.exp(log_std)
    u = mu + std * eps                      # Normal.rsample with injected eps
    k = spec.action_scale
    act = k * tanh_tagged(u, None if tag is None else f"tanh:{tag}")
    var = std ** 2                          # torch.distributions.Normal.log_prob
    gauss = -((u - mu) ** 2) / (2 * var) - std.log() - math.log(math.sqrt(2 * math.pi))
    logp = gauss - torch.log(k * (1 - (act / k) ** 2 + 1e-6))
    return act, logp.sum(-1, keepdim=True), torch.log(std)


def task_ids(spec, obs):
    if spec.num_tasks > 0:
        return torch.argmax(obs[:, -spec.num_tasks:], dim=1)
    return torch.zeros(obs.shape[0], dtype=torch.long)


class PortLearner:
    """One learner: parameters, 3 Adam optimizers, update_SAC()."""

    def __init__(self, spec: SacSpec, params, adam_state=None):
        self.spec = spec
        self.p = {k: torch.nn.Parameter(v.detach().clone().float(), requires_grad=not ("_target" in k))
                  for k, v in params.items()}
        actor_ps = [self.p[n] for n in param_names(spec, ("actor",), False)]
        critic_ps = [self.p[n] for n in param_names(spec, ("q1", "q2"), False)]
        self.opt_actor = torch.optim.Adam(actor_ps, lr=spec.lr_actor)
        self.opt_critic = torch.optim.Adam(critic_ps, lr=spec.lr_critic)
        self.opt_alpha = torch.optim.Adam([self.p["log_alpha"]], lr=spec.lr_actor)
        if adam_state is not None:
            self.load_adam(adam_state)

    # ---- Adam state as {name: (m, v)} + {"step": (critic, actor, alpha)} ----
    def _opt_of(self, name):
        if name == "log_alpha":
            return self.opt_alpha
        return self.opt_actor if name.startswith("actor.") else self.opt_critic

    def load_adam(self, st):
        steps = dict(zip(("critic", "actor", "alpha"), st["step"]))
        for name in param_names(self.spec, TRAINABLE_NETS):
            opt = self._opt_of(name)
            which = "alpha" if name == "log_alpha" else ("actor" if name.startswith("actor.") else "critic")
            opt.state[self.p[name]] = {
                "step": torch.tensor(float(steps[which])),
                "exp_avg": torch.as_tensor(st["m"][name]).clone().float(),
                "exp_avg_sq": torch.as_tensor(st["v"][name]).clone().float(),
            }

    def adam_state(self):
        m, v = {}, {}
        steps = {"critic": 0, "actor": 0, "alpha": 0}
        for name in param_names(self.spec, TRAINABLE_NETS):
            st = self._opt_of(name).state.get(self.p[name], None)
            which = "alpha" if name == "log_alpha" else ("actor" if name.startswith("actor.") else "critic")
            if st is None or len(st) == 0:
                m[name] = torch.zeros_like(self.p[name].data)
                v[name] = torch.zeros_like(self.p[name].data)
            else:
                m[name], v[name] = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
                steps[which] = int(st["step"])
        return {"m": m, "v": v, "step": (steps["critic"], steps["actor"], steps["alpha"])}

    def params(self):
        return {k: v.detach().clone() for k, v in self.p.items()}

    def update_SAC(self, s, a, r, s2, d, eps_next=None, eps_cur=None, want_intermediates=False):
        """One gradient step. Order of operations follows LL/learner.py:246-264,203-239."""
        spec, p = self.spec, self.p
        B = s.shape[0]
        if eps_next is None:
            eps_next = torch.randn(B, spec.act_dim)
        if eps_cur is None:
            eps_cur = torch.randn(B, spec.act_dim)
        tid = task_ids(spec, s)
        # update(): alpha snapshot before anything moves (LL:250 / MS:337)
        alpha = p["log_alpha"].detach()[tid].exp().unsqueeze(1)
        for opt in (self.opt_critic, self.opt_actor, self.opt_alpha):
            opt.zero_grad()
        div = float(B) if spec.weighted_loss else 1.0   # SURVEY §0.6

        with torch.no_grad():
            a2, logp2, _ = policy_sample(spec, p, s2, eps_next, "next")
            x2 = torch.cat([s2, a2], -1)
            qt = torch.min(mlp(p, "q1_target", x2, "next"), mlp(p, "q2_target", x2, "next"))
            y = spec.reward_scale * r + spec.gamma * (1 - d) * (qt - alpha * logp2)

        x = torch.cat([s, a], -1)
        q1, q2 = mlp(p, "q1", x, "cur"), mlp(p, "q2", x, "cur")
        q_loss = torch.mean((y - q1) ** 2) / div + torch.mean((y - q2) ** 2) / div
        q_loss.backward()
        self.opt_critic.step()

        keep = {} if want_intermediates else None
        a_cur, logp, log_std = policy_sample(spec, p, s, eps_cur, "cur", keep)
        xa = torch.cat([s, a_cur], -1)
        if want_intermediates:
            xa.retain_grad()          # its action columns: d(actor loss)/d(action) through the critics alone
        q1n, q2n = mlp(p, "q1", xa, "pi"), mlp(p, "q2", xa, "pi")      # already-updated critics
        qmin = min_tagged(q1n, q2n, "route:pi")
        pi_loss = torch.mean(-(qmin - alpha * logp)) / div
        pi_loss.backward()
        self.opt_actor.step()

        h_bar = -float(spec.act_dim)
        la = p["log_alpha"][tid].unsqueeze(1)
        alpha_loss = -(la * (logp.detach() + h_bar)).mean()
        alpha_loss.backward()
        self.opt_alpha.step()

        with torch.no_grad():
            for q in ("q1", "q2"):
                for i, _ in enumerate(layer_dims(spec, q)):
                    for kind in ("weight", "bias"):
                        t, l = p[f"{q}_target.{i}.{kind}"], p[f"{q}.{i}.{kind}"]
                        t.copy_(spec.tau * l + (1.0 - spec.tau) * t)

        entropy = (0.5 * spec.act_dim * (1.0 + math.log(2 * math.pi)) + log_std.detach().sum(-1)).mean()
        out = {"critic_loss": q_loss.item(), "actor_loss": pi_loss.item(),
               "alpha_loss": alpha_loss.item(), "entropy": entropy.item()}
        if want_intermediates:
            out.update(y=y, q1=q1.detach(), q2=q2.detach(), a_next=a2, logp_next=logp2,
                       a_cur=a_cur.detach(), logp_cur=logp.detach(), qmin=qmin.detach(),
                       d_action=xa.grad[:, spec.obs_dim:].clone(), d_head=keep["head"].grad.clone())
        return out


class PortReplay:
    """Uniform sampling without replacement (random.sample semantics,
    LL/replay_buffer.py:63-73); MT: B/T per task then one shuffle
    (MS/replay_buffers.py:67-100).  numpy-backed ring, used only for the CPU
    baseline timing and for sampler property tests."""

    def __init__(self, spec: SacSpec, capacity, seed=0):
        self.spec = spec
        self.cap = int(capacity)
        self.rng = np.random.default_rng(seed)
        w = 2 * spec.obs_dim + spec.act_dim + 2
        self.rows = np.zeros((self.cap, w), np.float32)
        self.task = np.zeros(self.cap, np.int64)
        self.n = 0
        self.head = 0

    def push_many(self, s, a, r, s2, d):
        rows = np.concatenate([np.asarray(t, np.float32).reshape(len(s), -1) for t in (s, a, r, s2, d)], 1)
        for row in rows:
            self.rows[self.head] = row
            if self.spec.num_tasks:
                self.task[self.head] = int(np.argmax(row[self.spec.state_dim:self.spec.obs_dim]))
            self.head = (self.head + 1) % self.cap
            self.n = min(self.n + 1, self.cap)

    def sample(self):
        spec, B = self.spec, self.spec.batch
        if spec.num_tasks:
            per = B // spec.num_tasks
            idx = []
            for t in range(spec.num_tasks):
                pool = np.nonzero(self.task[:self.n] == t)[0]
                idx.append(self.rng.choice(pool, per, replace=False))
            idx = np.concatenate(idx)
            self.rng.shuffle(idx)
        else:
            idx = self.rng.choice(self.n, B, replace=False)
        rows = torch.from_numpy(self.rows[idx])
        o, A = spec.obs_dim, spec.act_dim
        return rows[:, :o], rows[:, o:o + A], rows[:, o + A:o + A + 1], rows[:, o + A + 1:2 * o + A + 1], rows[:, -1:]
