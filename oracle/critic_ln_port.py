"""CPU oracle for layer-normalized critics (b200sac_cfg.critic_ln) -- TEST INFRASTRUCTURE, NOT PRODUCT.

The SAC port of oracle/sac_port.py with nn.LayerNorm(H, eps=1e-5) between every hidden Linear and its ReLU in q1, q2 and
their targets (DroQ, Hiraoka et al. 2022; Lyle et al. 2023; BRO, Nauman et al. 2024), as the library's critic_ln handles
run it.  The LayerNorm tensors are named like the library's layout table, right after their Linear's bias:
  q1.{l}.ln.weight|bias, q2.{l}.ln.weight|bias, q1_target.*, q2_target.*    l = 0..Lc-1, shape (H,)
The ReLU after each LayerNorm goes through sac_port.relu_tagged, so ReluTape records and forces the post-normalization
pre-activation exactly as for the plain critics.

ln_forward / ln_backward restate in numpy fp64 the math the CUDA kernels implement (distributed_sac_b200/csrc/
ln_kernels.cuh, include/b200sac.h "Layer-normalized critics").
"""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

import sac_port as sp

EPS = 1e-5


def is_critic(net):
    return net != "actor"


def param_names(spec, nets=sp.NETS, with_alpha=True):
    """sac_port.param_names with the critics' LayerNorm tensors, in the library's layout order."""
    names = []
    for net in nets:
        dims = sp.layer_dims(spec, net)
        for i, _ in enumerate(dims):
            names += [f"{net}.{i}.weight", f"{net}.{i}.bias"]
            if is_critic(net) and i < len(dims) - 1:
                names += [f"{net}.{i}.ln.weight", f"{net}.{i}.ln.bias"]
    if with_alpha:
        names.append("log_alpha")
    return names


def init_params(spec, seed=0, log_alpha=0.0):
    """sac_port.init_params (the same draws) plus LayerNorm weights 1 and biases 0; targets = locals."""
    p = sp.init_params(spec, seed=seed, log_alpha=log_alpha)
    for net in ("q1", "q2", "q1_target", "q2_target"):
        for i, H in enumerate(spec.critic_hidden):
            p[f"{net}.{i}.ln.weight"] = torch.ones(H)
            p[f"{net}.{i}.ln.bias"] = torch.zeros(H)
    return p


def mlp(params, net, x, tag=None):
    """sac_port.mlp with F.layer_norm before every hidden ReLU of a network that has LayerNorm tensors."""
    n = 0
    while f"{net}.{n}.weight" in params:
        n += 1
    for i in range(n):
        x = F.linear(x, params[f"{net}.{i}.weight"], params[f"{net}.{i}.bias"])
        if i < n - 1:
            g = params.get(f"{net}.{i}.ln.weight")
            if g is not None:
                x = F.layer_norm(x, (x.shape[-1],), g, params[f"{net}.{i}.ln.bias"], eps=EPS)
            x = sp.relu_tagged(x, None if tag is None else f"{net}:{tag}:{i}")
    return x


@contextlib.contextmanager
def _layer_norm_mlp():
    """sac_port's step, with this module's mlp in place of sac_port.mlp while it runs."""
    plain = sp.mlp
    sp.mlp = mlp
    try:
        yield
    finally:
        sp.mlp = plain


class LnPortLearner(sp.PortLearner):
    """sac_port.PortLearner whose critics carry LayerNorm: the same update_SAC (order of operations, losses, Adam), with
    the LayerNorm weights and biases in the critic optimizer and in the Polyak update of the targets."""

    def __init__(self, spec, params, adam_state=None):
        self.spec = spec
        self.p = {k: torch.nn.Parameter(v.detach().clone().float(), requires_grad=not ("_target" in k))
                  for k, v in params.items()}
        self.opt_actor = torch.optim.Adam([self.p[n] for n in param_names(spec, ("actor",), False)], lr=spec.lr_actor)
        self.opt_critic = torch.optim.Adam([self.p[n] for n in param_names(spec, ("q1", "q2"), False)], lr=spec.lr_critic)
        self.opt_alpha = torch.optim.Adam([self.p["log_alpha"]], lr=spec.lr_actor)
        if adam_state is not None:
            self.load_adam(adam_state)

    def _which(self, name):
        return "alpha" if name == "log_alpha" else ("actor" if name.startswith("actor.") else "critic")

    def load_adam(self, st):
        steps = dict(zip(("critic", "actor", "alpha"), st["step"]))
        for name in param_names(self.spec, sp.TRAINABLE_NETS):
            self._opt_of(name).state[self.p[name]] = {
                "step": torch.tensor(float(steps[self._which(name)])),
                "exp_avg": torch.as_tensor(st["m"][name]).clone().float(),
                "exp_avg_sq": torch.as_tensor(st["v"][name]).clone().float(),
            }

    def adam_state(self):
        m, v = {}, {}
        steps = {"critic": 0, "actor": 0, "alpha": 0}
        for name in param_names(self.spec, sp.TRAINABLE_NETS):
            st = self._opt_of(name).state.get(self.p[name], None)
            if st is None or len(st) == 0:
                m[name], v[name] = torch.zeros_like(self.p[name].data), torch.zeros_like(self.p[name].data)
            else:
                m[name], v[name] = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
                steps[self._which(name)] = int(st["step"])
        return {"m": m, "v": v, "step": (steps["critic"], steps["actor"], steps["alpha"])}

    def update_SAC(self, *args, **kw):
        with _layer_norm_mlp():
            out = super().update_SAC(*args, **kw)
        with torch.no_grad():           # sac_port's Polyak loop covers the Linear tensors
            for q in ("q1", "q2"):
                for i in range(len(self.spec.critic_hidden)):
                    for kind in ("weight", "bias"):
                        t, l = self.p[f"{q}_target.{i}.ln.{kind}"], self.p[f"{q}.{i}.ln.{kind}"]
                        t.copy_(self.spec.tau * l + (1.0 - self.spec.tau) * t)
        return out


# ---- the kernels' math in numpy fp64 -----------------------------------------------------------------------------------
def ln_forward(z, g, c):
    """z [rows][H] -> (h = relu(g * xhat + c), xhat, rstd [rows][1]), biased variance, eps 1e-5."""
    z = np.asarray(z, np.float64)
    mu = z.mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(((z - mu) ** 2).mean(-1, keepdims=True) + EPS)
    xhat = (z - mu) * rstd
    y = np.asarray(g, np.float64) * xhat + np.asarray(c, np.float64)
    return np.where(y < 0.0, 0.0, y), xhat, rstd


def ln_backward(dy, z, g):
    """dy = the ReLU-masked gradient at h [rows][H] -> (dz, dg, dc):
    dz = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)), dg = sum_rows dy*xhat, dc = sum_rows dy."""
    dy = np.asarray(dy, np.float64)
    g = np.asarray(g, np.float64)
    _, xhat, rstd = ln_forward(z, g, np.zeros_like(g))
    gd = g * dy
    dz = rstd * (gd - gd.mean(-1, keepdims=True) - xhat * (gd * xhat).mean(-1, keepdims=True))
    return dz, (dy * xhat).sum(0), dy.sum(0)
