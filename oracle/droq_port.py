"""CPU oracle for dropout Q-functions (b200sac_cfg.critic_dropout, DroQ) -- TEST INFRASTRUCTURE, NOT PRODUCT.

The LayerNorm critics of oracle/critic_ln_port.py with a dropout between every hidden Linear and its LayerNorm, in
training mode on every critic evaluation of the step (Hiraoka et al., ICLR 2022): after the Linear, x * (m * s), then
F.layer_norm and the ReLU.  s = (float)(1 / (1 - p)); m is the library's own draw (oracle/philox_ref.py), so the port
and the CUDA step drop the same elements.  The masks are keyed like sac_port's passes: (net, tag, layer) with net 0 for
q1 / q1_target and 1 for q2 / q2_target, and tag "cur" (critics on (s, a)), "next" (targets on (s', a')) or "pi"
(critics on (s, a~)).

_droq_mlp(masks) swaps this module's mlp in the way critic_ln_port._layer_norm_mlp does (and makes that context install
it too), so critic_ln_port.LnPortLearner and tests/_harness.py's checkers drive it unchanged; DroqPortLearner draws each
step's masks from its own step count.
"""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

import critic_ln_port as lnp
import philox_ref as pr
import sac_port as sp

TAGS = ("cur", "next", "pi")
_masks = None        # {(net, tag, layer): float32 [B][H] of m * s} while _droq_mlp runs


def step_masks(spec, seed, step, p, replica=0, nets=2):
    """{(net, tag, layer): bool [B][H]} of one step of one replica: the keep masks the CUDA step draws (nets = E: the
    masks of a critic ensemble's E critics, keyed like oracle/redq_port.ensemble_dropout's)."""
    return {(net, tag, l): torch.from_numpy(pr.drop_masks(seed, replica, step, tag, l, net, spec.batch, H, p, nets))
            for net in range(nets) for tag in TAGS for l, H in enumerate(spec.critic_hidden)}


def scaled(masks, p):
    """m * s per mask, in fp32 as torch evaluates it (s rounded to fp32 once)."""
    s = torch.tensor(pr.scale(p), dtype=torch.float32)
    return {k: m.float() * s for k, m in masks.items()}


def mlp(params, net, x, tag=None):
    """critic_ln_port.mlp with x * (m * s) after every hidden Linear of a critic (before its LayerNorm)."""
    n = 0
    while f"{net}.{n}.weight" in params:
        n += 1
    for i in range(n):
        x = F.linear(x, params[f"{net}.{i}.weight"], params[f"{net}.{i}.bias"])
        if i < n - 1:
            g = params.get(f"{net}.{i}.ln.weight")
            if g is not None:
                x = x * _masks[(0 if net.startswith("q1") else 1, tag, i)]
                x = F.layer_norm(x, (x.shape[-1],), g, params[f"{net}.{i}.ln.bias"], eps=lnp.EPS)
            x = sp.relu_tagged(x, None if tag is None else f"{net}:{tag}:{i}")
    return x


@contextlib.contextmanager
def _droq_mlp(masks):
    """sac_port's step (and critic_ln_port's, whose context installs critic_ln_port.mlp) with this module's mlp and
    `masks` = {(net, tag, layer): m * s} in place while it runs."""
    global _masks
    saved = sp.mlp, lnp.mlp, _masks
    sp.mlp, lnp.mlp, _masks = mlp, mlp, masks
    try:
        yield
    finally:
        sp.mlp, lnp.mlp, _masks = saved


class DroqPortLearner(lnp.LnPortLearner):
    """LnPortLearner whose critics drop at rate p: step k of its replica (k = 1 on the first step after create, as the
    library counts) uses the masks of philox_ref under (seed, replica, k).  step = the steps the replica already ran."""

    def __init__(self, spec, params, p, seed, replica=0, step=0, adam_state=None):
        super().__init__(spec, params, adam_state)
        self.rate, self.seed, self.replica, self.step = float(p), int(seed), int(replica), int(step)

    def update_SAC(self, *args, **kw):
        self.step += 1
        with _droq_mlp(scaled(step_masks(self.spec, self.seed, self.step, self.rate, self.replica), self.rate)):
            return super().update_SAC(*args, **kw)


def drop_backward(dy, z, g, m, s):
    """The kernels' backward in numpy fp64 for z' = z * (m ? s : 0): (dz, dg, dc), dz = (m ? s : 0) * dz' with dz' the
    LayerNorm backward at z' (critic_ln_port.ln_backward)."""
    ms = np.where(np.asarray(m, bool), np.float64(s), 0.0)
    zp = np.asarray(z, np.float64) * ms
    dzp, dg, dc = lnp.ln_backward(dy, zp, g)
    return ms * dzp, dg, dc
