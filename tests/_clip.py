"""The autograd oracles with gradient-norm clipping, for the tests of b200sac_cfg.grad_clip: the reference learners
(oracle/sac_port.PortLearner, oracle/care_port.CarePortLearner) stay as they are, and clip_oracle() puts
torch.nn.utils.clip_grad_norm_ in front of their optimizers' step() -- the place the feature defines."""
import torch


def clip_oracle(port, max_grad_norm):
    """Make `port` call clip_grad_norm_(params, max_grad_norm) on the critic's, the actor's and (CARE(O)) the context
    encoder's parameters right before that optimizer's step() (not the temperature's), and keep the norms it returned in
    port.grad_norms = {"critic", "actor"[, "ctx"]} (overwritten by every update).  max_grad_norm=None: the port is left
    unclipped and grad_norms stays empty.  Returns the port."""
    port.grad_norms = {}
    if max_grad_norm is None:
        return port
    for key, opt in (("critic", port.opt_critic), ("actor", port.opt_actor), ("ctx", getattr(port, "opt_ctx", None))):
        if opt is None:
            continue

        def step(*a, _opt=opt, _orig=opt.step, _key=key, **kw):
            ps = [t for grp in _opt.param_groups for t in grp["params"]]
            port.grad_norms[_key] = float(torch.nn.utils.clip_grad_norm_(ps, max_grad_norm))
            return _orig(*a, **kw)
        opt.step = step
    return port
