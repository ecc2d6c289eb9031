"""Helpers shared by the CPU (oracle) and GPU (product) parity tests."""
import json
import os

import numpy as np
import torch

import sac_port as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_npz(name):
    """tests/golden/<name>.npz as {key: array}; a fixture of more than 1 MB is stored as parts <name>.0.npz, <name>.1.npz, ..."""
    paths = [os.path.join(GOLDEN, name + ".npz")]
    if not os.path.exists(paths[0]):
        paths = []
        while os.path.exists(os.path.join(GOLDEN, f"{name}.{len(paths)}.npz")):
            paths.append(os.path.join(GOLDEN, f"{name}.{len(paths)}.npz"))
        if not paths:
            raise FileNotFoundError(os.path.join(GOLDEN, name + ".npz"))
    out = {}
    for p in paths:
        with np.load(p, allow_pickle=False) as z:
            out.update({k: z[k] for k in z.files})
    return out


def golden_file(name, dst_dir):
    """Path of tests/golden/<name>; a file of more than 1 MB is stored as byte parts <name>.0, <name>.1, ... and joined
    into dst_dir/<name>."""
    path = os.path.join(GOLDEN, name)
    if os.path.exists(path):
        return path
    parts = []
    while os.path.exists(f"{path}.{len(parts)}"):
        parts.append(f"{path}.{len(parts)}")
    if not parts:
        raise FileNotFoundError(path)
    out = os.path.join(str(dst_dir), name)
    with open(out, "wb") as f:
        for p in parts:
            with open(p, "rb") as part:
                f.write(part.read())
    return out


CASES = ["ll_xavier_s2", "ll_ckpt_s3", "vs_small_s10", "ms_small_s5", "ms_small_unweighted_s3"]

# Parity tolerances (SURVEY.md §8(c)): rel 1e-4 on losses / intermediates and
# per-tensor rel-L2 1e-4 on parameters, targets and Adam moments; log_alpha abs 1e-6.
REL = 1e-4


class Case:
    def __init__(self, name):
        z = load_npz(name)
        self.name = name
        self.spec = sp.SacSpec(**json.loads(str(z["spec"])))
        self.family = str(z["family"])
        self.n_steps = int(z["n_steps"])
        grab = lambda pre: {k[len(pre):]: torch.from_numpy(z[k]) for k in z if k.startswith(pre)}
        self.p_in, self.m_in, self.v_in = grab("p_in/"), grab("m_in/"), grab("v_in/")
        self.p_out, self.m_out, self.v_out = grab("p_out/"), grab("m_out/"), grab("v_out/")
        self.i0 = grab("i0/")
        self.batch = grab("batch/")
        self.eps_next, self.eps_cur = torch.from_numpy(z["eps_next"]), torch.from_numpy(z["eps_cur"])
        self.step_in, self.step_out = z["step_in"], z["step_out"]
        self.losses = z["losses"]

    def step_batch(self, i):
        return tuple(self.batch[k][i] for k in ("s", "a", "r", "s2", "d"))


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double().flatten(), torch.as_tensor(b).double().flatten()
    den = b.norm().item()
    return (a - b).norm().item() / den if den > 0 else (a - b).norm().item()


def rel_scalar(a, b):
    return abs(a - b) / max(abs(b), 1e-12)


def check_state(case, params, m, v, steps, tol=REL, what="state"):
    bad = []
    for k, ref in case.p_out.items():
        if k == "log_alpha":
            err = (params[k].double() - ref.double()).abs().max().item()
            if err > 1e-6:
                bad.append((k, "abs", err))
        else:
            err = rel_l2(params[k], ref)
            if err > tol:
                bad.append((k, "p", err))
    for k, ref in case.m_out.items():
        e1, e2 = rel_l2(m[k], ref), rel_l2(v[k], case.v_out[k])
        if e1 > tol:
            bad.append((k, "m", e1))
        if e2 > tol:
            bad.append((k, "v", e2))
    assert not bad, f"{what} mismatch in {case.name}: {bad[:8]}"
    assert tuple(int(x) for x in steps) == tuple(int(x) for x in case.step_out)


def core_config(spec, replicas=1, **kw):
    from distributed_sac_b200.core import CoreConfig
    d = dict(state_dim=spec.state_dim, act_dim=spec.act_dim, actor_hidden=list(spec.actor_hidden),
             critic_hidden=list(spec.critic_hidden), batch=spec.batch, num_tasks=spec.num_tasks,
             weighted_loss=spec.weighted_loss, replicas=replicas, gamma=spec.gamma, tau=spec.tau,
             reward_scale=spec.reward_scale, lr_actor=spec.lr_actor, lr_critic=spec.lr_critic,
             action_scale=spec.action_scale, beta1=spec.beta1, beta2=spec.beta2, adam_eps=spec.adam_eps)
    d.update(kw)
    return CoreConfig(**d)


class CareCase:
    """Fixture of the CARE(M) learner (oracle/care_port.py names)."""

    def __init__(self, name="care_small_s4"):
        import care_port as cp
        z = load_npz(name)
        self.name = name
        self.spec = cp.CareSpec(**json.loads(str(z["spec"])))
        self.n_steps = int(z["n_steps"])
        grab = lambda pre: {k[len(pre):]: torch.from_numpy(z[k]) for k in z if k.startswith(pre)}
        self.p_in, self.m_in, self.v_in = grab("p_in/"), grab("m_in/"), grab("v_in/")
        self.p_out, self.m_out, self.v_out = grab("p_out/"), grab("m_out/"), grab("v_out/")
        self.i0, self.batch = grab("i0/"), grab("batch/")
        self.eps_next, self.eps_cur = torch.from_numpy(z["eps_next"]), torch.from_numpy(z["eps_cur"])
        self.step_in, self.step_out, self.losses = z["step_in"], z["step_out"], z["losses"]

    step_batch = Case.step_batch


def care_core_config(spec, replicas=1, **kw):
    from distributed_sac_b200.core import CoreConfig
    d = dict(state_dim=spec.state_dim, act_dim=spec.act_dim, actor_hidden=list(spec.actor_hidden),
             critic_hidden=list(spec.critic_hidden), batch=spec.batch, num_tasks=spec.num_tasks,
             weighted_loss=spec.weighted_loss, replicas=replicas, gamma=spec.gamma, tau=spec.tau,
             reward_scale=spec.reward_scale, lr_actor=spec.lr_actor, lr_critic=spec.lr_critic,
             action_scale=spec.action_scale, beta1=spec.beta1, beta2=spec.beta2, adam_eps=spec.adam_eps,
             care=True, num_encoders=spec.num_encoders, mix_hidden=list(spec.mix_hidden), mix_out=spec.mix_out,
             ctx_in=spec.ctx_in, ctx_hidden=list(spec.ctx_hidden), ctx_out=spec.ctx_out, tau_se=spec.tau_se,
             care_original=not spec.modified, emb_dim=spec.emb_dim, lr_ctx=spec.lr_ctx)
    d.update(kw)
    return CoreConfig(**d)


# ---------------------------------------------------------------------------------------------------------------
# ReLU-kink analysis for randomly drawn full-size problems (replaces the old "kink budget").
# Two correct fp32 evaluations of one step can put a pre-activation that is zero at the parity bar's resolution on
# different sides of the ReLU (different summation order); one flipped mask bit moves the gradients upstream of it by
# ~1/sqrt(batch*width) ~ 1e-3.  Instead of tolerating "a few tensors beyond 1e-4", the tests PROVE what happened:
#   (1) the masks the CUDA step actually used (sign pattern of its stored activations) are forced into the oracle
#       (oracle/sac_port.ReluTape) and EVERYTHING must then agree to 1e-4 -- losses, parameters, targets, Adam moments;
#   (2) every forced mask bit that differs from the oracle's own sits on a pre-activation with |z| <= 1e-4 * max(1, mean|z|)
#       (the parity bar itself): a kink, not an arithmetic error.
# Every step starts from the oracle's state (copied into the CUDA arena), so differences never compound.
# ---------------------------------------------------------------------------------------------------------------
def sync_core_to_port(core, port, replica=0):
    from distributed_sac_b200 import _lib
    st = port.adam_state()
    core.set_named(port.params(), _lib.PARAMS, replica)
    core.set_named(st["m"], _lib.ADAM_M, replica)
    core.set_named(st["v"], _lib.ADAM_V, replica)
    core.set_steps(st["step"], replica)


def cuda_relu_masks(core, spec, replica=0, care=False, E=2):
    """{ReluTape tag: bool mask} from the activations the last CUDA step stored.  E: the critics of a critic_ensemble
    handle, whose hQ / hP are [E][B][H]; with E > 2 the actor routing of a "min" replica is "amin:pi" [E][B] (critic k
    took a share of the actor gradient: oracle/redq_port.amin_tagged), and a "mean" replica has none."""
    B = spec.batch
    masks = {}
    for l, H in enumerate(spec.actor_hidden):
        hA = core.debug(f"hA.{l}", replica).reshape(2 * B, H) > 0
        masks[f"actor:next:{l}"], masks[f"actor:cur:{l}"] = hA[:B], hA[B:]
    for l, H in enumerate(spec.critic_hidden):
        hQ = core.debug(f"hQ.{l}", replica).reshape(E, B, H) > 0
        hP = core.debug(f"hP.{l}", replica).reshape(E, B, H) > 0
        for net in range(E):
            masks[f"q{net + 1}:cur:{l}"], masks[f"q{net + 1}:pi:{l}"] = hQ[net], hP[net]
    # saturated tanh: the policy head's own tanh(u) per (row, action) -- value + derivative forced into the oracle, which then
    # has to agree with it to the parity tolerance (sac_port.tanh_tagged; psave = [2B][A][8], entry 2 = tanh(u))
    t = core.debug("psave", replica).reshape(2 * B, spec.act_dim, 8)[:, :, 2]
    masks["tanh:next"], masks["tanh:cur"] = t[:B].clone(), t[B:].clone()
    # the other discontinuity of the step: which twin min(Q1, Q2)(s, a~) routes the actor gradient to (tag "route:pi",
    # True = Q1).  Handled like a ReLU bit: forced into the oracle, and a differing bit must sit on |Q1 - Q2| ~ 0
    if E == 2:
        masks["route:pi"] = (core.debug("dq_pi", replica).reshape(2, B)[0] != 0).reshape(B, 1)
    elif core.get_ensemble(replica)[1] == "min":
        masks["amin:pi"] = core.debug("dq_pi", replica).reshape(E, B) != 0
    if care:
        K = spec.num_encoders
        for l, H in enumerate(spec.mix_hidden):
            pw = (H + 3) // 4 * 4
            m0 = core.debug(f"mixH.0.{l}", replica).reshape(K, 2 * B, pw)[:, :, :H] > 0     # critic's (== actor's, tied) on [s';s]
            m1 = core.debug(f"mixH.1.{l}", replica).reshape(K, B, pw)[:, :, :H] > 0         # target's on s'
            m2 = core.debug(f"mixH.2.{l}", replica).reshape(K, B, pw)[:, :, :H] > 0         # updated critic's on s
            masks[f"ase.mix:next:{l}"], masks[f"ase.mix:cur:{l}"] = m0[:, :B], m0[:, B:]
            masks[f"cse.mix:cur:{l}"], masks[f"tse.mix:next:{l}"], masks[f"cse.mix:pi:{l}"] = m0[:, B:], m1, m2
    return masks


def check_forced(tape, forced, what=""):
    """Every forced bit that differs from the oracle's own decision must sit on a numerically-zero pre-activation (a ReLU
    kink / a tie of min(Q1,Q2) / a critic within rounding of an ensemble's minimum, where the tape's z = Q_k - min and the
    oracle's own bit is z <= 0); every forced tanh value must agree with the oracle's own to the parity tolerance.
    Returns {tag: differing bits}."""
    flips = {}
    for tag, m in forced.items():
        z = tape.z[tag]
        if tag.startswith("tanh:"):
            worst = float((z - m.reshape(z.shape)).abs().max())
            assert worst <= REL, f"{what}tanh(u) of {tag} differs by {worst:.3e} > {REL}"
            continue
        diff = ((z <= 0) if tag.startswith("amin:") else (z > 0)) != m
        n = int(diff.sum())
        if n:
            tol = REL * max(1.0, float(z.abs().mean()))
            worst = float(z[diff].abs().max())
            assert worst <= tol, f"{what}mask bit of {tag} differs at |z| = {worst:.3e} > {tol:.3e}: not a ReLU kink"
            flips[tag] = n
    return flips


def kink_checked_step(core, port, spec, batch, e1, e2, replica=0, care=False, step_cuda=None, want_intermediates=False,
                      E=2):
    """One step of `core` (from the port's state) and of `port` with the CUDA masks forced; returns (port outputs,
    {tag: flipped bits}).  Raises AssertionError if a flipped bit is not a kink.  want_intermediates: the port's outputs
    include its per-row intermediates (computed with the forced masks).  E: the handle's critics (cuda_relu_masks)."""
    sync_core_to_port(core, port, replica)
    (step_cuda or (lambda: core.step(*batch, e1, e2)))()
    forced = cuda_relu_masks(core, spec, replica, care, E)
    with sp.ReluTape(forced) as tape:
        out = (port.update if care else port.update_SAC)(*batch, e1, e2, want_intermediates=want_intermediates)
    flips = check_forced(tape, forced)
    return out, flips


def check_port_state(core, port, replica=0, tol=REL, params=True):
    """CUDA state == port state to 1e-4 per tensor (parameters, targets, Adam moments), log_alpha to 1e-6.  params=False:
    the Adam moments only, for a caller that checks the parameters through the gradients and the exact optimizer step."""
    from distributed_sac_b200 import _lib
    got, ref = core.get_named(_lib.PARAMS, replica), port.params()
    st = port.adam_state()
    gm, gv = core.get_named(_lib.ADAM_M, replica), core.get_named(_lib.ADAM_V, replica)
    bad = []
    for k, v in ref.items():
        if k == "log_alpha":
            assert (got[k] - v).abs().max().item() <= 1e-6
            continue
        errs = [rel_l2(got[k], v)]
        if k in st["m"]:
            errs += [rel_l2(gm[k], st["m"][k]), rel_l2(gv[k], st["v"][k])]
        if not params:
            errs = errs[1:]
        if errs and max(errs) > tol:
            bad.append((k, errs))
    assert not bad, f"state differs beyond {tol} with the CUDA masks forced into the oracle: {[(k, [float(f"{e:.1e}") for e in es]) for k, es in bad]}"


# ---------------------------------------------------------------------------------------------------------------
# Full-size "summary" fixtures from the UNMODIFIED reference (oracle/gen_golden.py: FULL_CASES / FULL_CARE_CASES).
# Inputs are regenerated from the stored seeds; outputs are per-step losses, the first step's forward intermediates
# and, per tensor, sum / L2 norm / 1024 sample elements of the reference's result.
# ---------------------------------------------------------------------------------------------------------------
FULL_CASES = ["full_vs_s3", "full_ms_s3", "full_ll_s100"]
FULL_CARE_CASES = ["full_c10m_s2", "full_c10o_s2"]


class FullCase:
    def __init__(self, name):
        z = load_npz(name)
        self.name, self.z = name, z
        self.care = str(z["family"]) == "C10"
        if self.care:
            import care_port as cp
            self.spec = cp.CareSpec(**json.loads(str(z["spec"])))
            self.params = cp.init_params(self.spec, seed=int(z["param_seed"]))
            self._batch = lambda seed: cp.synthetic_batch(self.spec, seed=seed)
        else:
            self.spec = sp.SacSpec(**json.loads(str(z["spec"])))
            self.params = sp.init_params(self.spec, seed=int(z["param_seed"]))
            self._batch = lambda seed: sp.synthetic_batch(self.spec, seed=seed)
        self.n_steps = int(z["n_steps"])
        self.losses = z["losses"]
        self.i0 = {k[3:]: torch.from_numpy(z[k]) for k in z if k.startswith("i0/")}
        self.step_out = z["step_out"]
        g = torch.Generator().manual_seed(int(z["data_seed"]) + 17)
        self.batches, self.eps_next, self.eps_cur = [], [], []
        for i in range(self.n_steps):
            self.batches.append(self._batch(int(z["data_seed"]) + i))
            self.eps_next.append(torch.randn(self.spec.batch, self.spec.act_dim, generator=g))
            self.eps_cur.append(torch.randn(self.spec.batch, self.spec.act_dim, generator=g))

    def make_port(self):
        if self.care:
            import care_port as cp
            return cp.CarePortLearner(self.spec, self.params)
        return sp.PortLearner(self.spec, self.params)

    def tensors(self, prefix):
        return sorted({k.split("/")[1] for k in self.z if k.startswith(prefix + "/")})

    def check_summary(self, prefix, tensors, tol, what):
        """sampled elements (rel-L2 over the sample), L2 norm and sum of every tensor against the reference's."""
        bad = []
        for k in self.tensors(prefix):
            t = torch.as_tensor(tensors[k]).reshape(-1).double()
            idx = torch.from_numpy(self.z[f"{prefix}/{k}/idx"])
            ref = torch.from_numpy(self.z[f"{prefix}/{k}/val"]).double()
            if k == "log_alpha":
                if (t[idx] - ref).abs().max().item() > 1e-6:
                    bad.append((k, "abs", (t[idx] - ref).abs().max().item()))
                continue
            e_s = rel_l2(t[idx], ref)
            l2 = float(self.z[f"{prefix}/{k}/l2"])
            e_n = abs(t.norm().item() - l2) / max(l2, 1e-30)
            if e_s > tol or e_n > tol:
                bad.append((k, e_s, e_n))
        assert not bad, f"{what}: {prefix} differs from the reference summary of {self.name} beyond {tol}: {bad[:6]}"
