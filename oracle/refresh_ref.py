"""CPU oracle of critic inference and the priority refresh (include/b200sac.h: b200sac_critic_values,
b200sac_replay_refresh_priorities) -- TEST INFRASTRUCTURE, NOT PRODUCT.

critic_values   Q of a critic pair on any rows, in eval mode: critic_ln_port.mlp, which is sac_port.mlp for plain critics
                and adds the LayerNorm for critic_ln parameters (no dropout).
refresh_eps     the refresh's slot-keyed policy noise: per action k of ring slot i with task t, z0 of Box-Muller on the first
                two words of Philox4x32-10 keyed by seed ^ (0xC2B2AE3D27D4EB4F * (replica + 1)) at counter
                (i & 0xFFFFFFFF, i >> 32, t, 0x7E00 + k).
slot_rows       the row the step trains on for ring slots: (s, a, r, s', d) with g = gamma, or the n-step fold of a linked
                ring (nstep_ref.fold) with s' taken from the fold's last hop.
td_priorities   per row: a', log pi' from sac_port.policy_sample on s' with the given noise, y = rs R + g (1 - d)
                (min(Qt1, Qt2) - alpha log pi'), alpha = exp(log_alpha[task]), and per_ref.td_priority(y, Q1, Q2).
"""
import numpy as np
import torch

import critic_ln_port as lnp
import nstep_ref
import per_ref
import philox_ref
import sac_port as sp

REFRESH_KEY_MUL = 0xC2B2AE3D27D4EB4F
NOISE_TAG = 0x7E00


def refresh_key(seed, replica):
    return (int(seed) ^ (REFRESH_KEY_MUL * (int(replica) + 1))) & (2 ** 64 - 1)


def box_muller_z0(w0, w1):
    """common.cuh's box_muller, first output, in fp64: u = ((w >> 8) + 1) / 2^24, z0 = sqrt(-2 log u0) cos(2 pi u1)."""
    u = ((np.asarray(w0, np.uint32) >> 8).astype(np.float64) + 1.0) / 16777216.0
    v = ((np.asarray(w1, np.uint32) >> 8).astype(np.float64) + 1.0) / 16777216.0
    return np.sqrt(-2.0 * np.log(u)) * np.cos(2.0 * np.pi * v)


def refresh_eps(seed, replica, slots, tasks, act_dim):
    """[n][act_dim] fp32 noise of the ring slots `slots` (int64) with tasks `tasks`."""
    slots = np.asarray(slots, np.int64).astype(np.uint64)[:, None]
    tasks = np.asarray(tasks, np.int64).astype(np.uint32)[:, None]
    k = np.arange(act_dim, dtype=np.uint32)[None, :]
    w0, w1, _, _ = philox_ref.philox(refresh_key(seed, replica), (slots & np.uint64(0xFFFFFFFF)).astype(np.uint32),
                                     (slots >> np.uint64(32)).astype(np.uint32), tasks, np.uint32(NOISE_TAG) + k)
    return box_muller_z0(w0, w1).astype(np.float32)


def critic_values(params, obs, act, target=False):
    """(q1, q2) or their targets on rows obs [n][obs_dim], act [n][act_dim]: two fp32 numpy arrays [n]."""
    x = torch.cat([torch.as_tensor(obs, dtype=torch.float32), torch.as_tensor(act, dtype=torch.float32)], -1)
    sfx = "_target" if target else ""
    with torch.no_grad():
        return tuple(lnp.mlp(params, f"{net}{sfx}", x).reshape(-1).numpy() for net in ("q1", "q2"))


def slot_rows(ring, slots, cap_t, gamma, link=None, n=1):
    """The training rows of ring slots: ring = (s, a, r, s2, d) numpy arrays over the replica's ring indices; link (the
    replica's link table over ring indices) and n fold n-step returns.  Returns dict(s, a, R, s2, d, g, task)."""
    s, a, r, s2, d = (np.asarray(x, np.float32) for x in ring)
    slots = np.asarray(slots, np.int64)
    if link is None:
        R, g, dd, last = r.reshape(-1)[slots], np.full(len(slots), np.float32(gamma)), d.reshape(-1)[slots], slots
    else:
        R, g, dd, last, _ = nstep_ref.fold(r.reshape(-1), d.reshape(-1), link, cap_t, slots, n, gamma)
    return dict(s=s[slots], a=a[slots], R=R, s2=s2[last], d=dd, g=g, task=slots // cap_t)


def td_priorities(spec, params, rows, eps):
    """(prio fp64 [n], y, q1, q2 fp32 [n]) of the rows (slot_rows' dict) under the noise eps [n][act_dim]."""
    f = lambda k: torch.as_tensor(np.asarray(rows[k], np.float32))
    s, a, s2 = f("s"), f("a"), f("s2")
    R, d, g = f("R").reshape(-1, 1), f("d").reshape(-1, 1), f("g").reshape(-1, 1)
    task = torch.as_tensor(np.asarray(rows["task"], np.int64))
    with torch.no_grad():
        a2, logp2, _ = sp.policy_sample(spec, params, s2, torch.as_tensor(np.asarray(eps, np.float32)))
        x2, x = torch.cat([s2, a2], -1), torch.cat([s, a], -1)
        qt = torch.min(lnp.mlp(params, "q1_target", x2), lnp.mlp(params, "q2_target", x2))
        q1, q2 = lnp.mlp(params, "q1", x), lnp.mlp(params, "q2", x)
        alpha = params["log_alpha"].detach().reshape(-1)[task].double().exp().float().reshape(-1, 1)
        y = spec.reward_scale * R + g * (1 - d) * (qt - alpha * logp2)
    y, q1, q2 = (v.reshape(-1).numpy() for v in (y, q1, q2))
    return per_ref.td_priority(y, q1, q2), y, q1, q2
