"""Drop-in `Learner` classes: the reference's Python surface over the CUDA hot path.

Same constructor signatures, cfg JSONs, method names, return values, state_dict
keys and checkpoint format as the reference learners; `update()` /
`update_SAC()` run in libb200sac instead of ~2000 eager ATen ops.

  LunarLanderLearner  <- LunarLander_Distributed_SAC/src/learner.py:21-316
  VSACLearner         <- MT1_Distributed_VSAC/src/learner.py:22-322
  MTSACLearner        <- MT10_Distributed_MTSAC/src/learner.py:22-414

What is deliberately NOT copied (SURVEY.md §0.7): `to_device` forgetting the second
critics, `load_checkpoint` touching a non-existent `actor.optimizer` (ours loads),
the checkpoint filename concatenated onto the directory name without a slash (ours
joins paths), `buffer_size` hard-coded to 1e5 in the LL learner (kept as the LL default
but overridable).  Redis / Ray / TensorBoard are out of scope: the learner takes a
`server` object (anything with redis-py's set/get/rpush/delete/scan_iter/pipeline API);
if none is given and `redis` is importable it connects to localhost like the reference.
"""
import itertools
import json
import math
import re
import os
import pickle as _pickle
import time
from datetime import datetime

import numpy as np
import torch

from . import _lib, names
from .core import ENSEMBLE_ACTOR, REDO_NETS, CoreConfig, Replay, SacCore, redo_taus, reset_spec
from .replay_buffer import ReplayBuffer, MTReplayBuffer


class Decoder(json.JSONDecoder):
    """Numeric *strings* become ints (LL/utils.py:4-20)."""

    def decode(self, s):
        return self._coerce(super().decode(s))

    def _coerce(self, o):
        if isinstance(o, str):
            try:
                return int(o)
            except ValueError:
                return o
        if isinstance(o, dict):
            return {k: self._coerce(v) for k, v in o.items()}
        if isinstance(o, list):
            return [self._coerce(v) for v in o]
        return o


def cfg_read(path):
    with open(path, "r") as f:
        return json.loads(f.read(), cls=Decoder)


def _default_server():
    try:
        import redis
    except ImportError as e:       # pragma: no cover - environment dependent
        raise RuntimeError("no `server` given and the `redis` package is not installed") from e
    return redis.StrictRedis(host="localhost")


class _Handle:
    """Stand-in for the nn.Module arguments of Learner.soft_update(local, target, tau)."""

    def __init__(self, learner, net):
        self._learner, self.net = learner, net

    def state_dict(self):
        return self._learner._module_state_dict(self.net)

    def load_state_dict(self, sd):
        self._learner._load_module_state_dict(self.net, sd)


class _BaseLearner:
    family = "LL"
    log_name = "LunarLander_Distributed_SAC"
    _iteration_key = "episode_idx"
    _pcgrad_ok = False          # PCGrad and CAGrad need task-block minibatches: the multi-task learners (MTSAC and CARE)
    _critic_ln_ok = True        # LayerNorm in the critics' hidden layers: the plain-MLP critics (not CARE's)
    critic_ensemble = None      # E critics (critic_ensemble=E), None: the twins; target_subset and actor_q go with it
    target_subset, actor_q = 2, "mean"

    # ---- construction ---------------------------------------------------------------------
    def _init_common(self, cfg_path, write_mode, save_period, checkpoint_path, server, device_index, seed,
                     replay_where, precision=1, prioritized=None, actor_update_interval=1, target_update_interval=1,
                     n_step=1, max_grad_norm=None, pcgrad=False, cagrad=None, reset_interval=None, reset=None,
                     redo_interval=None, redo=None, critic_layer_norm=False, critic_dropout=None, prior=None,
                     critic_ensemble=None, target_subset=2, actor_q="mean"):
        self.critic_layer_norm = bool(critic_layer_norm)
        # DroQ (Hiraoka et al. 2022): dropout at rate p before every critic LayerNorm; it needs the LayerNorm critics
        if critic_dropout is not None:
            if not self.critic_layer_norm:
                raise ValueError("critic_dropout= needs critic_layer_norm=True (DroQ's critics are Linear -> Dropout -> "
                                 "LayerNorm -> ReLU)")
            if isinstance(critic_dropout, bool) or not 0.0 <= float(critic_dropout) < 1.0:     # (NaN fails too)
                raise ValueError(f"critic_dropout must be a rate in [0, 1) (got {critic_dropout!r})")
        self.critic_dropout = None if critic_dropout is None else float(critic_dropout)
        if prioritized is not None and replay_where != "device":
            raise ValueError("prioritized replay needs replay_where='device' (the sum-trees live beside the device ring)")
        # prioritized=dict(..., refresh_after_reset=True): every reset and recycle is followed by a full priority refresh of
        # every replica under that reset's or recycle's seed, so the sampler does not follow the discarded network's errors
        self.refresh_after_reset = False
        if prioritized is not None:
            prioritized = dict(prioritized)
            self.refresh_after_reset = prioritized.pop("refresh_after_reset", False)
            if not isinstance(self.refresh_after_reset, (bool, np.bool_)):
                raise ValueError(f"refresh_after_reset must be a bool (got {self.refresh_after_reset!r})")
            self.refresh_after_reset = bool(self.refresh_after_reset)
            if self.refresh_after_reset and not self._critic_ln_ok:
                raise ValueError(f"refresh_after_reset=True needs plain-MLP critics ({type(self).__name__} has CARE critics)")
        self.prioritized = prioritized
        if not 1 <= int(n_step) <= 16:
            raise ValueError(f"n_step must be in [1, 16] (got {n_step})")
        if int(n_step) > 1 and replay_where != "device":
            raise ValueError("n-step returns need replay_where='device' (the trajectory links live beside the device ring)")
        self.n_step = int(n_step)
        # prior=dict(capacity=N, fraction=f): a prior-data ring beside the online ring, and every minibatch takes
        # floor(f * P + 0.5) rows of each task block of P rows from it (RLPD's symmetric sampling: f = 0.5)
        self.prior = None
        if prior is not None:
            if not isinstance(prior, dict) or set(prior) != {"capacity", "fraction"}:
                raise ValueError(f"prior= takes exactly capacity and fraction (got {prior!r})")
            if replay_where != "device":
                raise ValueError("prior= needs replay_where='device' (the prior ring is a device ring)")
            if prioritized is not None or self.n_step > 1:
                raise ValueError("prior= needs a uniform, unlinked online ring (no prioritized=, n_step=1)")
            cap = prior["capacity"]
            if isinstance(cap, bool) or not isinstance(cap, (int, np.integer)) or cap < 1:
                raise ValueError(f"prior capacity must be an int >= 1 (got {cap!r})")
            self.prior = dict(capacity=int(cap), fraction=self._prior_fraction(prior["fraction"]))
        self.max_grad_norm = max_grad_norm
        self.pcgrad = bool(pcgrad)
        self.cagrad = None if cagrad is None else float(cagrad)
        self.cfg = cfg_read(cfg_path)
        self.precision = precision
        self.write_mode = write_mode
        self.save_period = save_period
        self.total_step = 0
        self.episode_idx = 0
        self.datetime = str(datetime.now())[:-7]
        self._set_dims()
        if self.critic_layer_norm:
            if not self._critic_ln_ok:
                raise ValueError(f"critic_layer_norm=True needs plain-MLP critics ({type(self).__name__} has CARE critics)")
            if self.pcgrad or self.cagrad is not None:
                raise ValueError("critic_layer_norm=True and pcgrad= / cagrad= are exclusive")
            if redo is not None or redo_interval is not None:
                raise ValueError("critic_layer_norm=True and redo= / redo_interval= are exclusive (recycling a unit would "
                                 "change its LayerNorm row's statistics, so it would not preserve the network's function)")
        self._check_ensemble(critic_ensemble, target_subset, actor_q, prioritized, redo, redo_interval)
        if self.pcgrad and not (self._pcgrad_ok and self.num_tasks >= 2):
            raise ValueError(f"pcgrad=True needs a multi-task MTSAC or CARE learner with num_tasks >= 2 ({type(self).__name__}, "
                             f"num_tasks {self.num_tasks})")
        if self.cagrad is not None:
            if self.pcgrad:
                raise ValueError("pcgrad=True and cagrad= are exclusive (a CAGrad optimizer does not project)")
            if not (self._pcgrad_ok and self.num_tasks >= 2):
                raise ValueError(f"cagrad= needs a multi-task MTSAC or CARE learner with num_tasks >= 2 ({type(self).__name__}, "
                                 f"num_tasks {self.num_tasks})")
            if not (math.isfinite(self.cagrad) and self.cagrad >= 0):
                raise ValueError(f"cagrad must be finite and >= 0 (got {cagrad})")
        # periodic network resets (primacy bias at high replay ratios; Nikishin et al. 2022, D'Oro et al. 2023): reset k
        # (k = 1, 2, ...) with seed + k * 2^32 right before update k * reset_interval + 1, counted from construction
        if reset is not None and reset_interval is None:
            raise ValueError("reset= needs reset_interval=")
        if reset_interval is not None and (isinstance(reset_interval, bool) or not isinstance(reset_interval, int)
                                           or reset_interval < 1):
            raise ValueError(f"reset_interval must be an int >= 1 (got {reset_interval!r})")
        self.reset_interval = reset_interval
        self.reset = dict(reset or {})
        reset_spec(self._core_config(), **self.reset)          # ValueError on bad parts, before a handle is built
        # periodic dormant-neuron recycling (ReDo; Sokar et al. 2023): recycle k with seed + 2^62 + k * 2^32 right before
        # update k * redo_interval + 1, after a reset that falls on the same update; redo = {actor: tau, critic: tau}
        # (default: tau 0 for both, the neurons that are dead on the batch)
        if redo is not None and redo_interval is None:
            raise ValueError("redo= needs redo_interval=")
        if redo_interval is not None and (isinstance(redo_interval, bool) or not isinstance(redo_interval, int)
                                          or redo_interval < 1):
            raise ValueError(f"redo_interval must be an int >= 1 (got {redo_interval!r})")
        self.redo_interval = redo_interval
        self.redo = self._redo_taus(dict(actor=0.0, critic=0.0) if redo is None else redo)
        self.seed = int(seed)
        self._n_updates = 0
        self._n_manual_resets = 0
        self._n_manual_redos = 0
        self._n_manual_refreshes = 0
        self.device = torch.device(self.cfg.get("device", "cuda"))
        if self.device.type != "cuda":
            raise RuntimeError("the CUDA learner only runs on CUDA devices (cfg 'device' must be 'cuda')")
        self.device_index = device_index if self.device.index is None else self.device.index
        self.server = server if server is not None else _default_server()
        for key in list(self.server.scan_iter()):      # LL/learner.py:34-36
            self.server.delete(key)
        self.core = SacCore(self._core_config(), self.device_index, seed=seed)
        # update() on a critic-only step (critic step count not a multiple of actor_update_interval) updates the critics
        # only and reports NaN actor loss / entropy; the targets move when the count is a multiple of target_update_interval
        if (actor_update_interval, target_update_interval) != (1, 1):
            self.core.set_update_intervals(actor_update_interval, target_update_interval)
        if max_grad_norm is not None:
            self.set_max_grad_norm(max_grad_norm)
        if self.critic_dropout is not None:
            self.core.set_critic_dropout(self.critic_dropout)
        if self.critic_ensemble:
            self.core.set_ensemble(self.target_subset, self.actor_q)
        if self.cagrad is not None:
            self.core.set_pcgrad(critic=False, actor=False)
            self.set_cagrad(self.cagrad)
        self.memory = self._make_memory(replay_where)
        if self.prior is not None:
            self.memory.attach_prior(self.prior["capacity"])
            self.set_prior_fraction(self.prior["fraction"])
        self.memory.start()
        self.save_model_path = os.path.join("saved_models", self.log_name, self.datetime)
        self.log_file = os.path.join("log", "log_" + self.log_name, f"{self.log_name}_log_{self.datetime}.txt")
        self.alpha = torch.ones(max(self.num_tasks, 1))     # stale build-time value the reference also saves
        if checkpoint_path is not None:
            self.load_checkpoint(checkpoint_path)
            print("######## load checkpoint completely ########")

    def _check_ensemble(self, E, m, actor_q, prioritized, redo, redo_interval):
        """critic_ensemble=E (None: the twin critics), target_subset=m and actor_q= checked before any handle is built.
        Raises ValueError."""
        self.critic_ensemble, self.target_subset, self.actor_q = None, 2, "mean"
        if E is None:
            return
        if isinstance(E, bool) or not isinstance(E, (int, np.integer)) or not 2 <= E <= 10:
            raise ValueError(f"critic_ensemble must be an int in [2, 10] (got {E!r})")
        if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 1 <= m <= E:
            raise ValueError(f"target_subset must be an int in [1, critic_ensemble = {E}] (got {m!r})")
        if actor_q not in ENSEMBLE_ACTOR:
            raise ValueError(f"actor_q must be 'mean' or 'min' (got {actor_q!r})")
        if not self._critic_ln_ok:
            raise ValueError(f"critic_ensemble= needs plain-MLP critics ({type(self).__name__} has CARE critics)")
        if self.pcgrad or self.cagrad is not None:
            raise ValueError("critic_ensemble= and pcgrad= / cagrad= are exclusive")
        if redo is not None or redo_interval is not None:
            raise ValueError("critic_ensemble= and redo= / redo_interval= are exclusive")
        if prioritized is not None:
            raise ValueError("critic_ensemble= and prioritized= are exclusive")
        self.critic_ensemble, self.target_subset, self.actor_q = int(E), int(m), actor_q

    @property
    def n_critics(self) -> int:
        """Q-functions of the learner: critic_ensemble, or 2 (the twins)."""
        return self.critic_ensemble or 2

    @property
    def _critic_nets(self):
        return tuple(f"q{k}" for k in range(1, self.n_critics + 1))

    def set_ensemble(self, target_subset=None, actor_q=None):
        """Target subset size m in [1, E] and the actor's reduction over the E critics ("mean" or "min"), effective from
        the next update(); None keeps the current value.  The learner must have been built with critic_ensemble=."""
        if not self.critic_ensemble:
            raise ValueError("this learner was built without critic_ensemble=")
        m = self.target_subset if target_subset is None else target_subset
        a = self.actor_q if actor_q is None else actor_q
        if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 1 <= m <= self.critic_ensemble:
            raise ValueError(f"target_subset must be an int in [1, {self.critic_ensemble}] (got {m!r})")
        if a not in ENSEMBLE_ACTOR:
            raise ValueError(f"actor_q must be 'mean' or 'min' (got {a!r})")
        self.core.set_ensemble(int(m), a)
        self.target_subset, self.actor_q = int(m), a

    def _check_checkpoint_critics(self, present):
        """present: the critic indices k a checkpoint holds.  A checkpoint of another ensemble size raises ValueError."""
        if sorted(present) != list(range(1, self.n_critics + 1)):
            raise ValueError(f"the checkpoint holds critics {sorted(present)}, this learner has {self.n_critics}")

    def set_per_beta(self, beta: float):
        """Importance-sampling exponent of the prioritized ring (annealing), effective from the next update()."""
        if self.prioritized is None:
            raise ValueError("this learner was built without prioritized=")
        self.memory.ring.set_beta(beta)

    def set_max_grad_norm(self, max_norm: float):
        """clip_grad_norm_(params, max_norm) before every optimizer step (critic, actor and the CARE(O) context encoder;
        not the temperature), effective from the next update(); inf turns clipping off.  The learner must have been built
        with max_grad_norm= (its step plan computes the gradient norms); core.read_grad_norms() returns them."""
        if self.max_grad_norm is None:
            raise ValueError("this learner was built without max_grad_norm=")
        self.max_grad_norm = float(max_norm)
        self.core.set_grad_clip(critic=max_norm, actor=max_norm, ctx=max_norm)

    def set_pcgrad(self, critic=True, actor=True):
        """Turn PCGrad gradient surgery of the critic / actor optimizer on or off, effective from the next update().  Off,
        Adam reads the plain sum of the per-task gradients.  The learner must have been built with pcgrad=True;
        core.read_pcgrad() returns the last update's Gram matrix, weights and projections."""
        if not self.pcgrad:
            raise ValueError("this learner was built without pcgrad=True")
        self.core.set_pcgrad(critic=critic, actor=actor)

    def set_cagrad(self, c: float):
        """CAGrad coefficient c of the critic and actor optimizers, effective from the next update(); 0 gives the plain
        sum of the per-task gradients.  The learner must have been built with cagrad=; core.read_cagrad() returns the
        last update's dual solution and core.read_pcgrad() its Gram matrix and weights."""
        if self.cagrad is None:
            raise ValueError("this learner was built without cagrad=")
        self.core.set_cagrad(critic=c, actor=c)
        self.cagrad = float(c)

    @staticmethod
    def _prior_fraction(f):
        if isinstance(f, bool) or not isinstance(f, (int, float, np.integer, np.floating)) or not 0.0 <= float(f) <= 1.0:
            raise ValueError(f"the prior fraction must be a number in [0, 1] (got {f!r})")      # (NaN fails too)
        return float(f)

    def set_prior_fraction(self, f: float):
        """Share f of every task block that the next update()s take from the prior ring: floor(f * P + 0.5) rows of each
        block of P = batch / num_tasks rows.  The learner must have been built with prior=."""
        if self.prior is None:
            raise ValueError("this learner was built without prior=")
        f = self._prior_fraction(f)
        P = self.batch_size // max(self.num_tasks, 1)
        self.memory.ring.set_prior_rows(math.floor(f * P + 0.5))
        self.prior["fraction"] = f

    def push_prior(self, states, actions, rewards, next_states, dones):
        """Append prior-data transitions (the reference's tuple layout, the multi-task one-hot inside the states).  Not part
        of a checkpoint, like the online ring."""
        if self.prior is None:
            raise ValueError("this learner was built without prior=")
        self.memory.add_prior(states, actions, rewards, next_states, dones)

    def set_n_step(self, n: int):
        """Horizon of the n-step return, effective from the next update()."""
        if self.n_step == 1:
            raise ValueError("this learner was built without n_step= (its ring keeps no trajectory links)")
        self.memory.ring.set_nstep(n)

    def _core_config(self):
        c = self.cfg
        return CoreConfig(state_dim=self.state_dim, act_dim=self.action_dim, actor_hidden=list(self.actor_hidden_dim),
                          critic_hidden=list(self.critic_hidden_dim), batch=self.batch_size, num_tasks=self.num_tasks,
                          weighted_loss=self.use_weighted_loss, replicas=1, precision=self.precision, gamma=float(self.gamma), tau=float(self.tau),
                          reward_scale=float(self.reward_scale), lr_actor=float(self.lr_actor),
                          lr_critic=float(self.lr_critic),
                          action_scale=(self.action_bound[1] - self.action_bound[0]) / 2,
                          log_alpha_init=float(c["log_alpha"]), grad_clip=self.max_grad_norm is not None,
                          pcgrad=self.pcgrad or self.cagrad is not None, critic_layer_norm=self.critic_layer_norm,
                          critic_dropout=self.critic_dropout is not None, critic_ensemble=self.critic_ensemble or 0)

    # ---- reference method surface -------------------------------------------------------------
    def _chunks(self, n):
        """Split n updates at the reset and recycle boundaries: yields the sizes of the runs of updates to enqueue, and
        enqueues reset k (seed + k * 2^32) right before update k * reset_interval + 1 and recycle k (seed + 2^62 + k * 2^32)
        right before update k * redo_interval + 1, the reset first when both fall on one update."""
        Ns = [N for N in (self.reset_interval, self.redo_interval) if N is not None]
        while n > 0:
            u = self._n_updates
            if u > 0 and self.reset_interval is not None and u % self.reset_interval == 0:
                seed = self.seed + (u // self.reset_interval) * 2 ** 32
                self.core.reset(seed, **self.reset)
                self._refresh_after(seed)
            if u > 0 and self.redo_interval is not None and u % self.redo_interval == 0:
                seed = self.seed + 2 ** 62 + (u // self.redo_interval) * 2 ** 32
                self._recycle(seed, self.redo)
                self._refresh_after(seed)
            c = min([n] + [N - u % N for N in Ns])
            yield c
            self._n_updates += c
            n -= c

    @staticmethod
    def _redo_taus(taus):
        """{actor: tau, critic: tau} checked (redo_taus' rules; a network left out is scored only).  Raises ValueError."""
        if not isinstance(taus, dict) or set(taus) - {"actor", "critic"}:
            raise ValueError(f"redo takes dict(actor=tau, critic=tau), got {taus!r}")
        redo_taus(**taus)
        return dict(taus)

    def _recycle(self, seed, taus):
        """One SacCore.redo on a fresh reference-shaped draw from the ring (a prioritized ring's weights are ignored)."""
        if self.critic_layer_norm:
            raise ValueError("dormant-neuron recycling and scoring do not run on a learner with critic_layer_norm=True")
        if self.critic_ensemble:
            raise ValueError("dormant-neuron recycling and scoring do not run on a learner with critic_ensemble=")
        s, a = self.memory.sample()[:2]
        self.core.redo(seed, s, a, **taus)

    def reset_networks(self, seed=None, **parts):
        """Reset networks now, on the current stream (SacCore.reset's part keywords and shrink; none = a full reset).
        seed=None: the j-th such call uses seed + 2^63 + j * 2^32, apart from the scheduled resets' seeds.  Not part of
        the update count that reset_interval follows; that count starts at construction (a loaded checkpoint included),
        as the reference's checkpoint format does not hold it."""
        if seed is None:
            self._n_manual_resets += 1
            seed = self.seed + 2 ** 63 + self._n_manual_resets * 2 ** 32
        self.core.reset(seed, **parts)
        self._refresh_after(seed)

    def recycle_dormant(self, seed=None, **taus):
        """Recycle dormant neurons now, on the current stream, scored on a fresh replay batch: actor= / critic= thresholds
        (none given: the learner's redo= thresholds).  seed=None: the j-th such call uses seed + 2^63 + 2^62 + j * 2^32,
        apart from the reset and scheduled recycle seeds.  Not part of the update count that redo_interval follows."""
        taus = self.redo if not taus else self._redo_taus(taus)
        if seed is None:
            self._n_manual_redos += 1
            seed = self.seed + 2 ** 63 + 2 ** 62 + self._n_manual_redos * 2 ** 32
        self._recycle(seed, taus)
        self._refresh_after(seed)

    def _refresh_after(self, seed):
        """With refresh_after_reset: a full priority refresh of every replica right after a reset or recycle, same seed."""
        if self.refresh_after_reset:
            self.memory.ring.refresh_priorities(seed)

    def refresh_priorities(self, seed=None):
        """Recompute every filled slot's priority with the current networks now (Replay.refresh_priorities, stochastic next
        actions).  seed=None: the j-th such call uses seed + 2^63 + 2^61 + j * 2^32.  The learner must have been built with
        prioritized=."""
        if self.prioritized is None:
            raise ValueError("this learner was built without prioritized=")
        if seed is None:
            self._n_manual_refreshes += 1
            seed = self.seed + 2 ** 63 + 2 ** 61 + self._n_manual_refreshes * 2 ** 32
        self.memory.ring.refresh_priorities(seed)

    def q_values(self, states, actions, target=False):
        """(q1, q2), or their targets with target=True, on rows of states and actions: two (n, 1) tensors on the learner's
        device, as Critic.forward returns them, in eval mode (no dropout).  With critic_ensemble=E: one (E, n) tensor of
        q1 .. qE (or their targets)."""
        if self.critic_ensemble:
            return self.core.critic_values(torch.as_tensor(states).to(self.device), torch.as_tensor(actions).to(self.device),
                                           target=target)
        q1, q2 = self.core.critic_values(torch.as_tensor(states).to(self.device), torch.as_tensor(actions).to(self.device),
                                         target=target)
        return q1.reshape(-1, 1), q2.reshape(-1, 1)

    def dormant_fraction(self, tau=0.0):
        """The fraction of tau-dormant neurons (score <= tau) per network and hidden layer on a fresh replay batch: a
        measure-only recycle call, nothing changes.  {"actor" | "q1" | "q2": [fraction per hidden layer]}."""
        redo_taus(tau, tau)
        if self.critic_layer_norm:
            raise ValueError("dormant_fraction() does not run on a learner with critic_layer_norm=True")
        self._recycle(self.seed, {})
        rec = self.core.read_redo()
        return {net: [float(np.mean(s <= tau)) for s in rec[net]["score"]] for net in REDO_NETS}

    def update(self):
        """Learner.update(): sample a minibatch, one SAC gradient step, return python floats."""
        for _ in self._chunks(1):
            l = self.memory.step_core(self.core)      # (critic, actor, alpha loss, entropy) python floats
        return (l[0], l[1]) if self.num_tasks == 0 else (l[0], l[1], l[3])

    def update_SAC(self, states, actions, rewards, next_states, dones, alpha=None, retain_graph=False,
                   eps_next=None, eps_cur=None):
        """Learner.update_SAC() on an explicit minibatch (device or host tensors).  `alpha` is accepted
        for signature compatibility; the step uses exp(log_alpha) snapshotted in-kernel exactly like update()."""
        for _ in self._chunks(1):
            if states.is_cuda:
                self.core.step(states, actions, rewards, next_states, dones, eps_next, eps_cur)
                losses = self.core.read_losses(1)[0]
            else:
                losses = self.core.step_host(states, actions, rewards, next_states, dones, eps_next, eps_cur)
        return self._loss_tuple(losses)

    def update_many(self, n):
        """n pipelined update() calls; returns a [n][k] tensor of the per-step losses."""
        for c in self._chunks(n):
            self.core.step_sampled(self.memory.ring, c)
        L = self.core.read_losses(min(n, 1024))[:, 0]
        return L[:, [0, 1]] if self.num_tasks == 0 else L[:, [0, 1, 3]]

    def _loss_tuple(self, losses):
        l = losses.reshape(-1, 4)[0]
        if self.num_tasks == 0:
            return float(l[0]), float(l[1])
        return float(l[0]), float(l[1]), float(l[3])

    def optimizer_zero_grad(self):
        """No-op: gradients never outlive a step in the fused path."""

    def soft_update(self, local_model=None, target_model=None, tau=None):
        """theta_target = tau*theta_local + (1-tau)*theta_target (LL/learner.py:126-137) for the pair it is given:
        (local_critic_k, target_critic_k) updates critic k's target only, as the reference's per-critic calls do;
        (None, None) updates both critics' targets at once (run()'s hard copy, tau=1.0).  The step itself already applies
        the per-step Polyak update; this entry point is for the hard copy and for callers that drive it by hand."""
        tau = self.tau if tau is None else tau
        if local_model is None and target_model is None:
            self.core.soft_update(float(tau))
            return
        pairs = {(f"q{k}", f"q{k}_target"): k for k in range(1, self.n_critics + 1)}
        key = (getattr(local_model, "net", None), getattr(target_model, "net", None))
        if (key not in pairs or getattr(local_model, "_learner", None) is not self
                or getattr(target_model, "_learner", None) is not self):
            raise ValueError(f"soft_update takes (local_critic_k, target_critic_k) of this learner or (None, None), got {key}")
        self.core.soft_update(float(tau), critic=pairs[key])

    def wait_until_memoryReady(self):
        # (with prior rows in the minibatch, the prior must also hold what the step's sampler needs)
        while len(self.memory) <= self.start_memory_len or not self.memory.prior_ready():
            time.sleep(0.1)

    def act_batch(self, states, stochastic=True):
        """Actor.get_action (LL/model.py:67-82) for a batch of environments at once with the learner's current actor:
        states [n][obs_dim] (n <= 2*batch_size) -> actions [n][action_dim] on the CPU."""
        # the LunarLander actor's deterministic action is k*mu, every other family's k*tanh(mu) (LL/model.py:78-80, VS/model.py:78-80)
        return self.core.act(torch.as_tensor(states), stochastic=stochastic, no_tanh=(self.family == "LL"))

    # ---- parameter publication (LL/learner.py:272-276; consumed by Player.pull_parameters, player.py:75-85) ----
    _published = ("actor",)

    def get_parameters(self):
        """{'actor': state_dict on the CPU} with the reference's key names: the unpickled parameters_blob(blocking=True),
        so only the published floats cross PCIe, in one copy, and the object is exactly what run() publishes.  Like
        parameters_blob(blocking=True) it returns the OLDEST blob not collected yet: the state after the steps enqueued so
        far unless a blob_begin() is still outstanding."""
        return _pickle.loads(self.parameters_blob(blocking=True))

    def parameters_blob(self, blocking=True):
        """The bytes Learner.run() stores under the Redis key 'parameters' (LL/learner.py:298-299): _pickle.dumps of
        {'actor': state_dict_on_cpu[, ...]} with the reference's key names -- what Player.pull_parameters unpickles
        (LL/player.py:75-85).  The shapes never change, so the pickle stream is built ONCE (from tensors of the same shapes)
        and handed to the library as a byte image with the positions of the float payloads (b200sac_blob_template); per
        publication a kernel gathers the current floats into a device copy of the image and ONE D2H copy brings the finished
        byte string to pinned memory -- the host never touches a tensor.
        blocking=True: publish now (get_parameters + dumps semantics); False: collect the blob started by blob_begin()."""
        self._ensure_blob()
        if blocking:
            self.core.blob_begin()
        return self.core.blob_wait()[0]

    def _ensure_blob(self):
        if getattr(self, "_blob_ready", False):
            return
        self._pub_maps = [(net, self._key_map(net)) for net in self._published]
        rng = np.random.default_rng(12345)
        fake = {net: {ref: torch.from_numpy(rng.random(self.core.tensor_shape(canon), dtype=np.float32) + 1.0) for ref, canon in m.items()}
                for net, m in self._pub_maps}
        blob = _pickle.dumps(fake)
        slots = []
        for net, m in self._pub_maps:
            for ref, canon in m.items():
                payload = fake[net][ref].numpy().tobytes()
                at = blob.find(payload)
                if at < 0 or blob.find(payload, at + 1) >= 0:
                    raise RuntimeError(f"cannot locate the payload of {net}.{ref} in the pickle stream")
                slots.append((canon, at))
        # (+ the temperature behind the image: the logger's alpha then comes from the same consistent snapshot)
        self.core.blob_template(blob, slots, extra=("log_alpha",))
        self._blob_ready = True

    def my_print(self, content):
        os.makedirs(os.path.dirname(self.log_file), exist_ok=True)
        with open(self.log_file, "a") as writer:
            print(content)
            writer.write(content + "\n")

    # ---- state_dict plumbing -----------------------------------------------------------------
    def _key_map(self, net):
        na, nc = len(self.actor_hidden_dim) + 1, len(self.critic_hidden_dim) + 1
        if net == "actor":
            return names.actor_key_map(self.family, na)
        which = int(net.split("_")[0][1:])          # q<k> / q<k>_target
        return names.critic_key_map(self.family, nc, which, target="target" in net, layer_norm=self.critic_layer_norm,
                                    dropout=self.critic_dropout is not None)

    def _module_state_dict(self, net, which=_lib.PARAMS, named=None):
        named = named if named is not None else self.core.get_named(which)
        return {ref: named[canon].clone() for ref, canon in self._key_map(net).items()}

    def _load_module_state_dict(self, net, sd, which=_lib.PARAMS):
        km = self._key_map(net)
        missing = set(km) - set(sd)
        if missing:
            raise KeyError(f"state_dict for {net} lacks {sorted(missing)}")
        self.core.set_named({km[k]: v for k, v in sd.items() if k in km}, which, strict=False)

    @property
    def log_alpha(self):
        return self.core.read_named("log_alpha")

    # ---- checkpointing (reference format, LL/learner.py:144-182) ------------------------------
    def _adam_state_dict(self, canon_names, lr, step, n_frozen_first=0):
        """torch.optim.Adam.state_dict() layout.  n_frozen_first: parameters that sit in the optimizer's param group before
        the trainable ones but never get state (the frozen nn.Embedding of the CARE context encoder is parameter 0 of
        `Adam(context_encoder.parameters())`, MT10_Distributed_CARE/src/learner.py:137-141)."""
        m, v = self.core.get_named(_lib.ADAM_M), self.core.get_named(_lib.ADAM_V)
        state = {n_frozen_first + i: {"step": torch.tensor(float(step)), "exp_avg": m[n], "exp_avg_sq": v[n]}
                 for i, n in enumerate(canon_names)} if step > 0 else {}
        # the param-group keys are whatever this torch's Adam writes (they changed across releases); values = Adam defaults
        group = dict(torch.optim.Adam([torch.nn.Parameter(torch.zeros(1))], lr=lr).state_dict()["param_groups"][0])
        group["params"] = list(range(n_frozen_first + len(canon_names)))
        return {"state": state, "param_groups": [group]}

    def _canon(self, nets):
        out = []
        for net in nets:
            out += list(self._key_map(net).values())
        return out

    def _load_adam(self, sd, canon_names, slot, n_frozen_first=0):
        m, v, step = {}, {}, 0
        for i, n in enumerate(canon_names):
            st = sd["state"].get(n_frozen_first + i)
            if st is None:
                continue
            m[n], v[n] = st["exp_avg"], st["exp_avg_sq"]
            step = int(st["step"])
        if m:
            self.core.set_named(m, _lib.ADAM_M, strict=False)
            self.core.set_named(v, _lib.ADAM_V, strict=False)
        steps = list(self.core.get_steps())
        steps[slot] = step
        self.core.set_steps(steps)

    def _checkpoint_path(self, idx):
        return os.path.join(self.save_model_path, f"checkpoint_{idx}.tar")

    def save_checkpoint(self, episode_idx):
        named = self.core.get_named()
        sc, sa, sl = self.core.get_steps()[:3]
        # LL / VSAC write 'episode_idx' (LL/learner.py:146, VS:148); MTSAC / CARE / MT1-CARE write and READ 'update_iteration'
        # (MS/learner.py:159,178; C10:180,202; C1:147,169)
        state = {self._iteration_key: episode_idx, "total_step": self.total_step}
        state.update(self._critic_checkpoint_entries(named))
        state["critic_optimizer"] = self._adam_state_dict(self._canon(self._critic_nets), self.lr_critic, sc)
        state["actor"] = self._module_state_dict("actor", named=named)
        state["actor_optimizer"] = self._adam_state_dict(self._canon(("actor",)), self.lr_actor, sa)
        state["log_alpha"] = named["log_alpha"].clone()
        state["log_alpha_optimizer"] = self._adam_state_dict(["log_alpha"], self.lr_actor, sl)
        state["alpha"] = self.alpha.clone()
        os.makedirs(self.save_model_path, exist_ok=True)
        path = self._checkpoint_path(episode_idx)
        torch.save(state, path)
        return path

    def load_checkpoint(self, path):
        ck = torch.load(path, map_location="cpu", weights_only=False)
        self.episode_idx = ck.get("episode_idx", ck.get("update_iteration", 0))
        self.total_step = ck.get("total_step", 0)
        self._load_critic_checkpoint_entries(ck)
        self._load_module_state_dict("actor", ck["actor"])
        self.core.set_named({"log_alpha": ck["log_alpha"].detach().reshape(-1)}, strict=False)
        self._load_adam(ck["critic_optimizer"], self._canon(self._critic_nets), 0)
        self._load_adam(ck["actor_optimizer"], self._canon(("actor",)), 1)
        self._load_adam(ck["log_alpha_optimizer"], ["log_alpha"], 2)
        if "alpha" in ck:
            self.alpha = ck["alpha"].detach().reshape(-1).clone()
        if self.critic_dropout is not None:         # the rate is a setting of the learner, not part of the checkpoint
            self.core.set_critic_dropout(self.critic_dropout)

    # ---- Redis-facing loop (LL/learner.py:191-201,278-316) -------------------------------------
    def write(self, update_iteration, critic_loss, actor_loss, entropy=None, log_alpha=None):
        self.server.rpush("critic_loss", _pickle.dumps((update_iteration, critic_loss)))
        self.server.rpush("actor_loss", _pickle.dumps((update_iteration, actor_loss)))
        if entropy is not None:
            self.server.rpush("entropy", _pickle.dumps((update_iteration, entropy)))
        alphas = np.exp(np.array(log_alpha, dtype=np.float32)) if log_alpha is not None else self.log_alpha.exp().numpy()
        self.server.rpush("alpha", _pickle.dumps((update_iteration, alphas)))

    def run(self, max_updates=None):
        self.server.set("update_iteration", _pickle.dumps(-1))
        self.server.set("parameters", self.parameters_blob(blocking=True))
        self.wait_until_memoryReady()
        self.my_print("######################### Start train #########################")
        self.soft_update(None, None, 1.0)           # copy parameters to target
        # Pipelined like this: while the GPU runs step k+1 (enqueued together with the assembly of its blob), the host hands
        # blob k to Redis -- the reference does the same things strictly one after the other (learner.py:296-316).  Two
        # blob images in the library make that safe.
        done = 0
        iters = (i for i in itertools.count() if i % self.update_delay == 0)
        update_iteration = next(iters)
        core = self.core
        for _ in self._chunks(1):
            self.memory.enqueue_step(core)             # update(), split so that everything below overlaps the GPU
        core.blob_begin()
        while True:
            cur = update_iteration
            res = self._loss_tuple(core.read_losses(1)[0])             # step `cur` has finished
            last = max_updates is not None and done + 1 >= max_updates
            if cur % self.save_period == 0:
                self.save_checkpoint(cur)              # before step cur+1 is enqueued: the arena is the state after `cur`
            if not last:                               # the GPU goes on with step cur+1 while blob `cur` is still crossing PCIe
                update_iteration = next(iters)
                for _ in self._chunks(1):              # a scheduled reset lands after checkpoint `cur` and blob `cur`
                    self.memory.enqueue_step(core)
                core.blob_begin()
            blob, extra = core.blob_wait()             # the OLDEST uncollected blob = the one of step `cur`
            self.server.set("update_iteration", _pickle.dumps(cur))
            self.server.set("parameters", blob)
            if self.write_mode:
                self.write(cur, *res, log_alpha=extra["log_alpha"])
                if cur % self.print_period == 0:
                    self.my_print("[Learner] Update_iteration: {0:<6} \t | actor_loss : {1:5.3f} \t | critic_loss : {2:5.3f}".format(
                        cur, res[1], res[0]))
            done += 1
            if last:
                return done


class _TwoCriticMixin:
    """LL / VS: separate Critic modules in the checkpoint, local_critic_k and target_critic_k for k = 1, 2 (1 .. E with
    critic_ensemble=E)."""

    def _critic_entries(self):
        return [(f"{side}_critic_{k}", f"q{k}" + ("_target" if side == "target" else ""))
                for side in ("local", "target") for k in range(1, self.n_critics + 1)]

    def _critic_checkpoint_entries(self, named):
        return {k: self._module_state_dict(net, named=named) for k, net in self._critic_entries()}

    def _load_critic_checkpoint_entries(self, ck):
        self._check_checkpoint_critics({int(m.group(1)) for m in (re.fullmatch(r"local_critic_(\d+)", k) for k in ck) if m})
        for k, net in self._critic_entries():
            self._load_module_state_dict(net, ck[k])

    def __getattr__(self, name):
        # local_critic_k / target_critic_k for every critic k of an ensemble (1 and 2 are the properties below)
        m = re.fullmatch(r"(local|target)_critic_(\d+)", name)
        E = self.__dict__.get("critic_ensemble") or 2
        if m and 1 <= int(m.group(2)) <= E:
            return _Handle(self, f"q{m.group(2)}" + ("_target" if m.group(1) == "target" else ""))
        raise AttributeError(name)

    @property
    def local_critic_1(self): return _Handle(self, "q1")
    @property
    def local_critic_2(self): return _Handle(self, "q2")
    @property
    def target_critic_1(self): return _Handle(self, "q1_target")
    @property
    def target_critic_2(self): return _Handle(self, "q2_target")
    @property
    def actor(self): return _Handle(self, "actor")


class LunarLanderLearner(_TwoCriticMixin, _BaseLearner):
    """LunarLander_Distributed_SAC/src/learner.py: Learner(cfg_path, update_delay=3, print_period=10,
    write_mode=True, save_period=1000, checkpoint_path=None)."""
    family = "LL"
    log_name = "LunarLander_Distributed_SAC"

    def __init__(self, cfg_path, update_delay=3, print_period=10, write_mode=True, save_period=1000,
                 checkpoint_path=None, *, server=None, device_index=0, seed=0, replay_where="host", buffer_size=None,
                 precision=1, prioritized=None, actor_update_interval=1, target_update_interval=1, n_step=1, max_grad_norm=None,
                 pcgrad=False, cagrad=None, reset_interval=None, reset=None, redo_interval=None, redo=None,
                 critic_layer_norm=False, critic_dropout=None, prior=None,
                 critic_ensemble=None, target_subset=2, actor_q="mean"):
        self.update_delay, self.print_period = update_delay, print_period
        self._buffer_size_override = buffer_size
        self._init_common(cfg_path, write_mode, save_period, checkpoint_path, server, device_index, seed, replay_where,
                          precision, prioritized, actor_update_interval, target_update_interval, n_step, max_grad_norm, pcgrad,
                          cagrad, reset_interval, reset, redo_interval, redo, critic_layer_norm, critic_dropout,
                          prior, critic_ensemble=critic_ensemble, target_subset=target_subset, actor_q=actor_q)

    def _set_dims(self):
        c = self.cfg
        self.gamma, self.lr_actor, self.lr_critic = c["gamma"], c["lr_actor"], c["lr_critic"]
        self.batch_size, self.tau, self.reward_scale = int(c["batch_size"]), c["tau"], c["reward_scale"]
        self.start_memory_len = c["start_memory_len"]
        self.buffer_size = int(self._buffer_size_override or 1e5)      # LL/learner.py:72
        self.action_dim, self.state_dim, self.action_bound = 2, 8, [-1.0, 1.0]     # LL/learner.py:79-81
        self.actor_hidden_dim, self.critic_hidden_dim = [256, 256], [256, 256]     # LL/learner.py:102-107
        self.num_tasks, self.use_weighted_loss = 0, False

    def _make_memory(self, where):
        return ReplayBuffer(self.buffer_size, self.batch_size, 0, self.device, server=self.server, core=self.core,
                            where=where, prioritized=self.prioritized, n_step=self.n_step)


class VSACLearner(_TwoCriticMixin, _BaseLearner):
    """MT1_Distributed_VSAC/src/learner.py: Learner(cfg_path, write_mode, save_period, checkpoint_path)."""
    family = "VS"
    log_name = "MT1_Distributed_VSAC"

    def __init__(self, cfg_path, write_mode=True, save_period=1000, checkpoint_path=None, *, server=None,
                 device_index=0, seed=0, replay_where="host", precision=1, prioritized=None, actor_update_interval=1,
                 target_update_interval=1, n_step=1, max_grad_norm=None, pcgrad=False, cagrad=None, reset_interval=None, reset=None,
                 redo_interval=None, redo=None, critic_layer_norm=False, critic_dropout=None, prior=None,
                 critic_ensemble=None, target_subset=2, actor_q="mean"):
        self._init_common(cfg_path, write_mode, save_period, checkpoint_path, server, device_index, seed, replay_where,
                          precision, prioritized, actor_update_interval, target_update_interval, n_step, max_grad_norm, pcgrad,
                          cagrad, reset_interval, reset, redo_interval, redo, critic_layer_norm, critic_dropout,
                          prior, critic_ensemble=critic_ensemble, target_subset=target_subset, actor_q=actor_q)

    def _set_dims(self):
        c = self.cfg
        self.gamma, self.lr_actor, self.lr_critic = c["gamma"], c["lr_actor"], c["lr_critic"]
        self.batch_size, self.tau, self.reward_scale = int(c["batch_size"]), c["tau"], c["reward_scale"]
        self.start_memory_len, self.buffer_size = c["start_memory_len"], int(c["buffer_size"])
        self.print_period, self.update_delay = int(c["print_period_learner"]), c["update_delay"]
        self.actor_hidden_dim, self.critic_hidden_dim = c["actor_hidden_dim"], c["critic_hidden_dim"]
        self.action_dim, self.state_dim, self.action_bound = 4, 39, [-1.0, 1.0]    # VS/learner.py:80-82
        self.num_tasks, self.use_weighted_loss = 0, False

    def _make_memory(self, where):
        return ReplayBuffer(self.buffer_size, self.batch_size, 0, self.device, server=self.server, core=self.core,
                            where=where, prioritized=self.prioritized, n_step=self.n_step)


class MTSACLearner(_BaseLearner):
    """MT10_Distributed_MTSAC/src/learner.py: Learner(train_classes, train_tasks, cfg_path, write_mode,
    save_period, checkpoint_path).  One learner over T tasks, one-hot appended to the state."""
    family = "MS"
    log_name = "MT10_Distributed_MTSAC"
    _iteration_key = "update_iteration"
    _pcgrad_ok = True

    def __init__(self, train_classes, train_tasks, cfg_path, write_mode=True, save_period=1000, checkpoint_path=None,
                 *, server=None, device_index=0, seed=0, replay_where="host", precision=1, prioritized=None,
                 actor_update_interval=1, target_update_interval=1, n_step=1, max_grad_norm=None, pcgrad=False,
                 cagrad=None, reset_interval=None, reset=None, redo_interval=None, redo=None, critic_layer_norm=False,
                 critic_dropout=None, prior=None,
                 critic_ensemble=None, target_subset=2, actor_q="mean"):
        self.train_classes, self.train_tasks = train_classes, train_tasks
        self._init_common(cfg_path, write_mode, save_period, checkpoint_path, server, device_index, seed, replay_where,
                          precision, prioritized, actor_update_interval, target_update_interval, n_step, max_grad_norm, pcgrad,
                          cagrad, reset_interval, reset, redo_interval, redo, critic_layer_norm, critic_dropout,
                          prior, critic_ensemble=critic_ensemble, target_subset=target_subset, actor_q=actor_q)

    def _set_dims(self):
        c = self.cfg
        self.actor_cfg, self.critic_cfg = c["actor"], c["critic"]
        self.gamma = c["gamma"]
        self.lr_actor, self.lr_critic = self.actor_cfg["lr_actor"], self.critic_cfg["lr_critic"]
        self.batch_size, self.tau, self.reward_scale = int(c["batch_size"]), c["tau"], c["reward_scale"]
        self.start_memory_len, self.buffer_size = c["start_memory_len"], int(c["buffer_size"])
        self.print_period, self.update_delay = int(c["print_period_learner"]), c["update_delay"]
        self.num_tasks = int(c["num_tasks"])
        self.use_weighted_loss = bool(c.get("use_weighted_loss", False))
        self.state_dim, self.action_dim = int(self.actor_cfg["state_dim"]), int(self.actor_cfg["action_dim"])
        self.action_bound = self.actor_cfg["action_bound"]
        self.actor_hidden_dim = self.actor_cfg["actor_hidden_dim"]
        self.critic_hidden_dim = self.critic_cfg["critic_hidden_dim"]

    def _make_memory(self, where):
        return MTReplayBuffer(self.buffer_size, self.batch_size, 0, self.device, self.num_tasks, server=self.server,
                              core=self.core, where=where, prioritized=self.prioritized, n_step=self.n_step)

    def _critic_checkpoint_entries(self, named):
        # one Critic module holding Q_function_1 .. Q_function_E
        loc, tgt = {}, {}
        for q in self._critic_nets:
            loc.update(self._module_state_dict(q, named=named))
            tgt.update(self._module_state_dict(q + "_target", named=named))
        return {"local_critic": loc, "target_critic": tgt}

    def _load_critic_checkpoint_entries(self, ck):
        if self._critic_ln_ok:                     # (CARE's Critic also holds its state encoder, keyed differently)
            self._check_checkpoint_critics({int(m.group(1)) for m in (re.match(r"Q_function_(\d+)\.", k) for k in ck["local_critic"]) if m})
        for net in self._critic_nets:
            self._load_module_state_dict(net, ck["local_critic"])
            self._load_module_state_dict(net + "_target", ck["target_critic"])

    def get_log_alpha(self, mtobss):
        """(batch, 1) log_alpha of each row's task (MS/learner.py:213-233)."""
        one_hots = torch.as_tensor(mtobss)[:, -self.num_tasks:].float().cpu()
        return one_hots @ self.log_alpha.reshape(-1, 1)


class EncoderConfigError(KeyError, ValueError):
    """A CARE cfg whose 'encoder' block lacks keys the learner needs (a KeyError, as the lookup raised before, and a
    ValueError, as every other bad constructor argument raises)."""


class CARELearner(MTSACLearner):
    """MT10_Distributed_CARE/src/learner.py with `use_modified_care: true` (CARE(M)):
    Learner(train_classes, train_tasks, cfg_path, write_mode, save_period, checkpoint_path).

    One actor / twin-Q critic over the encoded state [mlp_context(z) | attention-mixed K encoders(state)],
    z = frozen RoBERTa embedding of the task (cfg 'encoder' block; metadata JSONs are read relative to the
    working directory exactly like context_encoder.py:31-36).  The actor's state encoder is a hard copy of the
    critic's after every update (learner.py:402), so it is exported from the same tensors."""
    family = "C10"
    log_name = "MT10_Distributed_CARE"
    _critic_ln_ok = False
    # the 'encoder' keys _core_config reads without a default
    _encoder_keys = ("num_encoders", "hidden_dims_mixtureEnc", "output_dim_mixtureEnc", "hidden_dims_contextEnc",
                     "output_dim_contextEnc", "embedding_dim_contextEnc", "lr_contextEnc")

    def _set_dims(self):
        super()._set_dims()
        c = self.cfg
        self.use_modified_care = bool(c.get("use_modified_care", False))
        self.use_weighted_loss = self.use_modified_care    # learner.py:313,349: use_weighted_loss = use_modified_care
        self.encoder_cfg = c["encoder"]
        missing = [k for k in self._encoder_keys if k not in self.encoder_cfg]
        if missing:             # before any other check, so an incomplete cfg fails the same way with or without pcgrad
            raise EncoderConfigError(f"cfg 'encoder' block lacks {missing}")

    def _core_config(self):
        cc = super()._core_config()
        e = self.encoder_cfg
        cc.care = True
        cc.num_encoders = int(e["num_encoders"])
        cc.mix_hidden = [int(x) for x in e["hidden_dims_mixtureEnc"]]
        cc.mix_out = int(e["output_dim_mixtureEnc"])
        cc.ctx_in = int(e.get("RoBERTa_embedding_dim", 768))      # MT1_Distributed_CARE's cfg has no such key (width of the JSON rows)
        cc.ctx_hidden = [int(x) for x in e["hidden_dims_contextEnc"]]
        cc.ctx_out = int(e["output_dim_contextEnc"])
        cc.tau_se = float(e.get("state_encoder_tau", 0.05))        # hard-coded 0.05 in MT1_Distributed_CARE/src/learner.py:311
        cc.care_original = not self.use_modified_care     # CARE(O): trainable context encoder with its own Adam
        cc.emb_dim = int(e["embedding_dim_contextEnc"])
        cc.lr_ctx = float(e["lr_contextEnc"])
        return cc

    def _init_common(self, *a, **kw):
        super()._init_common(*a, **kw)
        e = self.encoder_cfg
        emb_path, names_path = e.get("pretrained_embedding_json_path"), e.get("task_name_json_path")
        if emb_path and names_path and not (os.path.exists(emb_path) and os.path.exists(names_path)):
            # the reference fails fast here (context_encoder.py:31-36 opens both files); training on the random
            # stand-in table would publish meaningless context vectors without any error
            if not os.environ.get("B200SAC_ALLOW_RANDOM_EMBEDDING"):
                raise FileNotFoundError(f"CARE task-embedding files not found (cwd {os.getcwd()}): {emb_path}, {names_path}; "
                                        "set B200SAC_ALLOW_RANDOM_EMBEDDING=1 to train on a random embedding table")
        if emb_path and names_path and os.path.exists(emb_path) and os.path.exists(names_path):
            table, order = cfg_read(emb_path), cfg_read(names_path)
            E = torch.tensor([table[n] for n in order], dtype=torch.float32)       # context_encoder.py:43-47
            if E.shape != (self.num_tasks, self.core.cfg.ctx_in):
                raise ValueError(f"pretrained embedding has shape {tuple(E.shape)}, cfg says ({self.num_tasks}, {self.core.cfg.ctx_in})")
            self.core.set_named({"embedding": E}, strict=False)

    def _enc_map(self, prefix):
        cc = self.core.cfg
        n_ctx = len(cc.ctx_hidden) + 1 if self.use_modified_care else 0      # CARE(O) has no mlp_context in the state encoder
        return names.care_encoder_key_map(len(cc.mix_hidden) + 1, len(cc.mix_hidden) + 1, n_ctx, prefix)

    def _cenc_map(self):
        """CARE(O) context encoder keys: embedding = Sequential(Embedding, ReLU, header[Linear, ReLU, Linear, ReLU]),
        mlp = build_mlp(...) (context_encoder.py:59-89)."""
        m = {"embedding.2.0.weight": "cenc.0.weight", "embedding.2.0.bias": "cenc.0.bias",
             "embedding.2.2.weight": "cenc.1.weight", "embedding.2.2.bias": "cenc.1.bias"}
        for j in range(len(self.core.cfg.ctx_hidden) + 1):
            for kind in ("weight", "bias"):
                m[f"mlp.{2 * j}.{kind}"] = f"cenc.{2 + j}.{kind}"
        return m

    def _key_map(self, net):
        if net == "context_encoder":
            km = {"embedding.0.weight": "embedding"}
            if not self.use_modified_care:
                km.update(self._cenc_map())
            return km
        if net == "actor":            # policy MLP + the tied copy of the critic's state encoder
            return {**names.actor_key_map("MS", len(self.actor_hidden_dim) + 1), **self._enc_map("cse")}
        if net in ("critic_se", "target_se"):
            return self._enc_map("cse" if net == "critic_se" else "tse")
        which = 1 if "1" in net else 2
        return names.critic_key_map("MS", len(self.critic_hidden_dim) + 1, which, target="target" in net)

    _published = ("context_encoder", "actor")      # C10/learner.py:412-417

    def _critic_checkpoint_entries(self, named):
        d = super()._critic_checkpoint_entries(named)
        d["local_critic"].update(self._module_state_dict("critic_se", named=named))
        d["target_critic"].update(self._module_state_dict("target_se", named=named))
        d["context_encoder"] = self._module_state_dict("context_encoder", named=named)
        # Adam(context_encoder.parameters()): parameter 0 is the frozen embedding (no state); CARE(M) has nothing else, the
        # reference still saves -- and its load_checkpoint indexes -- the (empty) optimizer state (C10/learner.py:184,206)
        cenc = [] if self.use_modified_care else list(self._cenc_map().values())
        step = 0 if self.use_modified_care else self.core.get_steps()[3]
        d["context_encoder_optimizer"] = self._adam_state_dict(cenc, self.core.cfg.lr_ctx, step, n_frozen_first=1)
        return d

    def _load_critic_checkpoint_entries(self, ck):
        super()._load_critic_checkpoint_entries(ck)
        self._load_module_state_dict("critic_se", ck["local_critic"])
        self._load_module_state_dict("target_se", ck["target_critic"])
        if "context_encoder" in ck:
            self._load_module_state_dict("context_encoder", ck["context_encoder"])
        if not self.use_modified_care and "context_encoder_optimizer" in ck:
            self._load_adam(ck["context_encoder_optimizer"], list(self._cenc_map().values()), 3, n_frozen_first=1)

    def _canon(self, nets):
        out = []
        for net in nets:
            if net == "actor":        # actor_optimizer holds mu_log_std_layer only (learner.py:146-149)
                out += list(names.actor_key_map("MS", len(self.actor_hidden_dim) + 1).values())
            else:
                out += list(self._key_map(net).values())
        if tuple(nets) == ("q1", "q2"):   # critic_optimizer = local_critic.parameters(): state encoder first (learner.py:150-153)
            out = list(self._enc_map("cse").values()) + out
        return out


# the reference modules all call their class `Learner`
Learner = LunarLanderLearner
