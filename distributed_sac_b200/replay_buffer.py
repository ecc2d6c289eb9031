"""Drop-in `ReplayBuffer`: the reference's thread + sample() surface over the native ring.

  ReplayBuffer   <- LunarLander_Distributed_SAC/src/replay_buffer.py:13-77 (= VSAC)
  MTReplayBuffer <- MT10_Distributed_MTSAC/src/replay_buffers.py:13-107

The daemon thread drains the Redis list 'sample' exactly like the reference
(pipeline lrange + ltrim, pickled tuples) but appends into the C++ ring
(b200sac_replay_push: pinned host DRAM or HBM) instead of a deque of namedtuples;
`sample()` returns the same five fp32 tensors on `device`; `len()` is the fill
(min over tasks for the MT variant).  The ring takes its own lock, which fixes the
reference's unlocked sample()-vs-append race (SURVEY.md §5).
"""
import pickle as _pickle
import threading
import time

import numpy as np
import torch

from .core import Replay
from .stitch import Stitcher


class ReplayBuffer(threading.Thread):
    def __init__(self, buffer_size, batch_size, seed, device, server=None, *, core=None, where="host", prioritized=None,
                 n_step=1):
        super().__init__()
        self.daemon = True
        if core is None:
            raise ValueError("ReplayBuffer needs the learner's SacCore (core=...) to own its ring")
        if core.cfg.batch != int(batch_size):
            raise ValueError("batch_size must match the learner's batch")
        self.server = server
        if self.server is not None:
            self.server.delete("sample")
        self.batch_size = int(batch_size)
        self.device = torch.device(device)
        self.core = core
        # n_step > 1: the ring keeps trajectory links and the steps train on n-step returns.  The players push single
        # transitions, interleaved, so add_many stitches every drain back into trajectories (stitch.Stitcher)
        self.n_step = int(n_step)
        self.seed = int(seed)
        self.ring = Replay(core, int(buffer_size), where=where, seed=self.seed, prioritized=prioritized,
                           trajectories=self.n_step > 1)
        self.prior = None               # attach_prior: the prior-data ring
        self.stitcher = Stitcher() if self.n_step > 1 else None
        if self.n_step > 1:
            self.ring.set_nstep(self.n_step)
        self._stop_evt = threading.Event()

    # ---- ingestion (reference: run(), replay_buffer.py:43-61) -------------------------------
    def _unpack(self, data):
        state, action, reward, next_state, done = data
        return state, action, reward, next_state, done

    def add_many(self, states, actions, rewards, next_states, dones):
        n = len(rewards)
        f = lambda x, w: np.asarray(x, dtype=np.float32).reshape(n, w)
        c = self.core.cfg
        s, s2, d = f(states, c.obs_dim), f(next_states, c.obs_dim), f(np.asarray(dones).astype(np.uint8), 1)
        stream = None if self.stitcher is None else self.stitcher.assign(s, s2, d)
        self.ring.push(s, f(actions, c.act_dim), f(rewards, 1), s2, d, stream=stream)
        if self.stitcher is not None:
            self.ring.close_streams(self.stitcher.take_abandoned())

    def attach_prior(self, capacity):
        """A prior-data device ring of `capacity` transitions beside the online ring, attached to it.  Its seed is the online
        ring's + 1, so the two rings draw different indices."""
        self.prior = Replay(self.core, int(capacity), where="device", seed=self.seed + 1)
        self.ring.attach_prior(self.prior)

    def add_prior(self, states, actions, rewards, next_states, dones):
        """Append rows to the prior ring (add_many's layout; no trajectories)."""
        n = len(rewards)
        f = lambda x, w: np.asarray(x, dtype=np.float32).reshape(n, w)
        c = self.core.cfg
        self.prior.push(f(states, c.obs_dim), f(actions, c.act_dim), f(rewards, 1), f(next_states, c.obs_dim),
                        f(np.asarray(dones).astype(np.uint8), 1))

    def prior_ready(self):
        """False while steps take prior rows and a task of the prior holds fewer than 4 per-task batches (the step's rule)."""
        if self.prior is None or self.ring.get_prior_rows() == 0:
            return True
        return self.prior.size() >= 4 * (self.batch_size // max(self.core.cfg.num_tasks, 1))

    def drain_once(self):
        pipe = self.server.pipeline()
        pipe.lrange("sample", 0, -1)
        pipe.ltrim("sample", -1, 0)
        datas, _ = pipe.execute()
        if datas:
            rows = [self._unpack(_pickle.loads(d)) for d in datas]
            self.add_many(*[[r[i] for r in rows] for i in range(5)])
        return len(datas) if datas else 0

    def run(self):
        while not self._stop_evt.is_set():
            if self.server is not None:
                self.drain_once()
            time.sleep(0.01)

    def stop(self):
        self._stop_evt.set()

    # ---- sampling --------------------------------------------------------------------------
    def sample(self):
        """(states, actions, rewards, next_states, dones) fp32 on `device` (replay_buffer.py:63-73).  A prioritized ring
        draws with ring.sample_prioritized() instead (which also returns the indices and importance weights: call it
        directly to get them)."""
        batch = self.ring.sample() if self.ring.prioritized is None else self.ring.sample_prioritized()[:5]
        return tuple(t.to(self.device, non_blocking=False) for t in batch)

    def enqueue_step(self, core):
        """sample + one gradient step, fused in the library (pinned staging, side-stream H2D); asynchronous."""
        core.step_sampled(self.ring, 1)

    def step_core(self, core):
        """Learner.update(): sample + step + losses (critic, actor, alpha, entropy) as python floats, one library call."""
        return core.update_sampled(self.ring)

    def __len__(self):
        return self.ring.size()


class MTReplayBuffer(ReplayBuffer):
    """ReplayBuffer(buffer_size, batch_size, seed, device, num_tasks, server): one sub-ring per task,
    B/T samples from each, then one shuffle (MS/replay_buffers.py:67-100)."""

    def __init__(self, buffer_size, batch_size, seed, device, num_tasks, server=None, *, core=None, where="host",
                 prioritized=None, n_step=1):
        if core is not None and core.cfg.num_tasks != int(num_tasks):
            raise ValueError("num_tasks must match the learner's")
        super().__init__(buffer_size, batch_size, seed, device, server, core=core, where=where, prioritized=prioritized,
                         n_step=n_step)
        self.num_tasks = int(num_tasks)

    def _unpack(self, data):
        _task_idx, state, action, reward, next_state, done = data      # the one-hot inside `state` carries the task
        return state, action, reward, next_state, done
