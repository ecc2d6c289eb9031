"""Stitch an interleaved drain of single transitions back into trajectories.

The players of the reference push (state, action, reward, next_state, done) one at a time into one Redis list, so two
neighbouring entries of a drain are in general not consecutive steps of one episode, and nothing in an entry says which
player it came from.  What identifies a continuation is the data itself: a transition continues the open trajectory whose
last next_state equals its state, byte for byte.  A `done` closes the trajectory; after a time-limit reset the new state
matches no open tail, so a new trajectory starts and no link crosses the reset.  No change to the players is needed.
"""
from collections import OrderedDict

import numpy as np


class Stitcher:
    """assign() gives every row of a drain a stream id for Replay.push(stream=...): rows of one trajectory share an id.

    Ids are recycled.  A `done` closes the stream in the ring as well, so its id is free at once.  A tail that is given up
    here while the ring still holds it open (evicted as the oldest of more than max_open, or no longer distinguishable) must
    be closed there before its id names another trajectory: take_abandoned() lists those ids for Replay.close_streams()
    after the push, and they become reusable with the next assign()."""

    def __init__(self, max_open=4096, n_ids=65536):
        self.max_open = int(max_open)
        self._tails = OrderedDict()          # next_state bytes of an open tail -> stream id (oldest first)
        self._free = []                      # ids of closed streams, reused before new ones
        self._abandoned = []                 # ids given up since the last take_abandoned()
        self._closing = []                   # ids handed out by take_abandoned(): free from the next assign() on
        self._next = 0
        self._n_ids = int(n_ids)

    def _new_id(self):
        if self._free:
            return self._free.pop()
        if self._next >= self._n_ids:
            raise RuntimeError("out of stream ids")
        self._next += 1
        return self._next - 1

    def assign(self, states, next_states, dones) -> np.ndarray:
        states = np.ascontiguousarray(states, dtype=np.float32)
        next_states = np.ascontiguousarray(next_states, dtype=np.float32)
        dones = np.asarray(dones).reshape(-1)
        out = np.empty(len(dones), dtype=np.int32)
        self._free.extend(self._closing)
        self._closing = []
        for i in range(len(dones)):
            sid = self._tails.pop(states[i].tobytes(), None)
            if sid is None:
                sid = self._new_id()
            out[i] = sid
            if dones[i]:
                self._free.append(sid)       # the ring closes the stream at d != 0: the id can serve a new trajectory
                continue
            key = next_states[i].tobytes()
            old = self._tails.pop(key, None)
            if old is not None:              # two open tails end in the same state: the older one can no longer be told apart
                self._abandoned.append(old)
            self._tails[key] = sid
            if len(self._tails) > self.max_open:
                _, ev = self._tails.popitem(last=False)
                self._abandoned.append(ev)
        return out

    def take_abandoned(self):
        """Stream ids to close in the ring (Replay.close_streams) before the next assign()."""
        ids, self._abandoned = self._abandoned, []
        self._closing.extend(ids)
        return ids

    @property
    def open_tails(self):
        return len(self._tails)
