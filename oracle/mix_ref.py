"""The device replay draw in numpy: sample_indices_kernel and sample_mixed_kernel -- TEST INFRASTRUCTURE, NOT PRODUCT.

draw(step, replica, batch, num_tasks, m, online, prior) restates include/b200sac.h "Prior-data rings": with
P = batch / num_tasks (batch when num_tasks = 0), slot i of task block t = i // P draws from the prior when i - tP < m, else
from the online ring.  A slot of ring X (seed, per-task fill, cap_per_task) draws
    key     = X.seed + 0x9E3779B97F4A7C15 * (replica + 1)  mod 2^64,
    counter = (step & 0xFFFFFFFF, step >> 32, i, attempt),
    local   = ((w0 << 32) | w1) % fill[t],  index = t * cap_per_task + local.
Rounds: every unresolved slot draws; an index already won in an earlier round is lost by every slot that draws it, and
among the slots that draw a free index in one round the lowest wins it; the others redraw with attempt + 1 (at most 64
rounds; the last draw stays).  Online and prior indices are separate spaces.  Output (int32): online index k as k, prior
index k as -1 - k.  With m = 0 this is the plain draw of the online ring (sample_indices_kernel).
"""
from collections import namedtuple

import numpy as np

from philox_ref import philox

DRAW_KEY_MUL = 0x9E3779B97F4A7C15
MAX_ROUNDS = 64

Ring = namedtuple("Ring", "seed fill cap_per_task")     # fill: the replica's per-task fill [max(num_tasks, 1)]


def draw_key(seed, replica):
    return (int(seed) + DRAW_KEY_MUL * (int(replica) + 1)) % 2 ** 64


def _draws(ring, replica, step, slots, att, tasks):
    w = philox(draw_key(ring.seed, replica), np.uint32(step & 0xFFFFFFFF), np.uint32(step >> 32),
               slots.astype(np.uint32), att.astype(np.uint32))
    r64 = (w[0].astype(np.uint64) << np.uint64(32)) | w[1].astype(np.uint64)
    fill = np.asarray(ring.fill, np.uint64)[tasks]
    return tasks.astype(np.int64) * int(ring.cap_per_task) + (r64 % fill).astype(np.int64)


def draw(step, replica, batch, num_tasks, m, online, prior=None):
    """The [batch] encoded indices (int32) one step with step counter `step` draws for `replica`."""
    Teff = max(int(num_tasks), 1)
    P = batch // Teff
    if m and prior is None:
        raise ValueError("m > 0 needs a prior ring")
    i_all = np.arange(batch)
    task = np.minimum(i_all // P, Teff - 1)
    from_prior = (i_all - (i_all // P) * P) < m
    att = np.zeros(batch, np.int64)
    done = np.zeros(batch, bool)
    out = np.zeros(batch, np.int64)
    won = set()                                  # ("o" | "p", index) already owned
    for _ in range(MAX_ROUNDS):
        todo = np.flatnonzero(~done)
        if todo.size == 0:
            break
        key = np.empty(todo.size, np.int64)
        for part, ring in (("o", online), ("p", prior)):
            sel = from_prior[todo] if part == "p" else ~from_prior[todo]
            if sel.any():
                key[sel] = _draws(ring, replica, step, todo[sel], att[todo[sel]], task[todo[sel]])
        claimed = {}
        lost = False
        for i, k in zip(todo, key):              # ascending slots: the lowest slot of a round takes a free index
            tag = ("p" if from_prior[i] else "o", int(k))
            out[i] = -1 - k if from_prior[i] else k
            if tag in won or tag in claimed:
                att[i] += 1
                lost = True
            else:
                claimed[tag] = i
                done[i] = True
        won.update(claimed)
        if not lost:
            break
    return out.astype(np.int32)


def decode(idx):
    """(from_prior [B] bool, ring index [B] int64) of encoded indices."""
    idx = np.asarray(idx, np.int64)
    return idx < 0, np.where(idx < 0, -1 - idx, idx)
