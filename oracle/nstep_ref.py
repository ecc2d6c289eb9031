"""Reference for n-step returns on the replay ring: the push-time link rules and the sample-time fold.

RingModel restates, in numpy, what b200sac_replay_push / _push_traj do to one replica's ring: rows bucketed by task,
appended to each task's sub-ring with wrap (a push larger than a sub-ring keeps only its newest rows), and the
trajectory links
    link[task][slot] = sub-ring-local slot of the transition that followed this one in its trajectory, or -1
maintained incrementally with the stream rule and the overwrite rule of include/b200sac.h.  fold() is the n-step fold
in fp32 with the device's operation order:
    j = i;  R = r_j;  g = gamma;  m = 1
    while d_j == 0 and m < n and link[j] >= 0:   j = link[j];  R = R + g * r_j;  g = g * gamma;  m += 1
TrajectoryModel is the brute-force statement of the invariant the links must satisfy, with no incremental state: it
remembers which pushed row sits in which slot and which row truly followed which.
"""
import numpy as np


def _slots(task, cap_t, head):
    """Slot of every row of one push (or -1 for a row a larger-than-the-ring push drops), and the new heads."""
    task = np.asarray(task, dtype=np.int64)
    slot = np.full(len(task), -1, dtype=np.int64)
    head = list(head)
    for t in np.unique(task):
        rows = np.nonzero(task == t)[0]
        skip = max(0, len(rows) - cap_t)
        for k, i in enumerate(rows[skip:]):
            slot[i] = (head[t] + k) % cap_t
        head[t] = (head[t] + len(rows) - skip) % cap_t
    return slot, head


class RingModel:
    def __init__(self, capacity, num_tasks=0):
        self.T = max(int(num_tasks), 1)
        self.cap_t = int(capacity) // self.T
        self.link = np.full((self.T, self.cap_t), -1, dtype=np.int32)
        self.pred = np.full((self.T, self.cap_t), -1, dtype=np.int32)
        self.head = [0] * self.T
        self.fill = [0] * self.T
        self.tail = {}                   # stream id -> (task, slot) of its open tail
        self.r = np.zeros((self.T, self.cap_t), np.float32)
        self.d = np.zeros((self.T, self.cap_t), np.float32)
        self.tag = np.full((self.T, self.cap_t), -1, dtype=np.int64)     # caller's row tag (e.g. index into its own table)

    def push(self, task, r, d, stream=None, cut=None, tag=None):
        n = len(task)
        slot, new_head = _slots(task, self.cap_t, self.head)
        for i in range(n):
            sid = -1 if stream is None else int(stream[i])
            if slot[i] < 0:
                self.tail.pop(sid, None)
                continue
            t, j = int(task[i]), int(slot[i])
            p, nx = self.pred[t, j], self.link[t, j]
            if p >= 0 and self.link[t, p] == j:
                self.link[t, p] = -1
            if nx >= 0 and self.pred[t, nx] == j:
                self.pred[t, nx] = -1
            for k in [k for k, v in self.tail.items() if v == (t, j)]:
                del self.tail[k]
            self.link[t, j] = self.pred[t, j] = -1
            self.r[t, j], self.d[t, j] = r[i], d[i]
            self.tag[t, j] = -1 if tag is None else tag[i]
            if sid < 0:
                continue
            prev = self.tail.pop(sid, None)
            if prev is not None and prev[0] == t:
                self.link[t, prev[1]] = j
                self.pred[t, j] = prev[1]
            if d[i] == 0 and not (cut is not None and cut[i]):
                self.tail[sid] = (t, j)
        for t in range(self.T):
            self.fill[t] = min(self.cap_t, self.fill[t] + int(np.sum(np.asarray(task) == t)))
        self.head = new_head
        return slot

    def filled(self):
        """Ring indices (task * cap_t + slot) of every filled slot."""
        return np.concatenate([t * self.cap_t + np.arange(self.fill[t]) for t in range(self.T)]).astype(np.int64)

    def fold(self, idx, n, gamma):
        return fold(self.r.reshape(-1), self.d.reshape(-1), self.link.reshape(-1), self.cap_t, idx, n, gamma)


def fold(r, d, link, cap_t, idx, n, gamma):
    """(R, disc, d, last, m) per index: fp32, R + g * r with two roundings, g * gamma."""
    r, d = np.asarray(r, np.float32), np.asarray(d, np.float32)
    g0 = np.float32(gamma)
    R, disc, dd = np.empty(len(idx), np.float32), np.empty(len(idx), np.float32), np.empty(len(idx), np.float32)
    last, m = np.empty(len(idx), np.int64), np.empty(len(idx), np.int32)
    for k, i in enumerate(np.asarray(idx, dtype=np.int64)):
        base, j = i - i % cap_t, int(i)
        acc, g, hops = np.float32(r[j]), g0, 1
        while d[j] == 0 and hops < n and link[j] >= 0:
            j = int(base + link[j])
            acc = np.float32(acc + np.float32(g * r[j]))
            g = np.float32(g * g0)
            hops += 1
        R[k], disc[k], dd[k], last[k], m[k] = acc, g, d[j], j, hops
    return R, disc, dd, last, m


def nstep_return_f64(rewards, dones, gamma, n):
    """Textbook n-step return of the first transition of a trajectory given as lists (fp64): (sum_k gamma^k r_k, gamma^m,
    d of the last hop, m)."""
    R, m = 0.0, 0
    for k in range(min(n, len(rewards))):
        R += float(gamma) ** k * float(rewards[k])
        m = k + 1
        if dones[k]:
            break
    return R, float(gamma) ** m, float(dones[m - 1]), m


class TrajectoryModel:
    """Brute force: every pushed row gets a serial number, succ[serial] = the serial of the row that truly followed it in
    its stream (none after a terminal or cut row), and at[task][slot] = the serial now stored there.  links() derives the
    table from the invariant alone: link[i] = j iff the row at j is the successor of the row at i, same sub-ring."""

    def __init__(self, capacity, num_tasks=0):
        self.T = max(int(num_tasks), 1)
        self.cap_t = int(capacity) // self.T
        self.at = np.full((self.T, self.cap_t), -1, dtype=np.int64)
        self.head = [0] * self.T
        self.succ = {}
        self.open = {}                   # stream id -> serial of its last row, if that row can have a successor
        self.serial = 0

    def push(self, task, d, stream=None, cut=None):
        slot, self.head = _slots(task, self.cap_t, self.head)
        for i in range(len(task)):
            me = self.serial
            self.serial += 1
            if stream is not None:
                sid = int(stream[i])
                prev = self.open.pop(sid, None)
                # a dropped row never was in the ring: the chain is broken on both sides of it
                if prev is not None and slot[i] >= 0:
                    self.succ[prev] = me
                if slot[i] >= 0 and d[i] == 0 and not (cut is not None and cut[i]):
                    self.open[sid] = me
            if slot[i] >= 0:
                self.at[int(task[i]), slot[i]] = me

    def links(self):
        out = np.full((self.T, self.cap_t), -1, dtype=np.int32)
        for t in range(self.T):
            where = {int(s): j for j, s in enumerate(self.at[t]) if s >= 0}
            for j, s in enumerate(self.at[t]):
                nxt = self.succ.get(int(s)) if s >= 0 else None
                if nxt is not None and nxt in where:
                    out[t, j] = where[nxt]
        return out
