"""Dormant-neuron recycling (ReDo; Sokar, Agarwal, Castro, Evci, ICML 2023) restated in numpy fp64, as include/b200sac.h
defines b200sac_redo: the neuron scores of a hidden layer, the dormant masks, the hidden forward of a network from a
parameter arena, and the recycle of a parameter arena and its Adam moments given the layout table and theta0 (the arena
b200sac_create(seed) draws)."""
import numpy as np

NETS = ("actor", "q1", "q2")        # the order of the record


def scores(h):
    """s_i of one hidden layer from its activations h [n][H]: a_i = (1/n) sum_rows max(h_ri, 0) (a NaN stays NaN),
    s_i = a_i / mean_j a_j, and every s_i = 0 when that mean is 0."""
    h = np.asarray(h, np.float64)
    a = np.where(h < 0.0, 0.0, h).mean(axis=0)
    mean = a.mean()
    return np.zeros_like(a) if mean == 0.0 else a / mean


def dormant(s, tau):
    """Neuron i is dormant iff s_i <= tau; a NaN score never is, and a negative tau flags nothing."""
    return np.asarray(s, np.float64) <= tau


def _weight(arena, table, name):
    off, rows, cols, _t, _o, pitch = table[name]
    return arena[off:off + rows * pitch].reshape(rows, pitch)[:, :cols]


def hidden(arena, table, net, x):
    """The hidden activations [relu(x W0^T + b0), ...] of network `net` ("actor", "q1", "q2") in fp64, x [n][in]."""
    out, h, l = [], np.asarray(x, np.float64), 0
    while f"{net}.{l + 1}.weight" in table:
        W = _weight(arena, table, f"{net}.{l}.weight").astype(np.float64)
        b = _weight(arena, table, f"{net}.{l}.bias").reshape(-1).astype(np.float64)
        h = np.maximum(h @ W.T + b, 0.0)
        out.append(h)
        l += 1
    return out


def output(arena, table, net, x):
    """The network's output layer (no activation) in fp64."""
    h = hidden(arena, table, net, x)
    l = len(h)
    W = _weight(arena, table, f"{net}.{l}.weight").astype(np.float64)
    b = _weight(arena, table, f"{net}.{l}.bias").reshape(-1).astype(np.float64)
    return h[-1] @ W.T + b


def recycle(arena, m, v, table, masks, theta0):
    """(arena, m, v) after recycling the neurons `masks` flags: {net: [bool [H] per hidden layer]}.  For flagged neuron i
    of layer l: row i of W_l = theta0's (pad columns untouched), b_l[i] = 0, column i of W_{l+1} = 0 except in rows the
    next hidden layer flags, which keep theta0's draw, and m = v = 0 at every one of those entries.  Copies; the inputs are
    not changed."""
    arena, m, v = (np.array(x, np.float32, copy=True) for x in (arena, m, v))
    writes = []                                    # incoming rows, drawn after every zeroing so that the draws win
    for net, ms in masks.items():
        for l, mask in enumerate(ms):
            i = np.flatnonzero(mask)
            if i.size == 0:
                continue
            off, _rows, cols, _t, _o, pitch = table[f"{net}.{l}.weight"]
            noff, nrows, _c, _t, _o, npitch = table[f"{net}.{l + 1}.weight"]
            for idx in (noff + np.arange(nrows)[:, None] * npitch + i[None, :], table[f"{net}.{l}.bias"][0] + i):
                arena[idx] = 0.0
                m[idx] = v[idx] = 0.0
            writes.append((off, cols, pitch, i))
    for off, cols, pitch, i in writes:
        idx = (off + i[:, None] * pitch + np.arange(cols)[None, :]).reshape(-1)
        arena[idx] = theta0[idx]
        m[idx] = v[idx] = 0.0
    return arena, m, v
