"""CPU: the properties of the ReDo restatement (redo_ref) that the device record and recycle are checked against: scores
are scale-free, an all-zero layer is all dormant, NaN is never dormant, and recycling exactly the dead neurons leaves the
fp64 network output unchanged."""
import numpy as np
import pytest

import redo_ref as rr


def _table(nets):
    """A layout table {name: (offset, rows, cols, trainable, opt, pitch)} of MLPs {net: [in, h0, ..., out]}, first weight
    rows padded to a multiple of 4 as the library lays them out."""
    table, off = {}, 0
    for net, dims in nets.items():
        for l in range(len(dims) - 1):
            cols = dims[l]
            pitch = (cols + 3) // 4 * 4 if l == 0 else cols
            for name, rows, c, p in ((f"{net}.{l}.weight", dims[l + 1], cols, pitch), (f"{net}.{l}.bias", dims[l + 1], 1, 1)):
                table[name] = (off, rows, c, 1, 0, p)
                off += (rows * p + 3) // 4 * 4
    return table, off


def _arena(table, n, rng):
    a = np.zeros(n, np.float32)
    for name, (off, rows, cols, _t, _o, pitch) in table.items():
        a[off:off + rows * pitch].reshape(rows, pitch)[:, :cols] = rng.standard_normal((rows, cols)) * (cols ** -0.5)
    return a


@pytest.mark.parametrize("k", [1e-6, 0.37, 1.0, 8.0, 1e6])
def test_scores_do_not_change_when_a_layer_is_scaled(k):
    rng = np.random.default_rng(3)
    h = np.maximum(rng.standard_normal((64, 40)), 0.0)
    h[:, 5] = 0.0
    s = rr.scores(h)
    np.testing.assert_allclose(rr.scores(k * h), s, rtol=1e-12, atol=0)
    assert s[5] == 0.0 and abs(s.mean() - 1.0) < 1e-12


def test_an_all_zero_layer_is_all_dormant():
    s = rr.scores(np.zeros((16, 9)))
    assert np.array_equal(s, np.zeros(9)) and rr.dormant(s, 0.0).all()
    assert not rr.dormant(s, -1e-300).any() and not rr.dormant(s, -np.inf).any()


def test_nan_is_never_dormant():
    rng = np.random.default_rng(4)
    h = np.maximum(rng.standard_normal((32, 6)), 0.0)
    h[3, 2] = np.nan
    s = rr.scores(h)
    assert np.isnan(s).all()                     # the NaN reaches the mean, so every score is NaN
    assert not rr.dormant(s, np.inf).any()
    h[3, 2] = 0.0
    h[:, 4] = np.nan
    s = rr.scores(h)
    assert not rr.dormant(s, 1e30).any()


def test_negative_activations_count_as_zero():
    h = np.array([[-1.0, 2.0], [-3.0, 4.0]])
    np.testing.assert_array_equal(rr.scores(h), [0.0, 2.0])


@pytest.mark.parametrize("seed", range(4))
def test_recycling_exactly_dead_neurons_keeps_the_output(seed):
    rng = np.random.default_rng(seed)
    nets = {"actor": [13, 48, 32, 6], "q1": [16, 40, 24, 1], "q2": [16, 40, 24, 1]}
    table, n = _table(nets)
    arena = _arena(table, n, rng)
    theta0 = _arena(table, n, rng)
    m, v = rng.standard_normal(n).astype(np.float32), rng.random(n).astype(np.float32)
    x = {"actor": rng.standard_normal((50, 13)), "q1": rng.standard_normal((50, 16))}
    x["q2"] = x["q1"]
    for net, dims in nets.items():                 # kill some neurons of every hidden layer on every input
        for l in range(len(dims) - 2):
            dead = rng.choice(dims[l + 1], size=3 + seed, replace=False)
            off = table[f"{net}.{l}.bias"][0]
            arena[off + dead] = -1e3
    masks = {net: [rr.dormant(rr.scores(h), 0.0) for h in rr.hidden(arena, table, net, x[net])] for net in nets}
    assert all(m_.sum() >= 3 + seed for ms in masks.values() for m_ in ms)
    new, m2, v2 = rr.recycle(arena, m, v, table, masks, theta0)
    for net in nets:
        np.testing.assert_array_equal(rr.output(new, table, net, x[net]), rr.output(arena, table, net, x[net]))
        after = rr.hidden(new, table, net, x[net])
        assert any((h[:, ms] > 0).any() for h, ms in zip(after, masks[net])), "the recycled neurons stayed dead"
    # the recycle touched exactly the flagged rows, their biases and outgoing columns, and m, v there
    changed = np.flatnonzero((new != arena) | (m2 != m) | (v2 != v))
    allowed = set()
    for net, ms in masks.items():
        for l, mask in enumerate(ms):
            i = np.flatnonzero(mask)
            off, _r, cols, _t, _o, pitch = table[f"{net}.{l}.weight"]
            allowed |= set((off + i[:, None] * pitch + np.arange(cols)).reshape(-1).tolist())
            allowed |= set((table[f"{net}.{l}.bias"][0] + i).tolist())
            noff, nrows, _c, _t, _o, npitch = table[f"{net}.{l + 1}.weight"]
            allowed |= set((noff + np.arange(nrows)[:, None] * npitch + i).reshape(-1).tolist())
    assert set(changed.tolist()) <= allowed
    assert not m2[sorted(allowed)].any() and not v2[sorted(allowed)].any()


def test_recycle_draws_win_over_outgoing_zeros():
    table, n = _table({"q1": [4, 5, 6, 1]})
    rng = np.random.default_rng(9)
    arena, theta0 = _arena(table, n, rng), _arena(table, n, rng)
    z = np.zeros(n, np.float32)
    masks = {"q1": [np.array([1, 0, 0, 0, 1], bool), np.array([0, 1, 0, 0, 0, 0], bool)]}
    new, _, _ = rr.recycle(arena, z, z, table, masks, theta0)
    off, _r, cols, _t, _o, pitch = table["q1.1.weight"]
    W1 = new[off:off + 6 * pitch].reshape(6, pitch)
    T1 = theta0[off:off + 6 * pitch].reshape(6, pitch)
    np.testing.assert_array_equal(W1[1], T1[1])             # flagged row: the draw, its flagged-column entries included
    assert not W1[[0, 2, 3, 4, 5]][:, [0, 4]].any()
    off = table["q1.2.weight"][0]
    assert new[off + 1] == 0.0 and new[off] == arena[off]
