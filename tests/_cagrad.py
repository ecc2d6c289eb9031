"""Gram matrices the CAGrad tests solve on the host and on the device."""
import numpy as np


def gram_sets():
    """(T, kind, G): random Gram matrices at T in {2, 3, 10, 50, 64}, rank-deficient ones and one task with a zero
    gradient, each with a c."""
    rng = np.random.default_rng(11)
    out = []
    for T in (2, 3, 10, 50, 64):
        for kind in ("random", "conflict", "rank", "zero"):
            n = 3 * T + 5
            g = rng.standard_normal((T, n))
            if kind == "conflict":
                g[1::2] = -0.8 * g[0::2][: T // 2] + 0.2 * rng.standard_normal((T // 2, n))
            if kind == "rank":                  # rank 1 (T = 2) or about T / 2
                basis = rng.standard_normal((max(1, T // 2), n))
                g = rng.standard_normal((T, basis.shape[0])) @ basis
            if kind == "zero":
                g[T - 1] = 0.0
            c = (0.5, 0.1, 0.9, 2.0)[len(out) % 4]
            out.append((T, kind, c, g @ g.T))
    return out
