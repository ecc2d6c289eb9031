"""numpy reference of prioritized replay's sum-tree (include/b200sac.h, per_kernels.cuh).

Leaves p_i = (prio_i + eps)^alpha in fp32 (the power in fp64, rounded once), internal nodes fp32 sums of their two children
over a tree padded to a power of two, importance weights w_i = (N p_i / S)^-beta divided by their batch maximum (fp64,
rounded once).  ImportanceWeights applies the weights to the autograd oracles' critic update.
"""
import numpy as np
import torch

import sac_port as sp


def td_priority(y, q1, q2):
    """(|y - Q1| + |y - Q2|) / 2 in fp64 from the step's fp32 y, Q1, Q2."""
    y, q1, q2 = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (y, q1, q2))
    return 0.5 * (np.abs(y - q1) + np.abs(y - q2))


def leaf_values(prio, alpha, eps):
    return np.power(np.asarray(prio, dtype=np.float64) + eps, alpha).astype(np.float32)


def build_tree(leaves, n_leaves=None):
    """Heap-ordered fp32 sum-tree (node 1 = root, leaf i = node P + i) over `leaves`, padded with zeros to P = 2^k."""
    leaves = np.asarray(leaves, dtype=np.float32)
    P = 1
    while P < max(len(leaves), n_leaves or 1):
        P *= 2
    tree = np.zeros(2 * P, dtype=np.float32)
    tree[P:P + len(leaves)] = leaves
    lo = P
    while lo > 1:
        lo //= 2
        tree[lo:2 * lo] = tree[2 * lo:4 * lo:2] + tree[2 * lo + 1:4 * lo:2]
    return tree


def root(leaves):
    return build_tree(leaves)[1]


U_MAX = 1.0 - 2.0 ** -53          # the largest U(0, 1) the sampler draws (53 random bits)


def descend(tree, u):
    """per_sample_kernel's descent of one draw through a heap-ordered fp32 tree from the fp64 offset u: into the left child
    while u < its sum, else into the right child with u reduced by the left sum (fp64); a zero-sum child is never entered,
    so rounding in u cannot reach an empty slot.  When both children are 0 -- a zero root -- it goes right at every level
    and ends on leaf P - 1.  Returns the leaf index in [0, P)."""
    P = len(tree) // 2
    node, u = 1, float(u)
    while node < P:
        lv, rv = tree[2 * node], tree[2 * node + 1]
        if lv > 0 and (u < float(lv) or not rv > 0):
            node = 2 * node
        else:
            u -= float(lv)
            node = 2 * node + 1
    return node - P


def stratified_draw(tree, per, U):
    """The leaves drawn by a task's per batch slots: slot j descends from u = (j + U[j]) S / per (S = the root, fp64)."""
    S = float(tree[1])
    return np.array([descend(tree, (j + float(U[j])) * S / per) for j in range(per)], dtype=np.int64)


def strata(tree, per):
    """(lo, hi): the lowest and highest leaf slot j of a task can draw, over every U in [0, 1).  The descent is monotone in
    u, so a draw of slot j lies in [lo[j], hi[j]] whatever its U."""
    return stratified_draw(tree, per, np.zeros(per)), stratified_draw(tree, per, np.full(per, U_MAX))


def is_weights(p, S, N, beta):
    """Batch-max-normalised importance weights of leaf values p drawn from trees with root sums S and fills N."""
    raw = np.power(np.asarray(N, dtype=np.float64) * np.asarray(p, dtype=np.float32).astype(np.float64)
                   / np.asarray(S, dtype=np.float32).astype(np.float64), -float(beta))
    return (raw / raw.max()).astype(np.float32)


def sample_probabilities(leaves):
    """p_i / S: the probability of drawing slot i in one draw (stratification leaves the marginal unchanged)."""
    p = np.asarray(leaves, dtype=np.float64)
    return p / p.sum()


class _GradScale(torch.autograd.Function):
    """Identity forward; the gradient is multiplied per row by w on the way back."""

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(w)
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        (w,) = ctx.saved_tensors
        return g * w, None


class ImportanceWeights:
    """Inside this context the autograd oracles' critic update (sac_port.PortLearner.update_SAC, care_port.CarePortLearner
    .update) is importance-weighted like the prioritized CUDA step: the gradient that reaches the (s, a) heads Q1, Q2 (tag
    "cur") from the critic loss is multiplied by w per row, dQk = (2c (Qk - y)) w.  Everything upstream follows; the actor
    and temperature losses are untouched.  The oracles' reported critic_loss stays the unweighted one: weighted_critic_loss
    gives the weighted value from their intermediates."""

    def __init__(self, w):
        self.w = torch.as_tensor(np.asarray(w, dtype=np.float32)).reshape(-1, 1)

    def __enter__(self):
        self._mlp = sp.mlp
        w, inner = self.w, sp.mlp

        def mlp(params, net, x, tag=None):
            out = inner(params, net, x, tag)
            return _GradScale.apply(out, w) if tag == "cur" and net in ("q1", "q2") else out

        sp.mlp = mlp
        return self

    def __exit__(self, *exc):
        sp.mlp = self._mlp
        return False


def weighted_critic_loss(out, w, weighted_loss=False):
    """mean(w (y - Q1)^2) / div + mean(w (y - Q2)^2) / div (fp64) from an oracle step's intermediates y, q1, q2."""
    y, q1, q2 = (np.asarray(out[k], dtype=np.float64).reshape(-1) for k in ("y", "q1", "q2"))
    w = np.asarray(w, dtype=np.float64).reshape(-1)
    div = float(len(y)) if weighted_loss else 1.0
    return float((w * (y - q1) ** 2).mean() / div + (w * (y - q2) ** 2).mean() / div)
