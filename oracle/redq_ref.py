"""The critic ensemble's target-subset draw in numpy -- TEST INFRASTRUCTURE, NOT PRODUCT.

subset(...) restates include/b200sac.h "Critic ensembles" with oracle/philox_ref.py's Philox4x32-10:
  m >= E: every critic, no draw;
  key     = seed ^ (0x8EBC6AF09C88C6E3 * (replica + 1)) mod 2^64;
  counter = (step & 0xFFFFFFFF, step >> 32, 0, q) -> words w_{4q} .. w_{4q+3};
  S       = the m indices k with the smallest pairs (w_k, k).
"""
import numpy as np

import philox_ref as pr

ENS_KEY_MUL = 0x8EBC6AF09C88C6E3


def ens_key(seed, replica):
    return (int(seed) ^ (ENS_KEY_MUL * (int(replica) + 1))) & (2 ** 64 - 1)


def words(seed, replica, step, E):
    """w_0 .. w_{E-1} of one step of one replica (uint32)."""
    q = np.arange((E + 3) // 4, dtype=np.uint32)
    c = pr.philox(ens_key(seed, replica), np.uint32(step & 0xFFFFFFFF), np.uint32(step >> 32), np.uint32(0), q)
    return np.stack(c, 1).reshape(-1)[:E]


def subset(seed, replica, step, E, m):
    """bool [E]: the critics whose targets the step's TD target takes the min over."""
    if m >= E:
        return np.ones(E, bool)
    w = words(seed, replica, step, E)
    order = sorted(range(E), key=lambda k: (int(w[k]), k))
    out = np.zeros(E, bool)
    out[order[:m]] = True
    return out
