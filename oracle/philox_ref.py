"""Philox4x32-10 in numpy uint32 and the critic dropout masks drawn from it -- TEST INFRASTRUCTURE, NOT PRODUCT.

philox(key, counter) restates distributed_sac_b200/csrc/common.cuh's Philox (Salmon et al., SC 2011; Random123's
philox4x32 with 10 rounds): key (k0, k1) = the low and high 32 bits of the 64-bit seed, counter (c0, c1, c2, c3), four
32-bit output words.  It is vectorised over any broadcastable counter arrays.

drop_masks(...) is the keep mask of include/b200sac.h "Dropout Q-functions":
  key     = seed ^ (0xE7037ED1A0B428DB * (replica + 1)) mod 2^64;
  counter = (step & 0xFFFFFFFF, step >> 32, row, (tag << 24) | (j // 4)),  tag = (pass * 8 + layer) * nets + net
            (nets = 2 for the twin critics, E for a critic ensemble);
  keep    = word[j % 4] >= floor(p * 2^32).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
DROP_KEY_MUL = 0xE7037ED1A0B428DB
PASSES = {"cur": 0, "next": 1, "pi": 2}      # A: critics on (s, a); B: targets on (s', a'); D: critics on (s, a~)
_MASK32 = np.uint64(0xFFFFFFFF)


def philox(seed, c0, c1, c2, c3):
    """Philox4x32-10 of counters (c0, c1, c2, c3) under the 64-bit seed: four uint32 arrays."""
    seed = int(seed) & (2 ** 64 - 1)
    k0, k1 = np.uint32(seed & 0xFFFFFFFF), np.uint32(seed >> 32)
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, np.uint32) for c in (c0, c1, c2, c3)))
    c0, c1, c2, c3 = (c.astype(np.uint32).copy() for c in (c0, c1, c2, c3))
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0.astype(np.uint64)
            p1 = M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _MASK32).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _MASK32).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = k0 + W0, k1 + W1
    return c0, c1, c2, c3


def drop_key(seed, replica):
    return (int(seed) ^ (DROP_KEY_MUL * (int(replica) + 1))) & (2 ** 64 - 1)


def threshold(p):
    """t = floor(p * 2^32) in fp64: an element is dropped iff its word < t."""
    return int(np.floor(float(p) * 4294967296.0))


def scale(p):
    """s = (float)(1 / (1 - p)), evaluated in fp64 and rounded once."""
    return np.float32(1.0 / (1.0 - float(p)))


def drop_masks(seed, replica, step, pass_, layer, net, B, H, p, nets=2):
    """The keep mask [B][H] (bool) of one (step, replica, pass, layer, net); pass_ in {0, 1, 2} or "cur"/"next"/"pi".
    nets: the critics of the handle (2 for the twins, E for a critic ensemble), tag = (pass * 8 + layer) * nets + net."""
    pass_ = PASSES.get(pass_, pass_)
    tag = (int(pass_) * 8 + int(layer)) * int(nets) + int(net)
    j = np.arange(H)
    rows = np.arange(B, dtype=np.uint32)[:, None]
    step = int(step)
    words = philox(drop_key(seed, replica), np.uint32(step & 0xFFFFFFFF), np.uint32(step >> 32), rows,
                   ((tag << 24) | (j // 4)).astype(np.uint32)[None, :])
    return np.choose(j % 4, words) >= np.uint32(threshold(p))
