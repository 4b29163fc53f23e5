"""The online table's hash layout restated in numpy (csrc/b2s_hash.cuh, b2s_table_create), so that tests can build tables
whose probe chains are laid out on purpose.

mix64 is the splitmix64 finaliser; every step of it is a bijection of 64-bit words, so `unmix64` undoes it and a key with
any wanted home slot (mix64(key) & (cap - 1)) is `unmix64` of a word with those low bits.
"""

import numpy as np

M1, M2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
M1_INV, M2_INV = pow(M1, -1, 1 << 64), pow(M2, -1, 1 << 64)


def _u64(x):
    a = np.atleast_1d(np.asarray(x))
    return a if a.dtype == np.uint64 else a.astype(np.int64).view(np.uint64)


def mix64(keys):
    """mix64 of int64 / uint64 keys, as uint64"""
    x = _u64(keys).copy()
    x ^= x >> np.uint64(30)
    x *= np.uint64(M1)
    x ^= x >> np.uint64(27)
    x *= np.uint64(M2)
    x ^= x >> np.uint64(31)
    return x


def _unxorshift(y, s):
    """x with x ^ (x >> s) == y: each pass fixes s more of the high bits"""
    x = y.copy()
    for _ in range(64 // s):
        x = y ^ (x >> np.uint64(s))
    return x


def unmix64(y):
    """the inverse of mix64, as int64 keys"""
    x = _u64(y).copy()
    x = _unxorshift(x, 31)
    x *= np.uint64(M2_INV)
    x = _unxorshift(x, 27)
    x *= np.uint64(M1_INV)
    x = _unxorshift(x, 30)
    return x.view(np.int64)


def capacity(n_keys):
    """slots of a table of n_keys keys: the smallest power of two >= 2 n_keys, at least 16 (load factor <= 0.5)"""
    cap = 16
    while cap < 2 * n_keys:
        cap *= 2
    return cap


def home_slot(keys, cap):
    return (mix64(keys) & np.uint64(cap - 1)).astype(np.int64)


def keys_with_home_slots(slots, cap, rng, exclude=()):
    """distinct int64 keys, key i homed at slots[i] of a table of `cap` slots, none of them in `exclude`"""
    slots = np.asarray(slots, dtype=np.uint64)
    assert cap & (cap - 1) == 0 and (slots < np.uint64(cap)).all()
    exclude = set(int(k) for k in exclude)
    while True:
        hi = rng.integers(0, 1 << 63, size=len(slots), dtype=np.int64).view(np.uint64) << np.uint64(1)
        hi |= rng.integers(0, 2, size=len(slots), dtype=np.int64).view(np.uint64)
        keys = unmix64((hi & ~np.uint64(cap - 1)) | slots)
        if len(set(keys.tolist())) == len(keys) and not exclude.intersection(keys.tolist()):
            return keys


def probe_layout(keys, cap):
    """slot -> key after inserting `keys` in order with linear probing, as b2s_table_create does"""
    table = {}
    for k, h in zip(keys.tolist(), home_slot(keys, cap).tolist()):
        while h in table:
            h = (h + 1) % cap
        table[h] = k
    return table
