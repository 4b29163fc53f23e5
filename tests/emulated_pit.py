"""The b2s_pit index and join in numpy, for the CPU suite (tests only): `install(monkeypatch)` puts them behind
mlrun_b200.feature_store.offline so that its host layer -- naming, aliases, dtype rules, row order, refusals -- runs without a
GPU.  The CUDA kernels are compared with the oracle in tests/test_gpu_offline.py; nothing in mlrun_b200 imports this."""

import numpy as np

from mlrun_b200.feature_store import offline


class EmulatedPitIndex:
    """rows sorted by (key, timestamp), equal pairs in input order; features as rows of 4-byte words"""

    def __init__(self, keys, ts_ns, cols):
        keys, ts_ns = np.asarray(keys, np.int64), np.asarray(ts_ns, np.int64)
        perm = np.lexsort((np.arange(len(keys)), ts_ns, keys))
        self.keys, self.ts = keys[perm], ts_ns[perm]
        words = [np.ascontiguousarray(c).view(np.uint32).reshape(len(keys), -1) for c in cols]
        self.rows = np.concatenate(words, axis=1)[perm] if words else np.zeros((len(keys), 0), np.uint32)
        _u, counts = np.unique(keys, return_counts=True)
        self.n_rows, self.n_keys, self.longest_run, self.row_words = len(keys), len(counts), int(counts.max()), self.rows.shape[1]

    def close(self):
        pass


def _last_le(ix, k, t):
    """index position of the last row of key k with ts <= t (vector bisection), -1 where there is none"""
    lo = np.searchsorted(ix.keys, k, side="left")
    hi = np.searchsorted(ix.keys, k, side="right")
    start = lo.copy()
    while (lo < hi).any():
        act = lo < hi
        mid = (lo + hi) // 2
        le = np.zeros(len(k), bool)
        le[act] = ix.ts[mid[act]] <= t[act]
        lo = np.where(act & le, mid + 1, lo)
        hi = np.where(act & ~le, mid, hi)
    return np.where(lo > start, lo - 1, -1)


def pit_join(ts, sets, cols, with_stats=False):
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    order = np.argsort(ts, kind="stable") if ts is not None else np.arange(n)
    t = ts[order] if ts is not None else np.zeros(n, np.int64)
    joined, misses = [], []
    for ix, keys, asof, outs in sets:
        k = np.asarray(keys, np.int64)[order]
        if asof:
            pos = _last_le(ix, k, t)
        else:
            lo = np.searchsorted(ix.keys, k)
            pos = np.where((lo < len(ix.keys)) & (ix.keys[np.minimum(lo, len(ix.keys) - 1)] == k), lo, -1)
        found = pos >= 0
        safe = np.maximum(pos, 0)
        arrays = []
        for w, dt, miss in outs:
            dt = np.dtype(dt)
            if dt.itemsize == 4:
                v = np.where(found, ix.rows[safe, w], np.uint32(miss & 0xFFFFFFFF)).astype(np.uint32)
            else:
                v = ix.rows[safe, w].astype(np.uint64) | (ix.rows[safe, w + 1].astype(np.uint64) << np.uint64(32))
                v = np.where(found, v, np.uint64(miss & 0xFFFFFFFFFFFFFFFF)).astype(np.uint64)
            arrays.append(v.view(dt))
        ts_out = np.where(found, ix.ts[safe], offline._NAT)
        joined.append((arrays, ts_out, found))
        misses.append(int((~found).sum()))
    res = (order.astype(np.int64), joined, [np.asarray(c)[order] for c in cols], np.array(misses, np.uint64))
    return res + ({"rows": n, "kernels": 0},) if with_stats else res


def install(monkeypatch):
    monkeypatch.setattr(offline, "PitIndex", EmulatedPitIndex)
    monkeypatch.setattr(offline, "pit_join", pit_join)
