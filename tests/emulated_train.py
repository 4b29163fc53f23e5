"""b2s_pit_train_host in numpy, for the CPU suite (tests only): the emulated join of tests/emulated_pit.py, then the rows a
training set keeps -- every exact-key set matched, the label present -- and the misses per set among the rows the
exact-key sets before it matched.  `install(monkeypatch)` puts it and the emulated index behind
mlrun_b200.feature_store.offline.  The CUDA kernels are compared with the oracle in tests/test_gpu_training_set.py."""

import numpy as np

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import offline
from tests import emulated_pit


def pit_train(ts, sets, cols, label, with_stats=False):
    order, joined, permuted, _miss = emulated_pit.pit_join(ts, sets, cols)
    alive = np.ones(len(order), bool)
    miss = []
    for (_ix, _keys, asof, _outs), (_arrays, _ts_out, found) in zip(sets, joined):
        miss.append(int((alive & ~found).sum()))
        if not asof:
            alive &= found
    keep = alive
    if label is not None:
        s, j, kind = label
        values = joined[s][0][j] if s >= 0 else permuted[j]
        if s >= 0:
            keep = keep & joined[s][2]
        if kind == nat.PIT_LABEL_NAN:
            keep = keep & ~np.isnan(values)
        elif kind == nat.PIT_LABEL_NAT:
            keep = keep & (values.view(np.int64) != offline._NAT)
    res = (order[keep], [([a[keep] for a in arrays], t[keep], f[keep]) for arrays, t, f in joined], [p[keep] for p in permuted],
           np.array(miss, np.uint64))
    return res + ({"rows": len(order), "kernels": 0, "kept": int(keep.sum())},) if with_stats else res


def install(monkeypatch):
    emulated_pit.install(monkeypatch)
    monkeypatch.setattr(offline, "pit_train", pit_train)
