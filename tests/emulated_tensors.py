"""b2s_pit_train_pack in numpy, for the CPU suite (tests only): the emulated training set of tests/emulated_train.py, its
kept rows packed into a [kept, F] matrix with the conversions of the pack kernel -- numpy's own casts, which round to
nearest; NaN where a set found no row; bool and the BOOL kind as 0 / 1 -- and the label vector (floats at their width,
ints as int64, bools as bool).  `install(monkeypatch)` puts it behind mlrun_b200.feature_store.offline; the arrays it hands
out are numpy arrays.  The CUDA kernel is compared with get_offline_features in tests/test_gpu_training_tensors.py."""

import numpy as np

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import offline
from tests import emulated_train


def _source(joined, permuted, feat):
    s, j, _width, _kind = feat
    return (joined[s][0][j], joined[s][2]) if s >= 0 else (permuted[j], None)


def pit_train_pack(ts, sets, cols, label, feats, label_vec, dtype):
    order, joined, permuted, _miss, stats = emulated_train.pit_train(ts, sets, cols, label, with_stats=True)
    x = np.empty((len(order), len(feats)), dtype)
    for i, feat in enumerate(feats):
        values, found = _source(joined, permuted, feat)
        with np.errstate(over="ignore"):  # float64 past float32's range: inf, as the device's conversion gives
            x[:, i] = (values != 0) if feat[3] == nat.PIT_FEAT_BOOL else values
        if found is not None:
            x[~found, i] = np.nan
    y = None
    if label_vec is not None:
        values, _found = _source(joined, permuted, label_vec)
        y = values.astype(offline._label_dtype(label_vec)) if label_vec[3] != nat.PIT_FEAT_BOOL else values != 0
    return x, y, order, dict(stats, sort_ms=0.0, join_ms=0.0, compact_ms=0.0, pack_ms=0.0)


def install(monkeypatch):
    emulated_train.install(monkeypatch)
    monkeypatch.setattr(offline, "pit_train_pack", pit_train_pack)
