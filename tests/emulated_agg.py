"""b2s_agg_run_host in numpy, for the CPU suite (tests only): `install(monkeypatch)` puts it behind
mlrun_b200.feature_store.ingest.aggregate_host so that the host layer -- names, column order, dtypes, index, key encoding,
refusals -- runs without a GPU.  It is also a second restatement of the semantics, independent of oracle/aggregate.py: rows
grouped by key with a stable sort, each row's window start found with searchsorted on its key's times.  The CUDA kernels are
compared with the oracle in tests/test_gpu_aggregate.py; nothing in mlrun_b200 imports this."""

import numpy as np

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import ingest

_INT64_MIN = -(1 << 63)
_BITS = sorted(nat.AGG_OPS.items(), key=lambda kv: kv[1])


def window_starts(ts, window_ns, period_ns):
    """first timestamp of each row's window (clamped at INT64_MIN), from Python integers"""
    out = np.empty(len(ts), dtype=np.int64)
    for i, t in enumerate(ts.tolist()):
        p = period_ns or window_ns
        first_bucket = t // p - (window_ns // period_ns - 1 if period_ns else 0)
        out[i] = max(first_bucket * p, _INT64_MIN)
    return out


def _value(x, op):
    n = len(x)
    if op == "count":
        return float(n)
    if op in ("sum", "avg"):
        s = float(np.sum(x))
        return s if op == "sum" else s / n
    if op == "sqr":
        return float(np.sum(x * x))
    if op in ("max", "min"):
        return float(x.max() if op == "max" else x.min())
    if op in ("first", "last"):
        return float(x[0] if op == "first" else x[-1])
    if n < 2:
        return np.nan
    var = float(np.var(x, ddof=1))
    return var if op == "stdvar" else float(np.sqrt(var))


def aggregate_host(keys, ts, specs, n):
    keys, ts = np.asarray(keys, np.int64), np.asarray(ts, np.int64)
    order = np.argsort(keys, kind="stable")
    ks, tss = keys[order], ts[order]
    run_start = np.searchsorted(ks, ks, side="left")
    late = int(sum(1 for i in range(1, n) if run_start[i] < i and tss[i] < tss[i - 1]))
    nat_rows = int((ts == _INT64_MIN).sum())
    seen, nans = set(), 0
    for src, kind, *_rest in specs:
        if id(src) not in seen and kind == nat.COL_F32:
            nans += int(np.isnan(src).sum())
        seen.add(id(src))
    for src, _kind, ops, period_ns, windows_ns, outs in specs:
        x = np.asarray(src, np.float64)[order]
        names = [name for name, bit in _BITS if ops & bit]
        for w, window_ns in enumerate(windows_ns):
            starts = window_starts(tss, window_ns, period_ns)
            for i in range(n):
                lo = run_start[i] + np.searchsorted(tss[run_start[i]:i + 1], starts[i], side="left")
                win = x[lo:i + 1]
                for j, op in enumerate(names):
                    outs[j * len(windows_ns) + w][order[i]] = _value(win, op)
    return np.array([late, nat_rows, nans], dtype=np.uint64), {"rows": n, "kernels": 0}


def install(monkeypatch):
    monkeypatch.setattr(ingest, "aggregate_host", aggregate_host)
