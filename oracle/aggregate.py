"""Windowed aggregations of feature-set ingest, restated as a per-row walk (the checker of b2s_agg.cu).

storey.AggregateByKey is not in the reference tree; its behaviour under FeatureSet.add_aggregation (feature_set.py:715-851,
docs/feature-store/transformations.md:89-147) is restated here, emitting every event:

- row i gains, per (operation, window), the aggregate over the rows j <= i (input order) of its key in row i's window;
- windows are aligned to the epoch, with floor division: sliding (a period dividing the window) takes the rows with
  floor(t_j / period) >= floor(t_i / period) - window / period + 1, fixed (no period) the rows with
  floor(t_j / window) == floor(t_i / window);
- count, sum, sqr (sum of squares), max, min, first (the window's earliest row in input order), last (the row itself), avg,
  stdvar (sample variance; NaN for one row) and stddev.

For each row this scans every earlier row of its key and tests it against the window by floor division, then reduces the
selected values in float64: exactly rounded sums (math.fsum) and a two-pass variance.  It shares no algorithm with the kernel
(no sort, no binary search, no range structure).  Rows the device refuses (late events, NaT timestamps, NaN values) are
counted, not aggregated."""

import math

import numpy as np

NAT = -(1 << 63)
OPS = ("count", "sum", "sqr", "max", "min", "first", "last", "avg", "stdvar", "stddev")


def in_window(t_j, t_i, window_ns, period_ns):
    """which rows at t_j (int64 array) are in the window of a row at t_i: floor division (numpy's // floors), and the
    window's first bucket in Python integers, so that nothing overflows near 1677 or 2262"""
    if period_ns:
        return t_j // period_ns >= int(t_i) // period_ns - window_ns // period_ns + 1
    return t_j // window_ns == int(t_i) // window_ns


def reduce(values, op):
    """one operation over the window's values, in input order, in float64"""
    v = [float(x) for x in values]
    n = len(v)
    if op == "count":
        return float(n)
    if op == "sum":
        return math.fsum(v)
    if op == "sqr":
        return math.fsum(x * x for x in v)
    if op == "max":
        return max(v)
    if op == "min":
        return min(v)
    if op == "first":
        return v[0]
    if op == "last":
        return v[-1]
    if op == "avg":
        return math.fsum(v) / n
    if op in ("stdvar", "stddev"):
        if n < 2:
            return math.nan
        mean = math.fsum(v) / n
        var = math.fsum((x - mean) ** 2 for x in v) / (n - 1)
        return var if op == "stdvar" else math.sqrt(var)
    raise ValueError(op)


def refusals(keys, ts, sources):
    """(late rows, NaT rows, NaN values): rows whose timestamp is below their key's previous row, rows at NaT, NaN source
    values (each distinct source counted once)"""
    last, late = {}, 0
    for k, t in zip(np.asarray(keys).tolist(), np.asarray(ts).tolist()):
        if k in last and t < last[k]:
            late += 1
        last[k] = t
    nat_rows = int((np.asarray(ts) == NAT).sum())
    nans = sum(int(np.isnan(np.asarray(a, dtype=np.float64)).sum()) for a in sources.values())
    return late, nat_rows, nans


def aggregate(keys, ts, sources, aggregates, rows=None):
    """keys: int64 [n]; ts: int64 ns [n]; sources: {column: array [n]}; aggregates: [{"name", "column", "operations",
    "windows", "period"}] with windows / period in nanoseconds (period 0 or None: fixed windows); a window may be a
    (label, nanoseconds) pair, named by its label.  -> {"{name}_{op}_{w}":
    float64 [n]} for every row, or for the positions in `rows` only (the other entries are NaN)."""
    ts = np.asarray(ts, dtype=np.int64)
    n = len(ts)
    history = {}  # key -> positions so far, input order
    mine = []     # (key, how many of its positions are row i's or earlier)
    for i, k in enumerate(np.asarray(keys, dtype=np.int64).tolist()):
        history.setdefault(k, []).append(i)
        mine.append((k, len(history[k])))
    history = {k: np.asarray(v, dtype=np.int64) for k, v in history.items()}
    want = range(n) if rows is None else sorted(set(int(r) for r in rows))
    out = {}
    for agg in aggregates:
        x = np.asarray(sources[agg["column"]])
        period = int(agg.get("period") or 0)
        windows = [w if isinstance(w, tuple) else (w, w) for w in agg["windows"]]  # (label, nanoseconds)
        for op in agg["operations"]:
            for label, _w in windows:
                out[f"{agg['name']}_{op}_{label}"] = np.full(n, np.nan)
        for i in want:
            k, upto = mine[i]
            earlier = history[k][:upto]
            for label, w in windows:
                vals = x[earlier[in_window(ts[earlier], ts[i], int(w), period)]]
                for op in agg["operations"]:
                    out[f"{agg['name']}_{op}_{label}"][i] = reduce(vals, op)
    return out
