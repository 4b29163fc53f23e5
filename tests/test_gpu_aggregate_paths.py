"""Every path of b2s_agg (csrc/b2s_agg.cu) on the H100, every output on every row against a vectorised exact reference.

The exact workload: float32 values on the dyadic grid mean + k / 1024 with |k| < 2^14 (int32 sources: |v| < 2^15).  Every
fp64 partial sum of up to 2^22 such rows is exact (multiples of 2^-10 below 2^43; squares multiples of 2^-20 below 2^33 when
the mean is 0), so count / sum / sqr / min / max / first / last equal their references exactly in any combine order, avg is
one correctly rounded division of exact values and equals sum / count bit for bit, and a range decomposition that drops or
repeats one element fails on every row it touches.  The references are integer prefix differences (sum, sqr), a sparse table
(min, max) and the Chan-Golub-LeVeque bound of tests/test_gpu_aggregate.py for stdvar / stddev against an M2 from integer
moments; half the cases offset the data by a mean of 1e6, where sqr is held to 128 eps sum x^2 and a variance taken as
sum x^2 - (sum x)^2 / count fails.

Cases: one key at four sizes whose windows reach every shape of range_reduce's walk at every level (tests/agg_ranges.py,
checked in tests/test_agg_ranges_cpu.py); key runs starting at offsets 0, 1, 31 and 32 of blocks at levels 0-3 under keys at
the int64 extremes and FNV-1a hashes; one column's structure serving aggregations that read subsets of its fields; the
limits and their refusals; windows at the int64 time range's ends (a 1 ns period at 1677); the device entry against the host
entry.  Every call's launches are checked."""

import ctypes as C

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from mlrun_b200.feature_store.keys import _encode_keys  # noqa: E402
from tests.agg_ranges import levels  # noqa: E402
from tests.test_gpu_aggregate import (ALL, DAY, EPS, HOUR, I64_MAX, I64_MIN, INVALID, K, MIN, _c_spec, check,  # noqa: E402
                                      expected_launches, run_host, std_tol, var_tol, workload)

SEC = 10**9
MEAN = 1e6
# one key, ts = i s, period 1 s: row i's range is [max(0, i - W + 1), i].  The first 15 windows sit at the level boundaries;
# the rest reach a full block, and a suffix on a block boundary with a prefix ending on one, at levels 1-3
LEVEL_WINDOWS = [1, 2, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769, 2**20 - 1, 2**20, 2**20 + 1, 1 << 23,
                 1026, 1058, 2050, 32834, 33858, 65602, 1050690, 1083458, 2099266]
LEVEL_SIZES = [(2**20 - 1, 0.0), (2**20 + 1, MEAN), (2**21 + 37, 0.0), (3 * 2**20 + 5, MEAN)]


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def grid(rng, n, mean=0.0, ints=False):
    """the exact workload: int32 |v| < 2^15, or float32 mean + k / 1024 with |k| < 2^14"""
    if ints:
        return rng.integers(-2**15 + 1, 2**15, n).astype(np.int32)
    return (mean + rng.integers(-2**14 + 1, 2**14, n) / 1024).astype(np.float32)


def _table(x, fn):
    """sparse table: t[k][i] = fn over x[i : i + 2^k]"""
    t = [x]
    while 2 << (len(t) - 1) <= len(x):
        h = 1 << (len(t) - 1)
        t.append(fn(t[-1][:-h], t[-1][h:]))
    return t


def _query(t, fn, lo, hi):
    k = np.floor(np.log2(hi - lo + 1)).astype(np.int64)
    out = np.empty(len(lo))
    for j in np.unique(k).tolist():
        m = k == j
        out[m] = fn(t[j][lo[m]], t[j][hi[m] - (1 << j) + 1])
    return out


def check_exact(got, agg, x, mean, ranges, order=None):
    """every output of `agg` on every row.  x: the source in sorted order (float32 on the grid around `mean`, or int32);
    ranges: {window label: (lo, hi)} in sorted positions; order: the input row of each sorted position (None: the same)"""
    scale = 1 if x.dtype == np.int32 else 1024
    xs = x.astype(np.float64)
    u = np.rint((xs - mean) * scale).astype(np.int64)
    assert np.array_equal(mean + u / scale, xs) and np.abs(u).max() < 2**15
    pu, pq = np.r_[0, np.cumsum(u)], np.r_[0, np.cumsum(u * u)]
    ops = agg["operations"]
    mins = _table(xs, np.minimum) if "min" in ops else None
    maxs = _table(xs, np.maximum) if "max" in ops else None
    ld = np.longdouble
    for label, (lo, hi) in ranges.items():
        c = hi - lo + 1
        su, sq = pu[hi + 1] - pu[lo], pq[hi + 1] - pq[lo]
        total = (c * int(mean * scale) + su) / scale  # int64 below 2^53, then a power-of-two division: exact
        # sum x^2 and M2 from the integer moments, in extended precision (only the bounds and the variance use them)
        s_sq = ((c.astype(ld) * ld(mean * scale) ** 2 + 2 * ld(mean * scale) * su + sq) / ld(scale) ** 2).astype(np.float64)
        m2 = ((c.astype(ld) * sq - su.astype(ld) ** 2) / (c.astype(ld) * ld(scale) ** 2)).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            var = np.where(c > 1, m2 / (c - 1), np.nan)
        for op in ops:
            name = f"{agg['name']}_{op}_{label}"
            g = got[name] if order is None else got[name][order]
            if op in ("stdvar", "stddev"):
                assert np.isnan(g[c == 1]).all() and not np.isnan(g[c > 1]).any(), name
                many = c > 1
                g, w, tol = g[many], var[many], var_tol(s_sq[many], m2[many], c[many])
                if op == "stddev":
                    w = np.sqrt(w)
                    tol = std_tol(tol, g, w)
                err = np.abs(g - w)
                assert (err <= tol).all(), (name, float(err.max()), float(tol[np.argmax(err - tol)]))
                continue
            if op == "sqr" and mean:
                err = np.abs(g - s_sq)
                assert (err <= K * EPS * s_sq).all(), (name, float((err / s_sq).max()))
                continue
            want = {"count": lambda: c.astype(np.float64), "sum": lambda: total, "avg": lambda: total / c,
                    "sqr": lambda: sq / float(scale * scale), "first": lambda: xs[lo], "last": lambda: xs[hi],
                    "min": lambda: _query(mins, np.minimum, lo, hi), "max": lambda: _query(maxs, np.maximum, lo, hi)}[op]()
            np.testing.assert_array_equal(g, want, err_msg=name)


# ------------------------------------------------------------------------------------------------------------ levels
@pytest.mark.parametrize("n,mean", LEVEL_SIZES)
def test_levels_every_row_every_window(n, mean):
    """levels 0 .. n_levels, the last block of each partial; the windows reach every shape of the walk at this n"""
    rng = np.random.default_rng(n)
    keys = np.zeros(n, np.int64)
    ts = np.arange(n, dtype=np.int64) * SEC
    x = grid(rng, n, mean)
    wins = [(f"{w}s", w * SEC) for w in LEVEL_WINDOWS]
    aggs = [dict(name="w", column="x", operations=ALL, windows=wins[:16], period=SEC),
            dict(name="v", column="x", operations=ALL, windows=wins[16:], period=SEC)]
    assert levels(n)[0] == (3 if n < 2**20 else 4)
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    i = np.arange(n, dtype=np.int64)
    for a in aggs:
        check_exact(got, a, x, mean, {label: (np.maximum(0, i - w // SEC + 1), i) for label, w in a["windows"]})


# ------------------------------------------------------------------------------------------------------------ key runs
def test_key_runs_out_of_block_alignment_at_the_int64_extremes():
    """runs start at offsets 0, 1, 31 and 32 of blocks at levels 0-3 (the prep kernel's signed binary search for each run's
    start), keys interleaved in input order; each window spans its row's whole run"""
    rng = np.random.default_rng(11)
    n = 2**21 + 100
    starts = sorted({0} | {j * 32**(L + 1) + off for L in range(4) for j in (1, 2) for off in (-1, 0, 1, 31, 32)})
    lengths = np.diff(starts + [n])
    special = [I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX]
    hashed = _encode_keys(pd.DataFrame({"k": [f"card-{i}" for i in range(len(lengths) - len(special))]}), ["k"], "str", "key")
    run_keys = np.sort(np.r_[np.array(special, np.int64), hashed])
    assert len(np.unique(run_keys)) == len(lengths)
    keys = rng.permutation(np.repeat(run_keys, lengths))
    ts = np.arange(n, dtype=np.int64) * SEC  # input order: each key's times increase
    src = {"x": grid(rng, n), "y": grid(rng, n, ints=True)}
    span = 1 << 23
    aggs = [dict(name=f"{c}{kind}", column=c, operations=ALL, windows=[("all", span * SEC)], period=SEC if kind == "s" else None)
            for c in src for kind in "sf"]
    got, counters = run_host(keys, ts, src, aggs)
    assert counters.tolist() == [0, 0, 0]
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    run_start = np.searchsorted(ks, ks, side="left")
    assert np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]]).tolist() == starts
    for a in aggs:
        check_exact(got, a, src[a["column"]][order], 0.0, {"all": (run_start, np.arange(n, dtype=np.int64))}, order)


# ------------------------------------------------------------------------------------------------------------ fields
def test_one_structure_serves_aggregations_reading_subsets_of_its_fields():
    rng = np.random.default_rng(12)
    n = 4000
    keys, ts = workload(rng, n, 7, 3 * DAY)
    src = {"x": rng.normal(size=n).astype(np.float32) * 10 + 3, "y": rng.normal(size=n).astype(np.float32)}
    aggs = [dict(name="mn", column="x", operations=["min"], windows=[("1h", HOUR), ("1d", DAY)], period=10 * MIN),
            dict(name="cf", column="x", operations=["count", "first"], windows=[("6h", 6 * HOUR)], period=None),
            dict(name="sd", column="x", operations=["stddev"], windows=[("2h", 2 * HOUR), ("2d", 2 * DAY)], period=HOUR),
            dict(name="sm", column="x", operations=["sqr", "max"], windows=[("30m", 30 * MIN)], period=5 * MIN),
            dict(name="av", column="x", operations=["avg"], windows=[("1d", DAY)], period=None),
            dict(name="y", column="y", operations=["count", "first", "last"], windows=[("1h", HOUR)], period=MIN)]
    got, counters = run_host(keys, ts, src, aggs)  # asserts 24 + 1 + levels(n) (x only) + 6 launches
    assert expected_launches(n, aggs) == 24 + 1 + levels(n)[0] + len(aggs)
    assert counters.tolist() == [0, 0, 0]
    check(keys, ts, src, aggs, got)


def test_feature_set_two_aggregations_of_one_column():
    rng = np.random.default_rng(13)
    n = 3000
    keys, ts = workload(rng, n, 30, 2 * DAY)
    df = pd.DataFrame({"card": np.array([f"c{k}" for k in keys], dtype=object), "ts": pd.to_datetime(ts),
                       "amount": rng.normal(size=n).astype(np.float32) * 100 + 1000})
    fset = bi.FeatureSet("tx", entities=["card"], timestamp_key="ts")
    fset.add_aggregation("amount", ["min"], ["1h", "1d"], "10m", name="low")
    fset.add_aggregation("amount", ["stddev"], ["6h"], "30m", name="spread")
    out = fset.ingest(df)
    aggs = [dict(name="low", column="amount", operations=["min"], windows=[("1h", HOUR), ("1d", DAY)], period=10 * MIN),
            dict(name="spread", column="amount", operations=["stddev"], windows=[("6h", 6 * HOUR)], period=30 * MIN)]
    names = ["low_min_1h", "low_min_1d", "spread_stddev_6h"]
    assert list(out.columns) == ["ts", "amount"] + names
    assert fset.plan.agg.stats["kernels"] == expected_launches(n, aggs)
    codes = pd.factorize(df["card"])[0].astype(np.int64)
    check(codes, ts, {"amount": df["amount"].to_numpy()}, aggs, {c: out[c].to_numpy() for c in names})


# ------------------------------------------------------------------------------------------------------------ limits
def _run_ranges(keys, ts, period, window):
    """each row's window (lo, hi) in sorted positions (stable by key), the window start from Python integers"""
    order = np.argsort(keys, kind="stable")
    ks, tss = keys[order], ts[order]
    run_start = np.searchsorted(ks, ks, side="left")
    p = period or window
    back = window // period - 1 if period else 0
    start = np.array([max((t // p - back) * p, I64_MIN) for t in tss.tolist()], dtype=np.int64)
    lo = np.empty(len(ks), np.int64)
    firsts = np.unique(run_start)
    for s, e in zip(firsts.tolist(), np.r_[firsts[1:], len(ks)].tolist()):
        lo[s:e] = s + np.searchsorted(tss[s:e], start[s:e], side="left")
    return lo, np.arange(len(ks), dtype=np.int64)


def test_limits_16_sources_64_specs_16_windows_and_all_ops():
    rng = np.random.default_rng(14)
    n = 3000
    keys, ts = workload(rng, n, 20, 2 * DAY)
    src = {f"s{c}": grid(rng, n, ints=c % 2 == 1) for c in range(16)}
    windows = [(f"{m}m", m * MIN) for m in (1, 2, 3, 5, 10, 15, 20, 30, 45, 60, 90, 120, 240, 480, 720, 1440)]
    single = ["count", "sum", "sqr", "max", "min", "first", "last", "avg", "stdvar", "stddev"]
    aggs = [dict(name="every", column="s0", operations=ALL, windows=windows, period=MIN)]
    for s in range(1, 64):
        aggs.append(dict(name=f"a{s}", column=f"s{s % 16}", operations=[single[s % 10]], windows=windows,
                         period=None if s % 3 == 0 else MIN))
    assert sum(len(a["operations"]) for a in aggs) * 16 == 160 + 63 * 16
    got, counters = run_host(keys, ts, src, aggs)
    assert counters.tolist() == [0, 0, 0]
    order = np.argsort(keys, kind="stable")
    ranges = {(p, w): _run_ranges(keys, ts, p, w) for p in (None, MIN) for _l, w in windows}
    for a in aggs:
        check_exact(got, a, src[a["column"]][order], 0.0, {label: ranges[a["period"], w] for label, w in a["windows"]}, order)


def test_over_the_limits_and_one_column_as_two_kinds_refused_with_no_launch():
    lib = nat.init()
    n = 64
    keys, ts, cnt = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(4, np.uint64)
    cols = [np.zeros(n, np.float32) for _ in range(17)]
    outs = [np.zeros(n, np.float64) for _ in range(17)]

    def call(spec_args):
        made = [_c_spec(*a) for a in spec_args]
        specs = (nat.AggSpec * len(made))(*[s for s, _k in made])
        before = nat.launch_count()
        rc = lib.b2s_agg_run_host(keys.ctypes.data, ts.ctypes.data, n, specs, len(made), cnt.ctypes.data, None)
        assert nat.launch_count() == before
        return rc

    def one(c, kind=nat.COL_F32, w=1):
        return cols[c].ctypes.data, kind, nat.AGG_OPS["sum"], MIN, [MIN * (k + 1) for k in range(w)], [o.ctypes.data for o in outs[:w]]

    assert call([one(c) for c in range(17)]) == INVALID                         # 17 distinct sources
    assert call([one(0)] * 65) == INVALID                                       # 65 aggregations
    assert call([one(0, w=17)]) == INVALID                                      # 17 windows
    assert call([one(0), one(0, kind=nat.COL_I32)]) == INVALID                  # one column read as f32 and i32


# ------------------------------------------------------------------------------------------------------------ time edges
def test_one_ns_period_at_the_ends_of_the_int64_range():
    """a 1 ns period and a window of 2^62 or INT64_MAX: the window's first bucket lies below INT64_MIN for rows near 1677"""
    ts = np.array([I64_MIN + 1, I64_MIN + 5, I64_MIN + 10, I64_MAX - 10, I64_MAX - 5, I64_MAX], np.int64)
    keys = np.repeat([0, 1], 3).astype(np.int64)
    x = np.arange(6, dtype=np.float32) + 1
    aggs = [dict(name="p", column="x", operations=ALL, windows=[("w62", 1 << 62), ("max", I64_MAX)], period=1)]
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    assert got["p_count_w62"].tolist() == got["p_count_max"].tolist() == [1, 2, 3, 1, 2, 3]
    check(keys, ts, {"x": x}, aggs, got)


def test_window_of_int64_max_fixed_and_with_a_period_of_7():
    ts = np.array([I64_MIN + 1, I64_MIN + 2, -HOUR, -1, 0, 1, HOUR, I64_MAX - 1, I64_MAX,    # key 0: across the whole range
                   -7, -6, 0, 6, 7], np.int64)                                             # key 1: around 0, period edges
    keys = np.repeat([0, 1], [9, 5]).astype(np.int64)
    x = np.linspace(-2, 2, len(ts)).astype(np.float32)
    assert I64_MAX % 7 == 0
    aggs = [dict(name="f", column="x", operations=ALL, windows=[("max", I64_MAX)], period=None),
            dict(name="s", column="x", operations=ALL, windows=[("max", I64_MAX), ("7", 7), ("14", 14)], period=7)]
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    check(keys, ts, {"x": x}, aggs, got)


def test_sliding_with_period_equal_to_window_is_the_fixed_window():
    rng = np.random.default_rng(15)
    n = 20000
    keys, ts = workload(rng, n, 100, 3 * DAY, t0=-DAY)
    x = rng.normal(size=n).astype(np.float32) * 50 + 7
    wins = [("1h", HOUR), ("1d", DAY), ("7m", 7 * MIN)]
    aggs = [dict(name="f", column="x", operations=ALL, windows=wins, period=None)]
    aggs += [dict(name=f"s{label}", column="x", operations=ALL, windows=[(label, w)], period=w) for label, w in wins]
    got, _c = run_host(keys, ts, {"x": x}, aggs)
    for op in ALL:
        for label, _w in wins:
            np.testing.assert_array_equal(got[f"s{label}_{op}_{label}"], got[f"f_{op}_{label}"], err_msg=f"{op} {label}")


# ------------------------------------------------------------------------------------------------------------ device entry
def test_device_entry_equals_the_host_entry_at_2_20_plus_1_rows():
    import torch

    rng = np.random.default_rng(16)
    n = 2**20 + 1
    keys, ts = workload(rng, n, 50, 2 * DAY)
    x = grid(rng, n, MEAN)
    aggs = [dict(name="s", column="x", operations=ALL, windows=[("1h", HOUR), ("1d", DAY)], period=10 * MIN),
            dict(name="f", column="x", operations=ALL, windows=[("6h", 6 * HOUR)], period=None)]
    host, _c = run_host(keys, ts, {"x": x}, aggs)
    dev = torch.device("cuda", 0)
    d_keys, d_ts, d_x = (torch.from_numpy(a).to(dev) for a in (keys, ts, x))
    d_cnt = torch.zeros(3, dtype=torch.int64, device=dev)
    d_outs, specs, keep = {}, [], []
    for a in aggs:
        ptrs = []
        for op in sorted(a["operations"], key=nat.AGG_OPS.get):
            for label, _w in a["windows"]:
                d_outs[f"{a['name']}_{op}_{label}"] = t = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)
                ptrs.append(t.data_ptr())
        spec, k = _c_spec(d_x.data_ptr(), nat.COL_F32, sum(nat.AGG_OPS[o] for o in a["operations"]), a["period"] or 0,
                          [w for _l, w in a["windows"]], ptrs)
        specs.append(spec)
        keep.append(k)
    c_specs = (nat.AggSpec * len(specs))(*specs)
    strm = torch.cuda.Stream(device=0)
    before = nat.launch_count()
    with torch.cuda.stream(strm):
        nat.check(nat.load().b2s_agg_run_device(d_keys.data_ptr(), d_ts.data_ptr(), n, c_specs, len(specs), d_cnt.data_ptr(),
                                                strm.cuda_stream))
    strm.synchronize()
    assert nat.launch_count() - before == expected_launches(n, aggs)
    assert d_cnt.cpu().tolist() == [0, 0, 0]
    for name, t in d_outs.items():
        np.testing.assert_array_equal(t.cpu().numpy(), host[name], err_msg=name)
