"""b2s_agg (csrc/b2s_agg.cu) against the per-row oracle (oracle/aggregate.py) on the H100.

count / min / max / first / last must equal the oracle exactly (they select or count values, and float32 / int32 widen exactly
to float64).  sum / sqr / avg / stdvar / stddev are fp64 accumulations in a different order from the oracle's exactly rounded
fsum, so they are held to a bound derived from the window's magnitudes: every partial combine rounds once, and a value passes
through at most 2 log2(n) + 64 combines (the hierarchy's levels, the warp scans, the final loop), so

    |sum - ref| <= 128 eps sum|x|,  |sqr - ref| <= 128 eps sum x^2,  |avg - ref| <= 128 eps sum|x| / count,
    |stdvar - ref| <= tol = 128 eps sqrt(sum x^2 M2) / (count - 1),  |stddev - ref| <= tol / (stddev + ref) + 2 eps ref

with eps = 2^-53, the sums over the window's rows alone and M2 the oracle's two-pass sum of squared deviations.  The variance
bound follows Chan, Golub and LeVeque: a pairwise (count, mean, M2) combine errs by O(combines kappa eps M2), with
kappa M2 = sqrt(sum x^2 M2); sum x^2 - (sum x)^2 / count errs by O(eps sum x^2) and fails it once the mean is large against
the spread (tests/test_agg_ranges_cpu.py).  A window of equal values must give exactly 0.  A prefix-difference
implementation fails the cancellation case: its running sums carry +-1e30 from rows outside the window.  Every case also
checks the launches the call made."""

import ctypes as C
import math

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from oracle import aggregate as oa  # noqa: E402

EPS = 2.0**-53
K = 128
HOUR, MIN, DAY = 3600 * 10**9, 60 * 10**9, 86400 * 10**9
INVALID = -1
ALL = list(oa.OPS)
EXACT = ("count", "max", "min", "first", "last")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def levels(n):
    L, m = 0, n
    while m > 32:
        m, L = (m + 31) // 32, L + 1
    return L


def expected_launches(n, aggs):
    """the sort's 24, the prep kernel, one per level of each column that needs a reduce, one per aggregation"""
    if n == 0:
        return 0
    reduce_ops = {"sum", "sqr", "max", "min", "avg", "stdvar", "stddev"}
    cols = {a["column"] for a in aggs if reduce_ops & set(a["operations"])}
    return 24 + 1 + levels(n) * len(cols) + len(aggs)


def _specs(sources, aggs, n):
    specs, outs = [], {}
    for a in aggs:
        by_bit = sorted(a["operations"], key=nat.AGG_OPS.get)
        arrays = []
        for op in by_bit:
            for label, _w in a["windows"]:
                outs[f"{a['name']}_{op}_{label}"] = arr = np.full(n, np.nan)
                arrays.append(arr)
        src = np.ascontiguousarray(sources[a["column"]])
        specs.append((src, nat.COL_I32 if src.dtype == np.int32 else nat.COL_F32, sum(nat.AGG_OPS[o] for o in a["operations"]),
                      a.get("period") or 0, [w for _l, w in a["windows"]], arrays))
    return specs, outs


def run_host(keys, ts, sources, aggs):
    n = len(keys)
    specs, outs = _specs(sources, aggs, n)
    before = nat.launch_count()
    counters, stats = bi.aggregate_host(keys, ts, specs, n)
    made = nat.launch_count() - before
    assert made == stats["kernels"] == expected_launches(n, aggs), (made, stats["kernels"], expected_launches(n, aggs))
    return outs, counters


def var_tol(s_sq, m2, cnt):
    """the stdvar bound: K eps sqrt(sum x^2 M2) / (count - 1), zero for a window of equal values"""
    return K * EPS * np.sqrt(s_sq * m2) / (cnt - 1)


def std_tol(tol_var, got, ref):
    """the stddev bound from the stdvar bound: |sqrt(u) - sqrt(v)| = |u - v| / (sqrt(u) + sqrt(v)), plus a rounding of each
    square root"""
    den = got + ref
    return np.divide(tol_var, den, out=np.zeros_like(den), where=den > 0) + 2 * EPS * ref


def check(keys, ts, sources, aggs, got, rows=None):
    """got vs the oracle on `rows` (all by default): exact ops exactly, the others within the stated bound"""
    want = oa.aggregate(keys, ts, sources, aggs, rows=rows)
    mags = oa.aggregate(keys, ts, {c: np.abs(np.asarray(v, np.float64)) for c, v in sources.items()},
                        [dict(a, operations=["sum", "sqr", "count"]) for a in aggs], rows=rows)
    sel = np.arange(len(keys)) if rows is None else np.asarray(sorted(set(rows)), dtype=np.int64)
    for a in aggs:
        for op in a["operations"]:
            for label, _w in a["windows"]:
                name = f"{a['name']}_{op}_{label}"
                g, w = got[name][sel], want[name][sel]
                if op in EXACT:
                    np.testing.assert_array_equal(g, w, err_msg=name)
                    continue
                s_abs = mags[f"{a['name']}_sum_{label}"][sel]
                s_sq = mags[f"{a['name']}_sqr_{label}"][sel]
                cnt = mags[f"{a['name']}_count_{label}"][sel]
                tol = {"sum": K * EPS * s_abs, "sqr": K * EPS * s_sq, "avg": K * EPS * s_abs / cnt}.get(op)
                if op in ("stdvar", "stddev"):
                    assert np.array_equal(np.isnan(g), np.isnan(w)) and np.isnan(w[cnt == 1]).all(), name
                    ok = ~np.isnan(w)
                    g, w, s_sq, cnt = g[ok], w[ok], s_sq[ok], cnt[ok]
                    m2 = (w if op == "stdvar" else w * w) * (cnt - 1)  # the oracle's two-pass M2
                    tol = var_tol(s_sq, m2, cnt)
                    if op == "stddev":
                        tol = std_tol(tol, g, w)
                err = np.abs(g - w)
                assert (err <= tol).all(), (name, float(err.max()), float(tol[np.argmax(err - tol)]))


def workload(rng, n, n_keys, span_ns, t0=1_700_000_000 * 10**9):
    keys = rng.integers(0, n_keys, n).astype(np.int64)
    draws = rng.integers(0, span_ns, n)
    draws[rng.random(n) < 0.1] = 0
    ts = np.empty(n, np.int64)
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    ends = np.r_[starts[1:], n]
    d = draws[order]
    for s, e in zip(starts, ends):  # per-key non-decreasing
        d[s:e] = np.sort(d[s:e])
    ts[order] = t0 + d
    return keys, ts


def aggs_all(windows_sliding, period, windows_fixed, col="x", name="a"):
    out = [dict(name=name + "s", column=col, operations=ALL, windows=windows_sliding, period=period)]
    if windows_fixed:
        out.append(dict(name=name + "f", column=col, operations=ALL, windows=windows_fixed, period=None))
    return out


# ------------------------------------------------------------------------------------------------------------ semantics
def test_every_op_sliding_and_fixed_several_periods_and_columns():
    rng = np.random.default_rng(1)
    n = 3000
    keys, ts = workload(rng, n, 50, 2 * DAY)
    x = rng.normal(size=n).astype(np.float32) * 100
    y = rng.integers(-2**31, 2**31, n).astype(np.int32)
    y[:4] = [-2**31, 2**31 - 1, -2**31, 2**31 - 1]
    aggs = (aggs_all([("1h", HOUR), ("6h", 6 * HOUR)], 10 * MIN, [("1h", HOUR)], "x", "x")
            + aggs_all([("30m", 30 * MIN), ("1d", DAY)], 30 * MIN, [("1d", DAY)], "y", "y"))
    got, counters = run_host(keys, ts, {"x": x, "y": y}, aggs)
    assert counters.tolist() == [0, 0, 0]
    check(keys, ts, {"x": x, "y": y}, aggs, got)


def test_bucket_edges_negative_and_extreme_timestamps_equal_timestamps():
    e = 7 * HOUR
    ts = np.array([e - HOUR - 1, e - HOUR, e - HOUR + 1, e - 1, e, e, e + 1,             # key 0: around a 1 h edge, ties
                   -2 * HOUR - 1, -2 * HOUR, -HOUR - 1, -HOUR, -1, 0, 1,                # key 1: before 1970
                   I64_MIN + 1, I64_MIN + 2, I64_MIN + HOUR,                             # key 2: 1677
                   I64_MAX - HOUR, I64_MAX - 1, I64_MAX], np.int64)                      # key 3: 2262
    keys = np.repeat([0, 1, 2, 3], [7, 7, 3, 3]).astype(np.int64)
    x = np.linspace(-3, 3, len(ts)).astype(np.float32)
    aggs = aggs_all([("1h", HOUR), ("2h", 2 * HOUR), ("1d", DAY)], HOUR, [("1h", HOUR), ("1d", DAY)])
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    check(keys, ts, {"x": x}, aggs, got)
    assert got["af_count_1h"][:7].tolist() == [1, 1, 2, 3, 1, 2, 3]


def test_windows_longer_than_the_history_and_all_distinct_keys():
    rng = np.random.default_rng(3)
    n = 200_000
    keys = rng.permutation(n).astype(np.int64) * 7919
    ts = rng.integers(0, DAY, n).astype(np.int64)
    x = rng.normal(size=n).astype(np.float32)
    aggs = aggs_all([("7d", 7 * DAY)], DAY, [("30d", 30 * DAY)])
    got, _c = run_host(keys, ts, {"x": x}, aggs)
    xx = x.astype(np.float64)
    for p in ("as", "af"):
        w = "7d" if p == "as" else "30d"
        assert (got[f"{p}_count_{w}"] == 1).all() and np.isnan(got[f"{p}_stdvar_{w}"]).all()
        for op in ("sum", "max", "min", "first", "last", "avg"):
            np.testing.assert_array_equal(got[f"{p}_{op}_{w}"], xx, err_msg=op)
        np.testing.assert_array_equal(got[f"{p}_sqr_{w}"], xx * xx)
    few_keys, few_ts = workload(rng, 3000, 5, 3 * HOUR)
    xs = rng.normal(size=3000).astype(np.float32)
    got, _c = run_host(few_keys, few_ts, {"x": xs}, aggs)
    check(few_keys, few_ts, {"x": xs}, aggs, got)


def test_one_key_of_2_20_rows():
    rng = np.random.default_rng(4)
    n = 1 << 20
    keys = np.zeros(n, np.int64)
    ts = np.arange(n, dtype=np.int64) * 10**9  # one row a second: 12 days
    x = rng.normal(size=n).astype(np.float32) + 5
    aggs = [dict(name="s", column="x", operations=ALL, windows=[("1h", HOUR), ("1d", DAY), ("7d", 7 * DAY)], period=10 * MIN),
            dict(name="f", column="x", operations=ALL, windows=[("1d", DAY)], period=None)]
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    rows = np.r_[0, 1, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769, rng.integers(0, n, 40), n - 1]
    check(keys, ts, {"x": x}, aggs, got, rows=rows)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1023, 1024, 1025, 32767, 32768, 32769])
def test_sizes_at_the_levels_of_the_range_structure(n):
    rng = np.random.default_rng(n)
    keys = (np.arange(n) >= n - 3).astype(np.int64)  # one long key (every row in the window) and a short one
    ts = np.arange(n, dtype=np.int64) * MIN
    x = rng.normal(size=n).astype(np.float32)
    aggs = aggs_all([("30d", 30 * DAY)], DAY, [("1h", HOUR)])
    got, counters = run_host(keys, ts, {"x": x}, aggs)
    assert counters.tolist() == [0, 0, 0]
    rows = None if n <= 1025 else np.r_[np.arange(0, n, 997), n - 4, n - 3, n - 1]
    check(keys, ts, {"x": x}, aggs, got, rows=rows)


def test_cancellation_history_outside_the_window_does_not_reach_the_sum():
    n_old, n_new = 5000, 300
    old = np.where(np.arange(n_old) % 2 == 0, 1e30, -1e30).astype(np.float32)
    new = (1 + np.random.default_rng(5).random(n_new) * 1e-3).astype(np.float32)
    x = np.r_[old, new]
    keys = np.zeros(n_old + n_new, np.int64)
    ts = np.r_[np.arange(n_old) * 10**9, 10 * DAY + np.arange(n_new) * 10**9].astype(np.int64)
    aggs = [dict(name="c", column="x", operations=ALL, windows=[("1h", HOUR)], period=10 * MIN)]
    got, _c = run_host(keys, ts, {"x": x}, aggs)
    rows = np.arange(n_old, n_old + n_new)
    check(keys, ts, {"x": x}, aggs, got, rows=rows)
    np.testing.assert_allclose(got["c_sum_1h"][-1], float(np.sum(new.astype(np.float64))), rtol=1e-14)


def test_device_counters_late_nat_and_nan():
    keys = np.array([1, 2, 1, 1, 2, 3, 3], np.int64)
    ts = np.array([10, 5, 20, 15, I64_MIN, 7, 8], np.int64) * 1  # key 1: 20 then 15 (late); key 2: NaT after 5
    x = np.array([1, np.nan, 2, 3, 4, np.nan, np.nan], np.float32)
    y = np.arange(7, dtype=np.int32)
    aggs = [dict(name="a", column="x", operations=["sum"], windows=[("1h", HOUR)], period=None),
            dict(name="b", column="x", operations=["count"], windows=[("1h", HOUR)], period=None),
            dict(name="c", column="y", operations=["max"], windows=[("1h", HOUR)], period=None)]
    _got, counters = run_host(keys, ts, {"x": x, "y": y}, aggs)
    want = oa.refusals(keys, ts, {"x": x, "y": y})
    assert tuple(counters.tolist()) == want == (2, 1, 3)  # the NaT row is also below its key's previous row


# ------------------------------------------------------------------------------------------------------------ C-ABI
def _c_spec(src, kind, ops, period, windows, outs):
    win = np.asarray(windows, np.int64)
    ptrs = (C.c_void_p * max(len(outs), 1))(*outs)
    return nat.AggSpec(src, kind, ops, period, len(win), win.ctypes.data_as(C.POINTER(C.c_int64)), ptrs), (win, ptrs)


def test_invalid_arguments_launch_nothing():
    lib = nat.init()
    n = 64
    keys = np.zeros(n + 1, np.int64)
    ts = np.zeros(n + 1, np.int64)
    x = np.zeros(n + 1, np.float32)
    out = np.zeros(n + 1, np.float64)
    cnt = np.zeros(4, np.uint64)
    k8, t8, x4, o8, c8 = (a.ctypes.data for a in (keys, ts, x, out, cnt))

    def call(spec_args, n=n, keys=k8, ts=t8, counters=c8):
        spec, keep = _c_spec(*spec_args)
        specs = (nat.AggSpec * 1)(spec)
        before = nat.launch_count()
        rc = lib.b2s_agg_run_host(keys, ts, n, specs, 1, counters, None)
        if rc == INVALID:
            assert nat.launch_count() == before, "an invalid call launched"
        return rc

    good = (x4, nat.COL_F32, nat.AGG_OPS["sum"], 10 * MIN, [HOUR], [o8])
    assert call(good) == 0 and out[:n].tolist() == x[:n].tolist()
    assert call(good, keys=None) == INVALID
    assert call(good, ts=None) == INVALID
    assert call(good, counters=None) == INVALID
    assert call(good, keys=k8 + 4) == INVALID
    assert call(good, ts=t8 + 4) == INVALID
    assert call(good, counters=c8 + 4) == INVALID
    assert call(good, n=1 << 32) == INVALID
    assert call(good, n=-1) == INVALID
    assert call((x4 + 2, nat.COL_F32, 2, 10 * MIN, [HOUR], [o8])) == INVALID       # source not 4-byte aligned
    assert call((None, nat.COL_F32, 2, 10 * MIN, [HOUR], [o8])) == INVALID
    assert call((x4, nat.COL_F32, 2, 10 * MIN, [HOUR], [o8 + 4])) == INVALID       # output not 8-byte aligned
    assert call((x4, nat.COL_F32, 2, 10 * MIN, [HOUR], [None])) == INVALID
    assert call((x4, nat.COL_F32, 2, 7 * MIN, [HOUR], [o8])) == INVALID            # period does not divide the window
    assert call((x4, nat.COL_F32, 2, 10 * MIN, [0], [o8])) == INVALID
    assert call((x4, nat.COL_F32, 0, 10 * MIN, [HOUR], [o8])) == INVALID           # empty op mask
    assert call((x4, nat.COL_F32, 1 << 10, 10 * MIN, [HOUR], [o8])) == INVALID     # unknown op bit
    assert call((x4, nat.COL_I64, 2, 10 * MIN, [HOUR], [o8])) == INVALID           # not a 4-byte kind


def test_device_entry_on_a_callers_stream_equals_the_host_entry():
    import torch

    rng = np.random.default_rng(6)
    n = 50_000
    keys, ts = workload(rng, n, 300, DAY)
    x = rng.normal(size=n).astype(np.float32)
    aggs = aggs_all([("1h", HOUR), ("6h", 6 * HOUR)], 10 * MIN, [("1h", HOUR)])
    host, _c = run_host(keys, ts, {"x": x}, aggs)
    dev = torch.device("cuda", 0)
    d_keys, d_ts, d_x = torch.from_numpy(keys).to(dev), torch.from_numpy(ts).to(dev), torch.from_numpy(x).to(dev)
    d_cnt = torch.zeros(3, dtype=torch.int64, device=dev)
    names, specs, keep = [], [], []
    d_outs = {}
    for a in aggs:
        by_bit = sorted(a["operations"], key=nat.AGG_OPS.get)
        ptrs = []
        for op in by_bit:
            for label, _w in a["windows"]:
                name = f"{a['name']}_{op}_{label}"
                d_outs[name] = t = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)
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


# ------------------------------------------------------------------------------------------------------- FeatureSet
def _ingest_case(rng, n):
    keys, ts = workload(rng, n, 40, 2 * DAY)
    df = pd.DataFrame({"card": np.array([f"c{k}" for k in keys], dtype=object), "ts": pd.to_datetime(ts),
                       "amount": (rng.random(n) * 500).astype(np.float32), "n": rng.integers(0, 9, n).astype(np.int32)})
    fset = bi.FeatureSet("tx", entities=["card"], timestamp_key="ts")
    fset.add_aggregation("amount", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "6h"], "10m")
    fset.add_aggregation("n", ["sum", "first", "last"], "1h", name="items")
    return df, fset


def _ingest_expected(df):
    codes = pd.factorize(df["card"])[0].astype(np.int64)
    ts = df["ts"].to_numpy().view(np.int64)
    src = {"amount": df["amount"].to_numpy(), "n": df["n"].to_numpy()}
    aggs = [dict(name="amount", column="amount", operations=["count", "sum", "avg", "min", "max", "stddev"],
                 windows=[("1h", HOUR), ("6h", 6 * HOUR)], period=10 * MIN),
            dict(name="items", column="n", operations=["sum", "first", "last"], windows=[("1h", HOUR)], period=None)]
    return codes, ts, src, aggs


def test_feature_set_ingest_from_a_frame_and_from_columns():
    rng = np.random.default_rng(7)
    df, fset = _ingest_case(rng, 4000)
    out = fset.ingest(df)
    codes, ts, src, aggs = _ingest_expected(df)
    names = [f"amount_{op}_{w}" for op in ["count", "sum", "avg", "min", "max", "stddev"] for w in ["1h", "6h"]]
    names += ["items_sum_1h", "items_first_1h", "items_last_1h"]
    assert list(out.columns) == ["ts", "amount", "n"] + names and list(out.index.names) == ["card"]
    assert (out[names].dtypes == np.float64).all()
    check(codes, ts, src, aggs, {c: out[c].to_numpy() for c in names})
    assert fset.plan.agg.stats["kernels"] == expected_launches(len(df), aggs)
    batch = fset.ingest({c: df[c].to_numpy() for c in df.columns})
    for c in names:
        np.testing.assert_array_equal(np.asarray(batch[c]), out[c].to_numpy(), err_msg=c)
    late = df.copy()
    late.loc[late.index[-1], "ts"] = late["ts"].min() - pd.Timedelta(days=1)
    with pytest.raises(bi.LoweringError, match="below the previous row"):
        fset.ingest(late)


def test_reference_literal_on_the_device():
    base = pd.Timestamp(2020, 12, 1, 17, 33, 15)
    data = pd.DataFrame({"time": [base, base - pd.Timedelta(minutes=1)], "first_name": np.array(["moshe", "yosi"], dtype=object),
                         "bid": np.array([2000, 10], np.int32)})
    data["time"] = data["time"].astype("datetime64[ns]")
    fset = bi.FeatureSet("measurements", entities=["first_name"], timestamp_key="time")
    fset.add_aggregation(name="bids", column="bid", operations=["sum", "max"], windows="1h", period="10m")
    out = fset.ingest(data, return_df=True)
    assert out.loc["moshe", "bids_sum_1h"] == 2000.0 and out.loc["moshe", "bids_max_1h"] == 2000.0
    assert not math.isnan(out.loc["yosi", "bids_sum_1h"])
