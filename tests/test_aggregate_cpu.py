"""FeatureSet.add_aggregation and the windowed aggregations of ingest on CPU: the oracle (oracle/aggregate.py) against a second,
independent restatement (tests/emulated_agg.py: stable sort by key, window starts by searchsorted); the host layer over that
emulation against the oracle -- names, column order, dtypes, index, int / pair / string keys, DataFrame and columnar sources;
every refusal, before any copy where the semantics allow it; add_aggregation and its merging against what the real reference
did (tests/golden/ref_add_aggregation.json); and the reference's own literal (a single event gives bids_sum_1h == 2000.0)."""

import json
import os

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import ingest as bi
from mlrun_b200.lowering import LoweringError
from mlrun_b200.serving.resolve import MLRunInvalidArgumentError
from oracle import aggregate as oa
from tests import device_emulator, emulated_agg

HOUR = 3600 * 10**9
MIN = 60 * 10**9
ALL_OPS = list(oa.OPS)


@pytest.fixture
def emulated(monkeypatch):
    device_emulator.install_columns(monkeypatch)
    emulated_agg.install(monkeypatch)


def _workload(rng, n, n_keys, span_ns, t0=1_700_000_000 * 10**9, ints=False):
    keys = rng.integers(0, n_keys, n).astype(np.int64)
    draws = rng.integers(0, span_ns, n)
    draws[rng.random(n) < 0.1] = 0  # some equal timestamps
    ts = np.empty(n, np.int64)
    for k in np.unique(keys):  # per-key non-decreasing times, keys interleaved in input order
        at = np.flatnonzero(keys == k)
        ts[at] = t0 + np.sort(draws[at])
    x = rng.integers(-2**31, 2**31, n).astype(np.int32) if ints else rng.normal(size=n).astype(np.float32)
    return keys, ts, x


def _emulate(keys, ts, sources, aggregates):
    specs, out = [], {}
    for agg in aggregates:
        ops = sum(nat.AGG_OPS[o] for o in agg["operations"])
        by_bit = sorted(agg["operations"], key=nat.AGG_OPS.get)
        arrays = []
        for op in by_bit:
            for label, _w in agg["windows"]:
                out[f"{agg['name']}_{op}_{label}"] = a = np.empty(len(keys))
                arrays.append(a)
        src = sources[agg["column"]]
        specs.append((src, nat.COL_I32 if src.dtype == np.int32 else nat.COL_F32, ops, agg["period"] or 0,
                      [w for _l, w in agg["windows"]], arrays))
    counters, _ = emulated_agg.aggregate_host(keys, ts, specs, len(keys))
    return out, counters


@pytest.mark.parametrize("seed", range(4))
def test_oracle_equals_a_second_restatement(seed):
    rng = np.random.default_rng(seed)
    keys, ts, x = _workload(rng, 400, [1, 3, 40, 400][seed], 6 * HOUR)
    _k, _t, y = _workload(rng, 400, 1, 1, ints=True)
    aggs = [dict(name="a", column="x", operations=ALL_OPS, windows=[("1h", HOUR), ("2h", 2 * HOUR)], period=10 * MIN),
            dict(name="b", column="y", operations=ALL_OPS, windows=[("30m", 30 * MIN)], period=None),
            dict(name="c", column="x", operations=["sum", "count"], windows=[("7d", 7 * 24 * HOUR)], period=HOUR)]
    want = oa.aggregate(keys, ts, {"x": x, "y": y}, aggs)
    got, counters = _emulate(keys, ts, {"x": x, "y": y}, aggs)
    assert counters.tolist() == [0, 0, 0] and oa.refusals(keys, ts, {"x": x}) == (0, 0, 0)
    assert set(got) == set(want)
    for name in want:
        exact = any(f"_{op}_" in name for op in ("count", "max", "min", "first", "last"))
        if exact:
            np.testing.assert_array_equal(got[name], want[name], err_msg=name)
        else:
            np.testing.assert_allclose(got[name], want[name], rtol=1e-9, atol=1e-6, err_msg=name)


def test_oracle_windows_at_bucket_edges_and_extreme_times():
    """rows exactly on, 1 ns before and 1 ns after a bucket edge; negative times (floor division); 1677 and 2262"""
    edge = 5 * HOUR
    ts = np.array([edge - HOUR - 1, edge - HOUR, edge - 1, edge, edge + 1], np.int64)
    x = np.arange(1, 6, dtype=np.float32)
    agg = [dict(name="s", column="x", operations=["count"], windows=[("1h", HOUR)], period=None)]
    assert oa.aggregate(np.zeros(5), ts, {"x": x}, agg)["s_count_1h"].tolist() == [1, 1, 2, 1, 2]
    neg = np.array([-HOUR - 1, -HOUR, -1, 0], np.int64)
    assert oa.aggregate(np.zeros(4), neg, {"x": x[:4]}, agg)["s_count_1h"].tolist() == [1, 1, 2, 1]
    lo, hi = np.iinfo(np.int64).min + 1, np.iinfo(np.int64).max
    far = np.array([lo, lo + 1, hi - 1, hi], np.int64)
    slide = [dict(name="s", column="x", operations=["count"], windows=[("1d", 24 * HOUR)], period=HOUR)]
    got = oa.aggregate(np.array([0, 0, 1, 1]), far, {"x": x[:4]}, slide)["s_count_1d"]
    assert got.tolist() == [1, 2, 1, 2]
    em, _ = _emulate(np.array([0, 0, 1, 1]), far, {"x": x[:4]}, slide)
    assert em["s_count_1d"].tolist() == [1, 2, 1, 2]


def _frame(rng, n, key_kind):
    keys, ts, x = _workload(rng, n, 7, 3 * HOUR)
    df = pd.DataFrame({"ts": pd.to_datetime(ts), "bid": x, "qty": rng.integers(-50, 50, n).astype(np.int32)})
    if key_kind == "int":
        df.insert(0, "k", keys)
        cols = ["k"]
    elif key_kind == "pair":
        df.insert(0, "k1", (keys % 3).astype(np.int32))
        df.insert(1, "k2", (keys // 3).astype(np.int32))
        cols = ["k1", "k2"]
    else:
        df.insert(0, "k", np.array([f"card-{k}" for k in keys], dtype=object))
        cols = ["k"]
    return df, cols, keys


def _fset(cols):
    fset = bi.FeatureSet("quotes", entities=cols, timestamp_key="ts")
    fset.add_aggregation("bid", ["sum", "max", "stddev"], ["1h", "2h"], "10m", name="bids")
    fset.add_aggregation("qty", ["count", "first", "last", "avg"], "30m")
    return fset


def _expected(df, keys):
    ts = df["ts"].to_numpy().view(np.int64)
    src = {"bid": df["bid"].to_numpy(), "qty": df["qty"].to_numpy()}
    a = oa.aggregate(keys, ts, src, [dict(name="bids", column="bid", operations=["sum", "max", "stddev"],
                                           windows=[("1h", HOUR), ("2h", 2 * HOUR)], period=10 * MIN)])
    a.update(oa.aggregate(keys, ts, src, [dict(name="qty", column="qty", operations=["count", "first", "last", "avg"],
                                                windows=[("30m", 30 * MIN)], period=None)]))
    return a


AGG_COLUMNS = ["bids_sum_1h", "bids_sum_2h", "bids_max_1h", "bids_max_2h", "bids_stddev_1h", "bids_stddev_2h",
               "qty_count_30m", "qty_first_30m", "qty_last_30m", "qty_avg_30m"]


@pytest.mark.parametrize("key_kind", ["int", "pair", "str"])
def test_ingest_frame_over_the_emulation_equals_the_oracle(emulated, key_kind):
    rng = np.random.default_rng(7)
    df, cols, keys = _frame(rng, 300, key_kind)
    out = _fset(cols).ingest(df)
    assert list(out.columns) == ["ts", "bid", "qty"] + AGG_COLUMNS  # after the graph's columns, operation-major
    assert list(out.index.names) == cols and out.index.equals(df.set_index(cols).index)
    want = _expected(df, keys)
    for name in AGG_COLUMNS:
        assert out[name].dtype == np.float64
        np.testing.assert_allclose(out[name].to_numpy(), want[name], rtol=1e-12, atol=1e-12, err_msg=name)
    np.testing.assert_array_equal(out["bid"].to_numpy(), df["bid"].to_numpy())


def test_ingest_columnar_source_equals_the_frame(emulated):
    rng = np.random.default_rng(8)
    df, cols, keys = _frame(rng, 200, "int")
    fset = _fset(cols)
    batch = fset.ingest({c: df[c].to_numpy() for c in df.columns})
    frame = fset.ingest(df)  # one feature set, both sources: each lowers its own plan
    assert list(fset.ingest({c: df[c].to_numpy() for c in df.columns}).columns) == list(batch.columns)
    assert list(batch.columns) == list(frame.columns)
    for name in frame.columns:
        np.testing.assert_array_equal(np.asarray(batch[name]), frame[name].to_numpy())
    np.testing.assert_array_equal(batch.index["k"], keys)


def test_aggregation_after_other_steps_reads_their_results(emulated):
    """the aggregation sees the graph's result columns: an Imputer fill is aggregated, not the NaN"""
    from mlrun_b200.feature_store import steps as bs

    df = pd.DataFrame({"k": np.array([1, 1, 2], np.int64), "ts": pd.to_datetime([0, 1, 2]),
                       "bid": np.array([1.0, np.nan, 4.0], np.float32)})
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.graph.to(bs.Imputer(mapping={"bid": 2.0}))
    fset.add_aggregation("bid", ["sum"], "1h")
    out = fset.ingest(df)
    assert out["bid_sum_1h"].tolist() == [1.0, 3.0, 4.0]


def test_reference_literal_single_event(emulated):
    """tests/system/feature_store/test_feature_store.py:1506-1539 (test_unaggregated_columns): bids sum over 1 h sliding every
    10 min; moshe's single event gives bids_sum_1h == 2000.0.  The reference's set has no timestamp key (storey then uses
    processing time); here the event time is given, which a single event's window cannot tell apart."""
    base = pd.Timestamp(2020, 12, 1, 17, 33, 15)
    data = pd.DataFrame({"time": [base, base - pd.Timedelta(minutes=1)], "first_name": np.array(["moshe", "yosi"], dtype=object),
                         "bid": np.array([2000, 10], np.int32)})
    data["time"] = data["time"].astype("datetime64[ns]")
    fset = bi.FeatureSet("measurements", entities=["first_name"], timestamp_key="time")
    fset.add_aggregation(name="bids", column="bid", operations=["sum", "max"], windows="1h", period="10m")
    out = fset.ingest(data, return_df=True)
    assert out.loc["moshe", "bids_sum_1h"] == 2000.0 and out.loc["yosi", "bids_sum_1h"] == 10.0
    assert out.loc["moshe", "bids_max_1h"] == 2000.0


# ---------------------------------------------------------------------------------------------------------------- refusals
@pytest.fixture
def no_copy(emulated, monkeypatch):
    """fails the test if the columns plan or the aggregation runs"""
    def boom(*a, **k):
        raise AssertionError("data was copied before the refusal")

    monkeypatch.setattr(device_emulator.EmulatedColumns, "run_host", boom)
    monkeypatch.setattr(bi, "aggregate_host", boom)


def _base():
    return pd.DataFrame({"k": np.array([1, 2, 1], np.int64), "ts": pd.to_datetime([0, 1, 2]),
                         "bid": np.array([1, 2, 3], np.float32), "n": np.array([1, 2, 3], np.int32),
                         "d": pd.to_datetime([5, 6, 7])})


@pytest.mark.parametrize("case,match", [
    (lambda: bi.FeatureSet("s", entities=["k"]), "timestamp_key"),
    (lambda: bi.FeatureSet("s", timestamp_key="ts"), "entities"),
    (lambda: bi.FeatureSet("s", entities=["k", "n"], timestamp_key="ts"), "not lowered"),   # int64 + int32 keys
    (lambda: bi.FeatureSet("s", entities=["k"], timestamp_key="ts"), None),
])
def test_feature_set_level_refusals_come_before_any_copy(no_copy, case, match):
    fset = case()
    fset.add_aggregation("bid", ["sum"], "1h")
    frame = _base() if fset.entities else _base().drop(columns="k")  # an int64 column is only taken as a key
    if match is None:  # the control: the same set refuses only when the run starts
        with pytest.raises(AssertionError, match="copied"):
            fset.ingest(frame)
        return
    with pytest.raises(LoweringError, match=match):
        fset.ingest(frame)


@pytest.mark.parametrize("column,ops,windows,period,match", [
    ("k", ["sum"], "1h", None, "entities and the timestamp"),
    ("ts", ["sum"], "1h", None, "entities and the timestamp"),
    ("d", ["sum"], "1h", None, "float32 or int32 result column"),
    ("nope", ["sum"], "1h", None, "float32 or int32 result column"),
    ("bid", ["median"], "1h", None, "operations"),
    ("bid", ["sum"], "1w", None, "unit s, m, h or d"),
    ("bid", ["sum"], "90m", "1h", "must divide every window"),
    ("bid", ["sum"], "1h", "7s", "must divide every window"),
])
def test_aggregation_refusals_come_before_any_copy(no_copy, column, ops, windows, period, match):
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.add_aggregation(column, ops, windows, period)
    with pytest.raises(LoweringError, match=match):
        fset.ingest(_base())


def test_emit_policy_and_graph_shape_refusals(no_copy):
    class EmitAfterMaxEvent:
        pass

    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.add_aggregation("bid", ["sum"], "1h", emit_policy=EmitAfterMaxEvent())
    with pytest.raises(LoweringError, match="emit policy"):
        fset.ingest(_base())

    class EmitEveryEvent:
        pass

    ok = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    ok.add_aggregation("bid", ["sum"], "1h", emit_policy=EmitEveryEvent())
    with pytest.raises(AssertionError, match="copied"):
        ok.ingest(_base())

    two = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    two.add_aggregation("bid", ["sum"], "1h", step_name="A1")
    two.add_aggregation("n", ["sum"], "1h", step_name="A2")
    with pytest.raises(LoweringError, match="second aggregation step"):
        two.ingest(_base())

    from mlrun_b200.feature_store import steps as bs

    after = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    after.add_aggregation("bid", ["sum"], "1h")
    after.add_step(bs.Imputer(mapping={"bid": 0.0}), name="late")
    with pytest.raises(LoweringError, match="after the aggregation step"):
        after.ingest(_base())


@pytest.mark.parametrize("mutate,match", [
    (lambda df: df.assign(ts=pd.to_datetime([5, 6, 4])), "1 rows have a timestamp below"),
    (lambda df: df.assign(ts=pd.to_datetime([0, None, 2])), "NaT"),
    (lambda df: df.assign(bid=np.array([1, np.nan, np.nan], np.float32)), "2 aggregated values are NaN"),
])
def test_device_counted_refusals_raise_after_the_run(emulated, mutate, match):
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.add_aggregation("bid", ["sum"], "1h")
    with pytest.raises(LoweringError, match=match):
        fset.ingest(mutate(_base()))


def test_plan_cache_key_includes_the_aggregations(emulated):
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.add_aggregation("bid", ["sum"], "1h", "10m")
    first = fset.ingest(_base())
    fset.add_aggregation("bid", ["max"], "1h", "10m")  # merged into the same aggregation: a new plan
    second = fset.ingest(_base())
    assert list(first.columns)[-1:] == ["bid_sum_1h"] and list(second.columns)[-2:] == ["bid_sum_1h", "bid_max_1h"]


def test_empty_frame(emulated):
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    fset.add_aggregation("bid", ["sum", "stdvar"], "1h")
    out = fset.ingest(_base().iloc[:0])
    assert len(out) == 0 and list(out.columns)[-2:] == ["bid_sum_1h", "bid_stdvar_1h"]


# ------------------------------------------------------------------------------------------------------ add_aggregation
def test_add_aggregation_equals_the_real_reference():
    """the graph steps, class arguments, registered features and errors of every recorded call sequence"""
    from tests.golden import gen_add_aggregation as gen

    with open(gen.GOLDEN) as f:
        want = json.load(f)
    got = [gen.observe(bi.FeatureSet, bi.Entity, kw, calls) for kw, calls in gen.SCENARIOS]
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, gen.SCENARIOS[i])


def test_add_aggregation_returns_the_step_and_rejects_string_operations():
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts")
    step = fset.add_aggregation("bid", ["sum"], "1h", "10m", name="asks")
    assert step is fset.graph.steps["Aggregates"] and step.class_name == "storey.AggregateByKey"
    assert fset["asks_sum_1h"].aggregate is True
    with pytest.raises(MLRunInvalidArgumentError, match="operations must be a list"):
        fset.add_aggregation("bid", "sum", "1h")


def test_spark_engine_is_not_lowered():
    fset = bi.FeatureSet("s", entities=["k"], timestamp_key="ts", engine="spark")
    with pytest.raises(LoweringError, match="spark"):
        fset.add_aggregation("bid", ["sum"], "1h")


def test_golden_file_is_present():
    assert os.path.exists(os.path.join(os.path.dirname(__file__), "golden", "ref_add_aggregation.json"))
