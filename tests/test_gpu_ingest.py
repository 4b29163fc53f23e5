"""Feature-set ingest on the device (columns_kernel through the b2s_cols_* C-ABI) vs the oracle.  Needs an H100."""

import contextlib
import io

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from mlrun_b200.feature_store import steps as bs  # noqa: E402
from mlrun_b200.synthetic import ingest_workload  # noqa: E402
from oracle import ingest as oi  # noqa: E402
from oracle import transforms as ot  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _same(got, want):
    """every value identical (float32 results are compared exactly, as float64); dtypes may differ in width"""
    assert list(got.columns) == list(want.columns)
    pd.testing.assert_frame_equal(got, want, check_dtype=False, check_exact=True)


@pytest.mark.parametrize("n_rows", [1, 5, 4095, 4096, 4097, 20000])
def test_config5_matches_the_per_row_reference_walk(n_rows):
    wl = ingest_workload(n_rows=n_rows, seed=60 + n_rows % 7)
    plan = bi.lower_steps(wl.build_steps(bs), wl.df)
    got = _quiet(plan.run, wl.df)
    if n_rows <= 5000:
        want, n_viol = _quiet(oi.ingest_rows, wl.build_steps(ot), wl.df)
        assert sum(plan.violations.values()) == n_viol
    else:
        want, viol = oi.ingest_columns(wl.build_steps(ot), wl.df)
        assert plan.violations == viol
    _same(got, want)
    oov = {c: int((wl.df[c] == 9).sum()) for c in wl.onehot_cols}
    assert plan.unmatched == {c: n for c, n in oov.items() if n}


def test_config5_full_size_against_the_vectorised_oracle():
    wl = ingest_workload(n_rows=300_000, seed=5)
    plan = bi.lower_steps(wl.build_steps(bs), wl.df)
    got = _quiet(plan.run, wl.df, reference_dtypes=True)
    want, viol = oi.ingest_columns(wl.build_steps(ot), wl.df)
    _same(got, want)
    assert plan.violations == viol and sum(viol.values()) > 0
    # size-independent properties: one-hot rows sum to 0/1, bucket ids follow the imputed value, dates in range
    for c in wl.onehot_cols:
        s = got[[f"{c}_{k}" for k in range(8)]].sum(axis=1)
        assert ((s == 1) == (wl.df[c] != 9)).all()
    assert got["timestamp_hour"].between(0, 23).all() and got["timestamp_day_of_week"].between(0, 6).all()
    assert not got[[c for c in wl.f32_cols if c in got.columns]].isna().any().any()


def test_edge_values_match_the_reference_semantics():
    df = pd.DataFrame({
        "v": np.array([-3.5, 0.0, 7.0, 10.0, 25.0, np.nan, np.inf, -np.inf], dtype=np.float32),
        "k": np.array([1, 2, 1, 1, 3, 2, -7, 2**30], dtype=np.int32),
        "c": np.array([0, 1, 2, 9, 1, 0, -1, 2], dtype=np.int32),
        "f": np.array([0, 1, 2, 2.5, np.nan, 1, 0, 2], dtype=np.float32),
        "timestamp": pd.to_datetime(["1969-12-31 23:59:59", "1970-01-01 00:00:00", "2000-02-29 13:14:15", "2024-12-31 00:00:01",
                                     "1900-03-01 00:00:00", "2038-01-19 03:14:08", "1677-09-22 00:00:00",
                                     "2262-04-11 23:47:16"]).astype("datetime64[ns]"),
    })

    def steps(api):
        return [
            api.Imputer(mapping={"f": 1, "v": 100.0}),
            api.MapValues(mapping={"v": {"ranges": {5: ["-inf", 0], 6: [0, 10], 7: [5, 20]}}, "k": {1: 10, 2: 0.5}},
                          with_original_features=True),
            api.OneHotEncoder(mapping={"c": [0, 1, 2]}),
            api.DateExtractor(parts=["year", "month", "day", "hour", "minute", "second", "day_of_week", "dayofweek",
                                     "day_of_year", "quarter"]),
            api.FeaturesetValidator(validators={"v": api.MinMaxValidator(severity="warn", min=-1, max=9),
                                                "k_mapped": api.MinMaxValidator(severity="warn", max=5)}),
        ]

    plan = bi.lower_steps(steps(bs), df)
    got = _quiet(plan.run, df)
    want, n_viol = _quiet(oi.ingest_rows, steps(ot), df)
    _same(got, want)
    assert sum(plan.violations.values()) == n_viol
    assert plan.unmatched == {"v_mapped": 3, "k_mapped": 3, "c": 2}
    assert not got["f"].isna().any()


def test_nat_and_wide_date_range():
    rng = np.random.default_rng(9)
    secs = rng.integers(-9_000_000_000, 9_000_000_000, size=50_000)  # 1684 .. 2255
    ts = (secs * 1_000_000_000).astype("datetime64[ns]")
    df = pd.DataFrame({"timestamp": ts, "x": rng.normal(size=len(ts)).astype(np.float32)})
    parts = ["year", "month", "day", "hour", "minute", "second", "day_of_week", "day_of_year", "quarter", "is_leap_year",
             "days_in_month", "is_month_start", "is_month_end", "is_quarter_start", "is_quarter_end", "is_year_start",
             "is_year_end", "week", "weekofyear"]
    plan = bi.lower_steps([bs.DateExtractor(parts=parts)], df)
    got = plan.run(df)
    want, _ = oi.ingest_columns([ot.DateExtractor(parts=parts)], df)
    _same(got, want)
    assert got["timestamp_is_leap_year"].dtype == np.bool_ and got["timestamp_week"].between(1, 53).all()
    rows_want, _ = oi.ingest_rows([ot.DateExtractor(parts=parts)], df.iloc[:300])
    _same(got.iloc[:300], rows_want)
    df.loc[[3, 77], "timestamp"] = pd.NaT
    got = plan.run(df)
    want, _ = oi.ingest_rows([ot.DateExtractor(parts=["hour", "year"])], df.iloc[:100])
    assert np.isnan(got.loc[3, "timestamp_hour"]) and np.isnan(got.loc[77, "timestamp_year"])
    pd.testing.assert_frame_equal(got.iloc[:100][["timestamp_hour", "timestamp_year"]], want[["timestamp_hour", "timestamp_year"]],
                                  check_dtype=False, check_exact=True)
    assert plan.unmatched["timestamp_hour"] == 2


def test_feature_set_ingest_api_and_dropped_validated_column():
    wl = ingest_workload(n_rows=3000, seed=61)
    df = wl.df.copy()
    df.insert(0, "id", np.arange(len(df), dtype=np.int32))
    fs = bi.FeatureSet("cfg5", entities=[bi.Entity("id")], timestamp_key="timestamp")
    cur = fs.graph
    fs["x30"] = bi.Feature(validator=bs.MinMaxValidator(severity="info", min=-1.0, max=1.0))
    fs["x31"] = bi.Feature(validator=bs.MinMaxValidator(severity="info", min=-9.0))  # not in `columns`: not validated
    for step in [bs.Imputer(mapping={"x30": 0.0}), bs.FeaturesetValidator(columns=["x30"]),
                 bs.DropFeatures(features=["x30", "c0"]), bs.OneHotEncoder(mapping={"c1": [0, 1, 2, 3, 4, 5, 6, 7]})]:
        cur = cur.to(step)
    got = _quiet(fs.ingest, df)
    assert got.index.name == "id" and "x30" not in got.columns and "c1_7" in got.columns
    x = df["x30"].fillna(0.0)
    assert fs.plan.violations == {"x30": int(((x < -1.0) | (x > 1.0)).sum())}
    ref_steps = [ot.Imputer(mapping={"x30": 0.0}), ot.DropFeatures(features=["x30", "c0"]),
                 ot.OneHotEncoder(mapping={"c1": [0, 1, 2, 3, 4, 5, 6, 7]})]
    want, _ = oi.ingest_columns(ref_steps, df.set_index("id"))
    _same(got, want)
    # second frame with the same schema re-uses the plan; a different schema re-lowers
    again = _quiet(fs.ingest, df.iloc[:100])
    _same(again, want.iloc[:100])


def test_device_resident_run_matches_the_host_run():
    wl = ingest_workload(n_rows=10_000, seed=62)
    plan = bi.lower_steps(wl.build_steps(bs), wl.df)
    want = _quiet(plan.run, wl.df)
    n = len(wl.df)
    stride = ((n * 4 + 255) // 256) * 256
    ins, _keep = plan._inputs(wl.df)
    d_in = nat.DeviceBuffer(stride * plan.plan.n_in)
    host_in = np.zeros(stride * plan.plan.n_in, dtype=np.uint8)
    for slot, a in ins.items():
        raw = a.view(np.uint8)
        host_in[slot * stride: slot * stride + raw.size] = raw
    d_in.upload(host_in)
    d_out = nat.DeviceBuffer(stride * plan.plan.n_out)
    d_cnt = nat.DeviceBuffer(8 * max(plan.plan.n_counters, 1)).upload(np.zeros(max(plan.plan.n_counters, 1), dtype=np.uint64))
    plan.plan.run_device(d_in.ptr, stride, n, d_out.ptr, stride, d_cnt.ptr)
    nat.load().b2s_device_sync()
    out = d_out.download(np.uint8, (plan.plan.n_out, stride))
    for name, slot, how in plan.out:
        col = want[name].to_numpy()
        if how == "dt":
            got = out[slot: slot + 2].reshape(-1)[: n * 8].view(np.int64)  # an 8-byte column spans two adjacent slots
            np.testing.assert_array_equal(got, col.astype("datetime64[ns]").view(np.int64))
        elif how == "f32" or (isinstance(how, tuple) and how[0] == "map"):
            np.testing.assert_array_equal(out[slot][: n * 4].view(np.float32).astype(np.float64), col.astype(np.float64))
        else:
            np.testing.assert_array_equal(out[slot][: n * 4].view(np.int32), col.astype(np.int32))
    counters = d_cnt.download(np.uint64, (max(plan.plan.n_counters, 1),))
    np.testing.assert_array_equal(counters[: plan.plan.n_counters], plan.counters)
