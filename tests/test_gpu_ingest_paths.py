"""Feature-set ingest on every path of columns_kernel and its host pipeline, against the reference walk.  Needs an H100:
`-m gpu`.

What can serve a frame (csrc/b2s_columns.cuh, csrc/b2s_columns.cu):
  * four item bodies: item_copy32 (4-byte copies), item_plain (imputed float32, validated int32, a validated column that
    DropFeatures removed), item_table (range maps, value maps, one-hot) and item_wide (8-byte copies, date parts);
  * each body moves 16 bytes per access when both bases and both slot strides are multiples of 16 bytes (host runs always
    are), and 4 or 8 bytes per access otherwise; the last chunk of a launch ends in a tail of rows % 4 (item_wide: rows % 2);
  * b2s_cols_run_host: one launch below 2 x 65 536 rows, else a pipeline of 65 536-row ranges whose columns cross PCIe in
    2-D copies wherever the host columns sit at a constant pitch;
  * B2S_COLS_2D, B2S_COLS_CHUNK and B2S_COL_GRID select other copy and launch schedules (read once per process).

References: oracle.ingest.ingest_rows, the per-row walk, up to 5 000 rows and oracle.ingest.ingest_columns above (and for
tables of thousands of entries); pandas Series.dt for dates (tests/ingest_dates.py).  Every comparison is exact: frames
value for value with NaN equal to NaN, device-resident runs word for word against the host run, pass-through copies bit
for bit against their input, and violation / unmatched counters as integers.  Device runs fill their output buffers and
the counter past the last with a sentinel that must survive outside the words the plan writes.  Every case asserts which
path it reached: `stats["kernels"]` of a host run (1, or the number of row ranges), the launch count of a device run.
"""

import contextlib
import io
import json
import math
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import columnar  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from mlrun_b200.feature_store import steps as bs  # noqa: E402
from mlrun_b200.synthetic import ingest_workload  # noqa: E402
from oracle import ingest as oi  # noqa: E402
from oracle import transforms as ot  # noqa: E402
from tests import ingest_dates as idt  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I32_MIN, I32_MAX = -2**31, 2**31 - 1
SENT = 0xA5                    # byte that fills device output buffers before a run
SENT_CNT = 0xA5A5A5A5A5A5A5A5  # the word past the plan's counters
PIPE = 65536                   # rows per range of a pipelined host run (B2S_COLS_CHUNK default)
# every remainder mod 4 in the last 4 096-row chunk, odd counts for the pair tail of item_wide, 1 ... 4 chunks
ROWS = [1, 2, 3, 4, 5, 4095, 4096, 4097, 4099, 8191, 3 * 4096 + 3]
# NaN payloads (quiet, negative, signalling), +-Inf, -0.0, a denormal and +-FLT_MAX: a plain copy keeps their bits
SPECIALS = np.array([0x7FC12345, 0xFFC0BEEF, 0x7F800001, 0x7F800000, 0xFF800000, 0x80000000, 0x00000001, 0x7F7FFFFF,
                     0xFF7FFFFF], dtype=np.uint32).view(np.float32)


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


# ------------------------------------------------------------------------------------------ runs and references
def expected_kernels(n):
    return 1 if n < 2 * PIPE else math.ceil(n / PIPE)


def check_frame(plan, df, steps, rows_walk=None, got=None):
    """the device frame of `plan` (lowered from steps(bs)) equals the reference frame of steps(ot), and the violation
    counters equal the reference's; -> the frame"""
    got = quiet(plan.run, df) if got is None else got
    assert plan.stats["kernels"] == expected_kernels(len(df))
    want, viol = oi.ingest_columns(steps(ot), df)
    if rows_walk if rows_walk is not None else len(df) <= 5000:
        want, n_viol = quiet(oi.ingest_rows, steps(ot), df)
        assert n_viol == sum(viol.values())
    assert list(got.columns) == list(want.columns)
    pd.testing.assert_frame_equal(got, want.astype({c: np.int64 for c in want.columns if want[c].dtype == bool}),
                                  check_dtype=False, check_exact=True)
    assert plan.violations == viol
    return got


def out_layout(iplan):
    """{output slot: dtype} of every slot the plan writes (an 8-byte column at its first slot)"""
    specs, extra = iplan._landing()
    lay = {slot: dt for _n, slot, dt in specs}
    lay.update({s: np.dtype(np.int32) for s in extra})
    assert sum(dt.itemsize // 4 for dt in lay.values()) == iplan.plan.n_out
    return lay


def host_raw(iplan, ins, n):
    """b2s_cols_run_host -> ({output slot: its words as uint32}, counters)"""
    outs = {s: np.empty(n, dtype=dt) for s, dt in out_layout(iplan).items()}
    counters, stats = iplan.plan.run_host(ins, n, outs, with_stats=True)
    assert stats["kernels"] == expected_kernels(n)
    return {s: a.view(np.uint32) for s, a in outs.items()}, counters


# device layouts: (slot stride past the 16-byte multiple, base offset of both buffers); only (0, 0) takes 16-byte accesses
LAYOUTS = {"vector": (0, 0), "stride8": (8, 0), "base8": (0, 8), "both": (8, 8)}


def device_raw(iplan, ins, n, layout):
    """b2s_cols_run_device over sentinel-filled buffers at a LAYOUTS entry (or an (extra, offset) pair)
    -> ({output slot: uint32 words}, counters)"""
    extra, off = LAYOUTS[layout] if isinstance(layout, str) else layout
    p = iplan.plan
    stride = (n * 4 + 15) // 16 * 16 + extra
    host_in = np.full(off + p.n_in * stride + 16, 0x5A, dtype=np.uint8)
    for slot, a in ins.items():
        raw = a.view(np.uint8)
        host_in[off + slot * stride: off + slot * stride + raw.size] = raw
    d_in = nat.DeviceBuffer(host_in.size).upload(host_in)
    out_bytes = off + p.n_out * stride + 64
    d_out = nat.DeviceBuffer(out_bytes).upload(np.full(out_bytes, SENT, dtype=np.uint8))
    cnt = np.zeros(p.n_counters + 1, dtype=np.uint64)
    cnt[-1] = SENT_CNT
    d_cnt = nat.DeviceBuffer(cnt.nbytes).upload(cnt)
    before = nat.launch_count()
    p.run_device(d_in.ptr + off, stride, n, d_out.ptr + off, stride, d_cnt.ptr)
    nat.load().b2s_device_sync()
    assert nat.launch_count() - before == 1
    raw = d_out.download(np.uint8, (out_bytes,))
    counters = d_cnt.download(np.uint64, (p.n_counters + 1,))
    assert counters[-1] == SENT_CNT
    written = np.zeros(out_bytes, dtype=bool)
    outs = {}
    for s, dt in out_layout(iplan).items():
        a = off + s * stride
        written[a: a + n * dt.itemsize] = True
        outs[s] = raw[a: a + n * dt.itemsize].view(np.uint32)
    untouched = raw[~written]
    assert (untouched == SENT).all(), f"{int((untouched != SENT).sum())} bytes outside the output words were written"
    return outs, counters[:-1]


def assert_same_words(got, want, what):
    assert got.keys() == want.keys()
    for s in want:
        bad = np.flatnonzero(got[s] != want[s])
        assert bad.size == 0, f"{what}: output slot {s} differs in {bad.size} words, first at word {bad[0]}"


def run_everywhere(steps, df, layouts=tuple(LAYOUTS), rows_walk=None):
    """frame vs reference, then the host run's words against every device layout; -> (plan, frame, host words, inputs)"""
    plan = bi.lower_steps(steps(bs), df)
    got = check_frame(plan, df, steps, rows_walk=rows_walk)
    ins, _keep = plan._inputs(df)
    words, counters = host_raw(plan, ins, len(df))
    np.testing.assert_array_equal(counters, plan.counters)
    for lay in layouts:
        dwords, dcounters = device_raw(plan, ins, len(df), lay)
        assert_same_words(dwords, words, lay)
        np.testing.assert_array_equal(dcounters, counters)
    return plan, got, words, ins


def out_slot(plan, name):
    return next(slot for n, slot, _how in plan.out if n == name)


# ------------------------------------------------------------------------------------------ 1. every item body
def bodies_frame(n, seed=0):
    rng = np.random.default_rng(seed)
    a = rng.normal(size=n).astype(np.float32)
    hit = rng.random(n) < 0.2
    a[hit] = rng.choice(SPECIALS, size=int(hit.sum()))
    a[: min(n, len(SPECIALS))] = SPECIALS[: min(n, len(SPECIALS))]
    f = rng.normal(size=n).astype(np.float32)
    f[rng.random(n) < 0.3] = np.nan
    r = (rng.normal(size=n) * 2).astype(np.float32)
    r[rng.random(n) < 0.1] = np.nan
    b = rng.integers(I32_MIN, I32_MAX, size=n, endpoint=True, dtype=np.int64).astype(np.int32)
    b[:2] = [I32_MIN, I32_MAX][: min(n, 2)]
    secs = rng.integers(-2_000_000_000, 4_000_000_000, size=n) * 1_000_000_000 + rng.integers(0, 10**9, size=n)
    return pd.DataFrame({
        "a": a, "b": b, "f": f,
        "k": rng.integers(-2000, 2000, size=n).astype(np.int32),
        "g": rng.normal(size=n).astype(np.float32),
        "r": r,
        "v": rng.integers(0, 5, size=n).astype(np.int32),
        "w": rng.choice(np.array([0.5, -1.0, 3.0, np.nan], dtype=np.float32), size=n),
        "c": rng.integers(0, 4, size=n).astype(np.int32),
        "t": secs.astype("datetime64[ns]"),
    })


def bodies_steps(api):
    return [
        api.FeaturesetValidator(validators={"k": api.MinMaxValidator(severity="info", min=-1000, max=1000),
                                            "g": api.MinMaxValidator(severity="info", min=-1.0, max=1.0)}),
        api.DropFeatures(features=["g"]),
        api.MapValues(mapping={"r": {"ranges": {1: ["-inf", -0.5], 2: [-0.5, 0.5], 3: [0.25, "inf"]}},
                               "v": {0: 10, 1: 11, 2: 12}, "w": {0.5: 1.5, -1.0: 2.0}}, with_original_features=True),
        api.OneHotEncoder(mapping={"c": [0, 1, 2]}),
        api.DateExtractor(parts=["year", "hour", "day_of_week", "week"], timestamp_col="t"),
        api.Imputer(mapping={"f": 0.25}),  # last: the reference's Imputer turns every other NaN into None
    ]


@pytest.mark.parametrize("n", ROWS)
def test_every_item_body_vector_and_scalar(n):
    """item_copy32 (a, b), item_plain (f imputed, k validated int32, g validated and dropped), item_table (r range, v / w value,
    c one-hot), item_wide (t copied, four date parts): the host run (16-byte accesses) and device runs at every layout agree
    word for word, and the frame equals the reference"""
    df = bodies_frame(n, seed=n)
    plan, got, words, ins = run_everywhere(bodies_steps, df)
    kinds = {op[0] for op in plan.ops}
    assert kinds == {"copy", "check", "range", "value", "onehot", "date"}
    for name in ("a", "b"):  # plain copies keep every bit, NaN payloads included
        np.testing.assert_array_equal(words[out_slot(plan, name)], df[name].to_numpy().view(np.uint32))
    np.testing.assert_array_equal(words[out_slot(plan, "t")].view(np.int64), df["t"].to_numpy().view(np.int64))
    assert plan.unmatched.get("r_mapped", 0) == int(np.isnan(df["r"]).sum())
    assert plan.unmatched.get("w_mapped", 0) == int((~df["w"].isin([0.5, -1.0])).sum())
    assert plan.unmatched.get("c", 0) == int((df["c"] == 3).sum())


# ------------------------------------------------------------------------------------------ 2. table edges
def test_range_table_edges():
    """1 and 4 096 entries; overlapping ranges (the first in mapping order wins); values exactly at lo and hi (half-open);
    +-inf bounds; NaN without a fill passes through and is counted, NaN with a fill lands in a range"""
    n = 4099
    rng = np.random.default_rng(1)
    edges = np.array([-1e30, -2048, -1, -0.5, 0, 0.5, 5, 10, 15, 2047, 2048, np.inf, -np.inf, np.nan], dtype=np.float32)
    base = rng.uniform(-2100, 2100, size=n).astype(np.float32)
    base[: len(edges)] = edges
    df = pd.DataFrame({"one": base, "big": np.roll(base, 7), "ovl": np.roll(base, 3) / 100})
    big = {i: [i / 2, i / 2 + 0.5] for i in range(-2048, 2048)}  # 4 096 ranges of width 0.5 over [-1024, 1024)

    def steps(api):
        return [api.MapValues(mapping={"one": {"ranges": {-3: [-1, 5]}},
                                       "big": {"ranges": big},
                                       "ovl": {"ranges": {1: [0, 10], 2: [5, 15], 3: ["-inf", "inf"], 4: [-100, 100]}}},
                              with_original_features=True)]

    plan, got, _w, _i = run_everywhere(steps, df, layouts=("vector", "both"), rows_walk=False)
    ovl = df["ovl"].to_numpy()
    assert len(big) == 4096 and plan.unmatched["ovl_mapped"] == int((np.isnan(ovl) | (ovl == np.inf)).sum()) > 0
    assert got["ovl_mapped"][(ovl >= 5) & (ovl < 10)].eq(1).all() and got["ovl_mapped"][(ovl >= 10) & (ovl < 15)].eq(2).all()
    assert got.loc[df["one"] == -1, "one_mapped"].eq(-3).all() and got.loc[df["one"] == 5, "one_mapped"].eq(5).all()
    check_frame(plan, df.iloc[:300], steps, rows_walk=True)  # the per-row walk on the same plan, 4 096-entry table included

    fill = pd.DataFrame({"fill": np.where(rng.random(n) < 0.3, np.nan, base).astype(np.float32)})

    def filled(api):
        return [api.Imputer(mapping={"fill": 7.0}),
                api.MapValues(mapping={"fill": {"ranges": {70: [5, 10], 80: ["-inf", 5]}}}, with_original_features=True)]

    _plan, got, _w, _i = run_everywhere(filled, fill, layouts=("vector", "both"))
    assert got["fill_mapped"][np.isnan(fill["fill"])].eq(70).all()


def test_value_map_edges():
    """4 096 keys; a -0.0 key matches 0.0 and a 0.0 key matches -0.0 (Python's ==); NaN never matches"""
    n = 4097
    rng = np.random.default_rng(2)
    keys = [-0.0] + [float(k) for k in range(1, 4096)]
    x = rng.integers(-10, 4200, size=n).astype(np.float32)
    x[:5] = [-0.0, 0.0, np.nan, 4095, 4096]
    df = pd.DataFrame({"p": x, "q": -x})

    def steps(api):
        return [api.MapValues(mapping={"p": {k: 2 * i + 1 for i, k in enumerate(keys)}, "q": {0.0: 9, -5.0: 8}},
                              with_original_features=True)]

    plan, got, _w, _i = run_everywhere(steps, df, layouts=("vector", "both"), rows_walk=False)
    assert got["p_mapped"][:5].tolist()[:2] == [1, 1] and got["q_mapped"][:2].tolist() == [9, 9]
    assert plan.unmatched["p_mapped"] == int((~((x == 0) | ((x >= 1) & (x <= 4095)))).sum())
    check_frame(plan, df.iloc[:200], steps, rows_walk=True)


@pytest.mark.parametrize("cats", [[5], list(range(4096)), [3, 1, 3, 2, 1], [-5, -1, 0, -2**31], [2**31, -2**31 - 1, 2**40, 7]],
                         ids=["one", "4096", "duplicates", "negative", "outside-int32"])
def test_onehot_edges(cats):
    n = 4099
    rng = np.random.default_rng(len(cats))
    c = rng.choice(np.array(list(dict.fromkeys(c for c in cats if I32_MIN <= c <= I32_MAX)) + [6, I32_MAX], dtype=np.int64),
                   size=n).astype(np.int32)

    def steps(api):
        return [api.OneHotEncoder(mapping={"c": cats})]

    plan, got, _w, _i = run_everywhere(steps, pd.DataFrame({"c": c}), layouts=("vector", "both"), rows_walk=len(cats) < 100)
    known = [k for k in dict.fromkeys(cats) if I32_MIN <= k <= I32_MAX]
    assert len(got.columns) == len(dict.fromkeys(cats))
    assert plan.unmatched.get("c", 0) == int((~np.isin(c, known)).sum())


def test_int_extremes_and_narrow_dtypes():
    """INT32_MIN / INT32_MAX through a copy, a validator, one-hot and a map; int8, int16, uint8, uint16 and bool sources"""
    n = 4097
    rng = np.random.default_rng(3)
    i32 = rng.choice(np.array([I32_MIN, I32_MAX, 0, -1, 1], dtype=np.int32), size=n)
    df = pd.DataFrame({
        "i32": i32, "j32": np.roll(i32, 1), "o32": np.roll(i32, 2),
        "i8": rng.integers(-128, 128, size=n).astype(np.int8),
        "i16": rng.integers(-32768, 32768, size=n).astype(np.int16),
        "u8": rng.integers(0, 256, size=n).astype(np.uint8),
        "u16": rng.integers(0, 65536, size=n).astype(np.uint16),
        "bo": rng.random(n) < 0.5,
    })

    def steps(api):
        return [
            api.FeaturesetValidator(validators={"i32": api.MinMaxValidator(severity="info", min=I32_MIN + 1, max=I32_MAX - 1),
                                                "i8": api.MinMaxValidator(severity="info", max=126)}),
            api.MapValues(mapping={"j32": {I32_MAX: 1, I32_MIN: 2}, "i8": {-128: 5, 127: 6},
                                   "u8": {"ranges": {1: [0, 128], 2: [128, 255]}}, "bo": {1: 7}},
                          with_original_features=True),
            api.OneHotEncoder(mapping={"o32": [I32_MIN, I32_MAX, 0], "i16": [-32768, 32767, 0], "u16": [65535, 0]}),
        ]

    plan, got, words, _i = run_everywhere(steps, df)
    np.testing.assert_array_equal(words[out_slot(plan, "i32")].view(np.int32), i32)
    assert plan.violations == {"i32": int(np.isin(i32, [I32_MIN, I32_MAX]).sum()), "i8": int((df["i8"] == 127).sum())}
    assert got["j32_mapped"].dtype == np.int32 and plan.unmatched["u8_mapped"] == int((df["u8"] == 255).sum())


# ------------------------------------------------------------------------------------------ 3. validators
@pytest.mark.parametrize("n", [4099, 100_003])
def test_validators(n):
    """min only, max only, both, min == max, an int column with fractional bounds, a validated column dropped after the
    check; NaN is never a violation.  At 100 003 rows more than 2^16 violations of one column spread over 25 items"""
    rng = np.random.default_rng(n)
    x = rng.normal(size=(6, n)).astype(np.float32)
    x[:, rng.random(n) < 0.05] = np.nan
    df = pd.DataFrame({"lo": x[0], "hi": x[1], "both": x[2], "eq": np.round(x[3]).astype(np.float32),
                       "int": rng.integers(-3, 5, size=n).astype(np.int32), "dropped": x[4], "many": x[5] * 10})
    def steps(api):
        v = api.MinMaxValidator
        return [api.FeaturesetValidator(validators={
            "lo": v(severity="info", min=-0.5), "hi": v(severity="info", max=0.25), "both": v(severity="info", min=-1, max=1),
            "eq": v(severity="info", min=0, max=0), "int": v(severity="info", min=-0.5, max=2.5),
            "dropped": v(severity="info", min=-0.1, max=0.1), "many": v(severity="info", min=5, max=6)}),
            api.DropFeatures(features=["dropped"])]

    plan, _got, _w, _i = run_everywhere(steps, df, layouts=("vector", "both"))
    assert plan.violations["int"] == int(((df["int"] < -0.5) | (df["int"] > 2.5)).sum())
    assert plan.violations["dropped"] > 0 and "dropped" not in _got.columns
    if n > 5000:
        assert plan.violations["many"] > 2**16


# ------------------------------------------------------------------------------------------ 4. dates, exhaustively
@pytest.fixture(scope="module")
def every_day():
    ts = idt.exhaustive_timestamps()
    nat_at = np.arange(17, len(ts), 9973)
    with_nat = np.insert(ts, nat_at, idt.I64_MIN)
    return with_nat, with_nat == idt.I64_MIN


def test_every_date_part_of_every_day(every_day):
    """every day of datetime64[ns] at eight offsets, the range ends and NaT rows through all 18 parts and their aliases:
    the pipelined host run and a device run with 8-byte accesses, against pandas"""
    ts, is_nat = every_day
    n = len(ts)
    df = pd.DataFrame({"t": ts.view("datetime64[ns]")})
    parts = list(nat.DATE_PARTS)
    plan = bi.lower_steps([bs.DateExtractor(parts=parts, timestamp_col="t")], df)
    ins, _keep = plan._inputs(df)
    words, counters = host_raw(plan, ins, n)
    assert (counters == is_nat.sum()).all() and len(counters) == len(parts)
    for name in parts:
        part = nat.DATE_PARTS[name]
        got = words[out_slot(plan, f"t_{name}")].view(np.int32)
        assert (got[is_nat] == -1).all()
        want = idt.pandas_part(ts[~is_nat], part)
        bad = np.flatnonzero(got[~is_nat] != want)
        assert bad.size == 0, f"{name}: {bad.size} differences, first at {ts[~is_nat][bad[0]].view('datetime64[ns]')}"
    dwords, dcounters = device_raw(plan, ins, n, "both")
    assert_same_words(dwords, words, "both")
    np.testing.assert_array_equal(dcounters, counters)


# ------------------------------------------------------------------------------------------ 5. the host pipeline
def pipeline_frame(n, seed):
    """4-byte columns either side of a datetime column, and a one-hot whose middle members are dropped: the 2-D copy runs
    break at the 8-byte column and at the dropped members' landing slots"""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(4, n)).astype(np.float32)
    x[1, rng.random(n) < 0.1] = np.nan
    secs = rng.integers(-3_000_000_000, 3_000_000_000, size=n).astype(np.int64) * 1_000_000_000
    ts = secs.view("datetime64[ns]").copy()
    ts[rng.random(n) < 0.01] = np.datetime64("NaT")
    return pd.DataFrame({"x0": x[0], "x1": x[1], "t": ts, "x2": x[2], "k": rng.integers(0, 100, size=n).astype(np.int32),
                         "c": rng.integers(0, 5, size=n).astype(np.int32), "x3": x[3]})


def pipeline_steps(api):
    return [api.Imputer(mapping={"x1": 0.5}),
            api.OneHotEncoder(mapping={"c": [0, 1, 2, 3]}),
            api.DateExtractor(parts=["hour", "year"], timestamp_col="t"),
            api.FeaturesetValidator(validators={"x2": api.MinMaxValidator(severity="info", min=-1, max=1)}),
            api.MapValues(mapping={"x3": {"ranges": {1: [-1, 0], 2: [0, 1]}}}, with_original_features=True),
            api.DropFeatures(features=["c_1", "c_2"])]


def pipeline_reference(df):
    want, viol = oi.ingest_columns(pipeline_steps(ot), df)
    unmatched = {"x3_mapped": int((~((df["x3"] >= -1) & (df["x3"] < 1))).sum()), "c": int((df["c"] == 4).sum()),
                 "t_hour": int(df["t"].isna().sum()), "t_year": int(df["t"].isna().sum())}
    return want, viol, unmatched


def test_host_pipeline_from_frames_and_pinned_columns():
    """one plan: 131 071 rows (one launch), 131 072 (2 ranges), 131 073 (3, the last of 1 row), 300 000, then small and
    large again so the staging shrinks and regrows; each from a pageable frame and from pinned columns (2-D copies)"""
    n0 = 300_001
    full = pipeline_frame(n0, seed=5)
    plan = bi.lower_steps(pipeline_steps(bs), full)
    assert len(plan._landing()[1]) == 2  # the dropped one-hot members still land somewhere
    for n in (131_071, 131_072, 131_073, 300_000, 131_071, 300_001):
        df = full.iloc[:n].reset_index(drop=True) if n < n0 else full
        want, viol, unmatched = pipeline_reference(df)
        # time columns NaT -> NaN: the frame holds float64, like the reference
        got = quiet(plan.run, df)
        assert plan.stats["kernels"] == expected_kernels(n)
        pd.testing.assert_frame_equal(got, want, check_dtype=False, check_exact=True)
        assert plan.violations == viol and plan.unmatched == unmatched
        pinned = columnar.pinned_columns([(name, df[name].dtype) for name in df.columns], n)
        for name in df.columns:
            pinned[name][:] = df[name].to_numpy()
        batch = quiet(plan.run_columns, pinned)
        assert plan.stats["kernels"] == expected_kernels(n)
        assert batch.names == list(want.columns)
        for name in want.columns:
            np.testing.assert_array_equal(np.asarray(batch[name]), want[name].to_numpy(), err_msg=f"{name} at n={n}")
        assert plan.violations == viol and plan.unmatched == unmatched


# ------------------------------------------------------------------------------------------ 6. environment switches
_SWITCH_CHILD = r"""
import contextlib, io, json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import columnar, ingest as bi, steps as bs
from tests.test_gpu_ingest_paths import pipeline_frame, pipeline_steps
nat.init(0)
res = {}
for n in (10_000, 300_000):
    df = pipeline_frame(n, seed=n)
    plan = bi.lower_steps(pipeline_steps(bs), df)
    cols = columnar.pinned_columns([(c, df[c].dtype) for c in df.columns], n)
    for c in df.columns:
        cols[c][:] = df[c].to_numpy()
    with contextlib.redirect_stdout(io.StringIO()):
        batch = plan.run_columns(cols)
    np.savez(f"{sys.argv[2]}_{n}.npz", counters=plan.counters,
             **{f"col{i}": np.asarray(batch[c]).view(np.uint8) for i, c in enumerate(batch.names)})
    res[n] = int(plan.stats["kernels"])
print(json.dumps(res))
"""


@pytest.fixture(scope="module")
def default_schedule(tmp_path_factory):
    return _switch_run(tmp_path_factory.mktemp("default"), "default", {})


def _switch_run(tmp_path, tag, env):
    script = tmp_path / "child.py"
    script.write_text(_SWITCH_CHILD)
    out = subprocess.run([sys.executable, str(script), ROOT, str(tmp_path / tag)], capture_output=True, text=True,
                         env=dict(os.environ, **env), cwd=ROOT, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    kernels = {int(k): v for k, v in json.loads(out.stdout.strip().splitlines()[-1]).items()}
    return kernels, {n: dict(np.load(tmp_path / f"{tag}_{n}.npz")) for n in kernels}


@pytest.mark.parametrize("env,kernels", [
    ({"B2S_COLS_2D": "0"}, {10_000: 1, 300_000: 5}),
    ({"B2S_COLS_CHUNK": "5000"}, {10_000: 2, 300_000: 37}),  # 5 000 rounds up to 8 192: ranges of 8 192 and 1 808
    ({"B2S_COL_GRID": "-1"}, {10_000: 1, 300_000: 5}),
    ({"B2S_COL_GRID": "1"}, {10_000: 1, 300_000: 5}),
], ids=["2d-off", "chunk-5000", "grid-per-item", "grid-x1"])
def test_environment_switches(tmp_path, default_schedule, env, kernels):
    """each schedule in a process of its own: output bytes and counters equal the default schedule's"""
    base_k, base = default_schedule
    assert base_k == {10_000: 1, 300_000: 5}
    got_k, got = _switch_run(tmp_path, "switched", env)
    assert got_k == kernels
    for n in base:
        assert base[n].keys() == got[n].keys()
        for k in base[n]:
            np.testing.assert_array_equal(got[n][k], base[n][k], err_msg=f"{k} at n={n}")


# ------------------------------------------------------------------------------------------ 7. the two fixes
BIG = np.array([16_777_217, -16_777_219, I32_MAX, I32_MIN, 16_777_216, 1, 2, 0], dtype=np.int32)


@pytest.mark.parametrize("how", ["value-partial", "value-full", "range-partial", "range-full", "value-halves", "range-halves"])
def test_int32_maps_keep_values_beyond_float32(how):
    """int32 values with |v| > 2^24 through range and value maps to int32 integers, partly and fully matched, with a
    validator on the mapped column: the map writes int32 words and every value that passes through is exact.  Maps to
    other values write float32: such a frame is refused before anything runs, and served once every value is float32-exact"""
    n = 4099
    k = np.resize(BIG, n)
    k[8::3] = np.random.default_rng(4).integers(I32_MIN, I32_MAX, size=len(k[8::3]), dtype=np.int64).astype(np.int32)
    if how == "value-partial":
        m = {1: 10, 2: 20}
    elif how == "value-full":
        m = {int(v): i for i, v in enumerate(np.unique(k))}
    elif how == "range-partial":
        m = {"ranges": {10: [1, 3], 20: [-16_777_219, -16_777_218]}}
    else:
        m = {"ranges": {1: ["-inf", -16_777_218], 2: [-16_777_218, 16_777_217], 3: [16_777_217, "inf"]}}
    if how == "value-halves":
        m = {1: 0.5, 2: 20}
    elif how == "range-halves":
        m = {"ranges": {0.5: [1, 3]}}
    df = pd.DataFrame({"k": k})

    def steps(api):
        return [api.MapValues(mapping={"k": m}, with_original_features=True),
                api.FeaturesetValidator(validators={"k_mapped": api.MinMaxValidator(severity="info", min=-2**24, max=2**24)})]

    if how.endswith("halves"):
        plan = bi.lower_steps(steps(bs), df)
        before = nat.launch_count()
        with pytest.raises(bi.LoweringError, match="float32 cannot represent"):
            quiet(plan.run, df)
        assert nat.launch_count() == before
        exact = df[df["k"].astype(np.float32).astype(np.int64) == df["k"]].reset_index(drop=True)
        plan, got, words, _i = run_everywhere(steps, exact)
        assert got["k_mapped"].dtype == np.float32
        return
    plan, got, words, _i = run_everywhere(steps, df)
    mapped = words[out_slot(plan, "k_mapped")].view(np.int32)
    if how.endswith("partial"):
        passes = ~np.isin(k, [1, 2]) if how == "value-partial" else ~(np.isin(k, [1, 2, -16_777_219]))
        np.testing.assert_array_equal(mapped[passes], k[passes])
        assert plan.unmatched["k_mapped"] == int(passes.sum()) and plan.violations["k_mapped"] > 0
    else:
        assert "k_mapped" not in plan.unmatched and got["k_mapped"].dtype.kind == "i"


def test_run_device_refuses_bad_buffers():
    """NULL or misaligned d_in / d_out / d_counters: B2S_ERR_INVALID before any launch.  8-byte alignment is needed only
    where the plan reads or writes an 8-byte column; bases 4 bytes off 16 are served by a plan without one"""
    n = 4099
    df = bodies_frame(n, seed=9)
    wide = bi.lower_steps(bodies_steps(bs), df)  # reads and writes 8-byte columns
    ins, _keep = wide._inputs(df)
    p = wide.plan
    stride = (n * 4 + 15) // 16 * 16
    d_in = nat.DeviceBuffer(p.n_in * stride + 64)
    d_out = nat.DeviceBuffer(p.n_out * stride + 64)
    d_cnt = nat.DeviceBuffer(8 * p.n_counters + 64)
    bad = {"d_in NULL": (0, d_out.ptr, d_cnt.ptr), "d_out NULL": (d_in.ptr, 0, d_cnt.ptr),
           "d_in +1": (d_in.ptr + 1, d_out.ptr, d_cnt.ptr), "d_in +2": (d_in.ptr + 2, d_out.ptr, d_cnt.ptr),
           "d_in +4": (d_in.ptr + 4, d_out.ptr, d_cnt.ptr), "d_out +2": (d_in.ptr, d_out.ptr + 2, d_cnt.ptr),
           "d_out +4": (d_in.ptr, d_out.ptr + 4, d_cnt.ptr), "d_counters +4": (d_in.ptr, d_out.ptr, d_cnt.ptr + 4),
           "d_counters NULL": (d_in.ptr, d_out.ptr, None)}
    for what, (i, o, c) in bad.items():
        before = nat.launch_count()
        with pytest.raises(nat.NativeError, match="aligned|NULL|counters"):
            p.run_device(i, stride, n, o, stride, c)
        assert nat.launch_count() == before, what
    nat.load().b2s_device_sync()

    # a plan of 4-byte columns only takes bases 4 bytes off 8, and gives the host run's words
    narrow_df = df[["a", "b", "f", "k", "r", "c"]]

    def steps(api):
        return [api.Imputer(mapping={"f": 0.25}),
                api.FeaturesetValidator(validators={"k": api.MinMaxValidator(severity="info", min=-1000, max=1000)}),
                api.MapValues(mapping={"r": {"ranges": {1: ["-inf", 0]}}}),
                api.OneHotEncoder(mapping={"c": [0, 1, 2]})]

    narrow = bi.lower_steps(steps(bs), narrow_df)
    ins, _keep = narrow._inputs(narrow_df)
    words, counters = host_raw(narrow, ins, n)
    dwords, dcounters = device_raw(narrow, ins, n, (8, 4))
    assert_same_words(dwords, words, "base4")
    np.testing.assert_array_equal(dcounters, counters)


# ------------------------------------------------------------------------------------------ 8. the ingest6 step shape
def test_ingest6_step_shape():
    """524 288 rows of the benchmark's 255-column schema through run_device: 128 chunks x ~290 ops, far more items than
    the grid's CTAs, so every CTA runs several items and resets its counters between them"""
    n = 524_288
    wl = ingest_workload(n_rows=n, seed=7)
    plan = bi.lower_steps(wl.build_steps(bs), wl.df)
    assert len(plan.ops) * (n // 4096) > 8 * 132 * 8
    got = quiet(plan.run, wl.df)
    assert plan.stats["kernels"] == n // PIPE
    want, viol = oi.ingest_columns(wl.build_steps(ot), wl.df)
    pd.testing.assert_frame_equal(got, want, check_dtype=False, check_exact=True)
    assert plan.violations == viol and sum(viol.values()) > 0
    ins, _keep = plan._inputs(wl.df)
    words, counters = host_raw(plan, ins, n)
    dwords, dcounters = device_raw(plan, ins, n, "vector")
    assert_same_words(dwords, words, "vector")
    np.testing.assert_array_equal(dcounters, counters)
