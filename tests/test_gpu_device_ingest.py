"""Feature-set ingest of CUDA columns (torch tensors, DeviceArrays, CUDA-array-interface producers) on the H100: every case
runs the same data through the host columnar path and the device path and asserts the same names, dtypes and bits, the same
counters, prints and refusals.  Needs an H100."""

import contextlib
import ctypes as C
import gc
import io

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import columnar  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from mlrun_b200.feature_store import steps as bs  # noqa: E402
from mlrun_b200.lowering import LoweringError  # noqa: E402
from mlrun_b200.synthetic import ingest_workload  # noqa: E402

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
HOUR = 3600 * 10**9


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


class CaiOnly:
    """a producer with a CUDA array interface (v3, with its stream) and no DLPack, over a torch tensor's memory"""

    def __init__(self, t, typestr=None, stream=None):
        self.t = t
        cai = dict(t.__cuda_array_interface__)
        cai.update(version=3, stream=stream)
        if typestr:
            cai["typestr"] = typestr
        self.__cuda_array_interface__ = cai


def on_device(a):
    """a numpy column -> a CUDA column: torch for what torch holds, a CUDA-array-interface view for the rest"""
    a = np.array(a, copy=True, order="C")
    if a.dtype.kind == "M":
        return torch.from_numpy(a.view(np.int64)).cuda()
    if a.dtype in (np.uint16, np.uint32):
        return CaiOnly(torch.from_numpy(a.view(a.dtype.str.replace("u", "i"))).cuda(), a.dtype.str)
    return torch.from_numpy(a).cuda()


class DLPackOnly:
    """a producer with DLPack and no CUDA array interface (as JAX arrays are), over a torch tensor"""

    def __init__(self, t):
        self.t = t

    def __dlpack_device__(self):
        return self.t.__dlpack_device__()

    def __dlpack__(self, stream=None):
        return self.t.__dlpack__(stream=stream)


def dlpack_only(a):
    a = np.array(a, copy=True, order="C")
    return DLPackOnly(torch.from_numpy(a.view(np.int64) if a.dtype.kind == "M" else a).cuda())


def quiet(fn, *a, **k):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        out = fn(*a, **k)
    return out, buf.getvalue()


def same_batch(dev, host):
    """a DeviceColumnBatch equals a ColumnBatch: names, dtypes and every byte"""
    assert isinstance(dev, columnar.DeviceColumnBatch)
    got = dev.to_host()
    assert got.names == host.names and len(got) == len(host)
    for name in host.names:
        a, b = got[name], host[name]
        assert a.dtype == b.dtype, (name, a.dtype, b.dtype)
        assert a.tobytes() == np.ascontiguousarray(b).tobytes(), name


def both(fs_factory, cols, entities=(), device=on_device, **kw):
    """the host columnar ingest and the device ingest of the same columns -> (device batch, host batch, feature sets)"""
    fh, fd = fs_factory(), fs_factory()
    host, host_out = quiet(fh.ingest, {k: np.ascontiguousarray(v) for k, v in cols.items()}, **kw)
    dev, dev_out = quiet(fd.ingest, {k: device(v) for k, v in cols.items()}, **kw)
    assert dev_out == host_out
    assert fd.plan.violations == fh.plan.violations and fd.plan.unmatched == fh.plan.unmatched
    np.testing.assert_array_equal(fd.plan.counters, fh.plan.counters)
    same_batch(dev, host)
    for k in entities:
        np.testing.assert_array_equal(columnar.DeviceColumn(dev.index[k], k).numpy(), host.index[k])
    return dev, host, fd, fh


def steps_set(steps_fn, **kw):
    def make():
        fs = bi.FeatureSet("s", **kw)
        cur = fs.graph
        for i, st in enumerate(steps_fn(bs)):
            cur = cur.to(st, name=f"step{i}")
        return fs
    return make


# ------------------------------------------------------------------------------------------------------------ ingest
@pytest.mark.parametrize("n_rows", [1, 4095, 4096, 4097, 2**20 + 3])
def test_config5_plans(n_rows):
    wl = ingest_workload(n_rows=n_rows, seed=70 + n_rows % 7)
    cols = {c: wl.df[c].to_numpy() for c in wl.df.columns}
    dev, _host, fd, _fh = both(steps_set(wl.build_steps), cols)
    # staging (1) + columns plan (1) + result dtypes (1 when a column changes dtype)
    assert fd.plan.stats["kernels"] in (2, 3)
    assert fd.plan.stats["staged_bytes"] == sum(a.nbytes for a in cols.values())


EDGE = {
    "v": np.array([-3.5, 0.0, 7.0, 10.0, 25.0, np.nan, np.inf, -np.inf], dtype=np.float32),
    "k": np.array([1, 2, 1, 1, 3, 2, -7, 2**30], dtype=np.int32),
    "c": np.array([0, 1, 2, 9, 1, 0, -1, 2], dtype=np.int32),
    "f": np.array([0, 1, 2, 2.5, np.nan, 1, 0, 2], dtype=np.float32),
    "timestamp": pd.to_datetime(["1969-12-31 23:59:59", "1970-01-01 00:00:00", "2000-02-29 13:14:15", "2024-12-31 00:00:01",
                                 "1900-03-01 00:00:00", "2038-01-19 03:14:08", "1677-09-22 00:00:00",
                                 "2262-04-11 23:47:16"]).to_numpy().astype("datetime64[ns]"),
}


@pytest.mark.parametrize("device", [on_device, dlpack_only], ids=["torch", "dlpack-only"])
def test_edge_values_validators_and_map_misses(device):
    def steps(api):
        return [api.Imputer(mapping={"f": 1, "v": 100.0}),
                api.MapValues(mapping={"v": {"ranges": {5: ["-inf", 0], 6: [0, 10], 7: [5, 20]}}, "k": {1: 10.0, 2: 0.5}},
                              with_original_features=True),
                api.OneHotEncoder(mapping={"c": [0, 1, 2]}),
                api.DateExtractor(parts=["year", "month", "day", "hour", "minute", "second", "day_of_week", "day_of_year",
                                         "quarter", "is_leap_year", "is_month_end"]),
                api.FeaturesetValidator(validators={"v": api.MinMaxValidator(severity="warn", min=-1, max=9),
                                                    "k_mapped": api.MinMaxValidator(severity="warn", max=5)})]
    _dev, _host, fd, _fh = both(steps_set(steps, timestamp_key="timestamp"), EDGE, device=device)
    assert fd.plan.unmatched == {"v_mapped": 3, "k_mapped": 3, "c": 2}


def test_every_conversion_kind_and_narrow_inputs():
    n = 5000
    rng = np.random.default_rng(3)
    ts = (rng.integers(-2_000_000_000, 2_000_000_000, n) * 10**9).astype("datetime64[ns]")
    ts[[5, 77]] = np.datetime64("NaT")
    cols = {"timestamp": ts, "when": (rng.integers(0, 2_000_000_000, n) * 10**9).astype("datetime64[ns]"),
            "a": rng.integers(0, 3, n).astype(np.int32), "b": rng.integers(0, 2, n).astype(np.int32),
            "r": rng.normal(size=n).astype(np.float32), "i8": rng.integers(-128, 128, n).astype(np.int8),
            "u8": rng.integers(0, 256, n).astype(np.uint8), "i16": rng.integers(-2**15, 2**15, n).astype(np.int16),
            "u16": rng.integers(0, 2**16, n).astype(np.uint16), "flag": rng.random(n) < 0.5}

    def steps(api):
        return [api.DateExtractor(parts=["hour", "is_leap_year"]),                          # NaT -> float64 NaN
                api.DateExtractor(parts=["is_year_end", "day"], timestamp_col="when"),      # is_* -> bool
                api.MapValues(mapping={"a": {0: 1.0, 1: 2.0, 2: 3.0},                      # int32 words, float labels -> float64
                                       "r": {"ranges": {1: ["-inf", 0], 2: [0, "inf"]}},    # float32, int labels, all hit -> int32
                                       "b": {0: 2**40, 1: 3}},                              # float32 words, int labels -> int32
                              with_original_features=True)]
    dev, host, fd, _fh = both(steps_set(steps, timestamp_key="timestamp"), cols)
    kinds = {k: str(host[k].dtype) for k in ("a_mapped", "r_mapped", "b_mapped", "timestamp_hour", "timestamp_is_leap_year",
                                              "when_is_year_end", "when_day", "i8", "u16", "flag")}
    assert kinds == {"a_mapped": "float64", "r_mapped": "int32", "b_mapped": "int32", "timestamp_hour": "float64",
                     "timestamp_is_leap_year": "float64", "when_is_year_end": "bool", "when_day": "int32", "i8": "int32",
                     "u16": "int32", "flag": "int32"}
    assert fd.plan.stats["kernels"] == 3
    assert dev["timestamp"].dtype == np.dtype("datetime64[ns]")
    assert torch.from_dlpack(dev["timestamp"]).dtype == torch.int64


def test_int32_map_sources_float32_would_round_are_refused_like_the_host():
    cols = {"k": np.array([1, 2**24 + 1, 3], dtype=np.int32)}

    def steps(api):
        return [api.MapValues(mapping={"k": {1: 0.5}})]
    msgs = []
    for src in (cols, {"k": on_device(cols["k"])}):
        with pytest.raises(LoweringError) as e:
            steps_set(steps)().ingest(src)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "beyond 2^24" in msgs[0]


# ------------------------------------------------------------------------------------------------------- aggregation
def agg_set(n_keys):
    def make():
        fs = bi.FeatureSet("tx", entities=["id"] if n_keys == 1 else ["hi", "lo"], timestamp_key="ts")
        fs.add_aggregation("x", ["count", "sum", "sqr", "max", "min", "first", "last", "avg", "stdvar", "stddev"],
                           ["1h", "1d"], "10m", name="xa")
        fs.add_aggregation("y", ["sum", "min"], ["6h"], name="yf")
        return fs
    return make


def agg_cols(rng, n, keys):
    ts = np.sort(rng.integers(0, 3 * 24 * HOUR, n)).astype("datetime64[ns]")  # each key's rows in time order
    return {**keys, "ts": ts,
            "x": (rng.integers(-2**14 + 1, 2**14, n) / 1024).astype(np.float32),
            "y": rng.integers(-2**15 + 1, 2**15, n).astype(np.int32)}


# the aggregations of test_gpu_aggregate_paths.test_one_structure_serves_aggregations_reading_subsets_of_its_fields
FIELDS = [("x", ["min"], ["1h", "1d"], "10m", "mn"), ("x", ["count", "first"], ["6h"], None, "cf"),
          ("x", ["stddev"], ["2h", "2d"], "1h", "sd"), ("x", ["sqr", "max"], ["30m"], "5m", "sm"),
          ("x", ["avg"], ["1d"], None, "av"), ("y", ["count", "first", "last"], ["1h"], "1m", "y")]
# seven keys per kind: the workload's keys 0..6 index these
KEY_VALUES = {"int64": {"id": np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX, 2**40], np.int64)},
              "int32": {"id": np.array([-2**31, -2**31 + 1, -1, 0, 1, 2**31 - 1, 77], np.int32)},
              "int16": {"id": np.array([-2**15, -1, 0, 1, 2**15 - 1, 5, 9], np.int16)},
              "uint32": {"id": np.array([0, 1, 2**31, 2**32 - 1, 7, 2**31 - 1, 2**16], np.uint32)},
              "pair": {"hi": np.array([-2**31, -1, 0, 0, 2**31 - 1, -1, 5], np.int32),
                       "lo": np.array([-2**31, -1, -1, 0, 2**31 - 1, -2**31, 5], np.int32)}}


@pytest.mark.parametrize("n", [4000, 2**20 + 1])
@pytest.mark.parametrize("kind", list(KEY_VALUES))
def test_aggregations_of_the_exact_workload_under_every_key_kind(kind, n):
    """test_gpu_aggregate's workload (per-key non-decreasing times, 10 % of draws at the window start) and the fields
    test's aggregations, with the seven keys spelt as each key kind, int64 and int32 extremes included"""
    from tests.test_gpu_aggregate import DAY, workload

    rng = np.random.default_rng(12)
    k, ts = workload(rng, n, 7, 3 * DAY)
    x = rng.normal(size=n).astype(np.float32) * 10 + 3
    y = rng.normal(size=n).astype(np.float32)
    ids = {name: vals[k] for name, vals in KEY_VALUES[kind].items()}
    cols = {**ids, "ts": ts.astype("datetime64[ns]"), "x": x, "y": y}

    def make():
        fs = bi.FeatureSet("tx", entities=list(ids), timestamp_key="ts")
        for column, ops, windows, period, name in FIELDS:
            fs.add_aggregation(column, ops, windows, period, name=name)
        return fs
    gc.collect()
    before = nat.darray_live()
    dev, _host, fd, fh = both(make, cols, entities=list(ids))
    assert fd.plan.agg.stats["kernels"] == fh.plan.agg.stats["kernels"]
    # staging + keys + columns plan + the aggregation's launches
    assert fd.plan.stats["kernels"] == 3 + fh.plan.agg.stats["kernels"]
    del dev
    gc.collect()
    assert nat.darray_live() == before


@pytest.mark.parametrize("kind", list(KEY_VALUES) + ["int8", "uint8", "uint16"])
def test_keys_kernel_encodes_exactly_as_encode_keys(kind):
    """every 64-bit key of b2s_keys_encode_device equals keys._encode_keys' on the same columns"""
    from mlrun_b200.feature_store.keys import _encode_keys, _key_kind

    rng = np.random.default_rng(8)
    n = 100_003
    if kind in KEY_VALUES:
        cols = {name: np.r_[vals, vals[rng.integers(0, len(vals), n - len(vals))]] for name, vals in KEY_VALUES[kind].items()}
    else:
        info = np.iinfo(kind)
        cols = {"id": np.r_[np.array([info.min, info.max, 0], kind), rng.integers(info.min, info.max + 1, n - 3).astype(kind)]}
    if kind == "pair":  # every combination of the extremes of both halves
        edge = np.array([-2**31, -2**31 + 1, -1, 0, 1, 2**31 - 1], np.int32)
        cols = {"hi": np.r_[np.repeat(edge, 6), cols["hi"]], "lo": np.r_[np.tile(edge, 6), cols["lo"]]}
        n = len(cols["hi"])
    names = list(cols)
    frame = pd.DataFrame(cols)
    want = _encode_keys(frame, names, _key_kind(frame, names, "k"), "k")
    held = [columnar.DeviceColumn(on_device(cols[c]), c).acquire() for c in names]
    out = nat.DeviceArray(nat.darray_alloc(8 * n), (n,), np.int64)
    kc = (nat.KeyCol * len(held))(*[nat.KeyCol(h.ptr, h.dtype.itemsize, int(h.dtype.kind == "i")) for h in held])
    before = nat.launch_count()
    nat.check(nat.load().b2s_keys_encode_device(kc, len(held), n, out.ptr, None))
    assert nat.launch_count() - before == 1
    np.testing.assert_array_equal(out.numpy(), want)
    for h in held:
        h.release()


def test_an_aggregation_step_added_by_class_checks_keys_like_the_host():
    """a step given as the AggregateByKey class aggregates without the step name the graph scan looks for: the keys are
    still refused, and still encoded, exactly as on the host"""
    rng = np.random.default_rng(4)
    n = 3000
    cols = {"id": rng.integers(0, 9, n).astype(np.float32), "ts": np.sort(rng.integers(0, 10**13, n)).astype("datetime64[ns]"),
            "x": rng.normal(size=n).astype(np.float32)}

    def make():
        fs = bi.FeatureSet("tx", entities=["id"], timestamp_key="ts")
        fs.graph.to(bi.AggregateByKey, name="agg", time_field="ts",
                    aggregates=[{"name": "x", "column": "x", "operations": ["sum", "max"], "windows": ["1h"], "period": "10m"}])
        return fs
    msgs = []
    for dev in (False, True):
        with pytest.raises(LoweringError) as e:
            make().ingest({k: on_device(v) if dev else v for k, v in cols.items()})
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "are not lowered" in msgs[0]
    cols["id"] = cols["id"].astype(np.int64)
    _dev, _host, fd, _fh = both(make, cols, entities=["id"])
    assert fd.plan.agg is not None and "x_sum_1h" in _host.names


@pytest.mark.parametrize("bad", ["late", "nat", "nan"])
def test_aggregation_refusals_carry_the_host_messages(bad):
    rng = np.random.default_rng(5)
    cols = agg_cols(rng, 1000, {"id": rng.integers(0, 5, 1000).astype(np.int64)})
    if bad == "late":
        cols["ts"] = cols["ts"][::-1].copy()
    elif bad == "nat":
        cols["ts"][[3, 9]] = np.datetime64("NaT")
    else:
        cols["x"][[4]] = np.nan
    msgs = []
    for dev in (False, True):
        with pytest.raises(LoweringError) as e:
            agg_set(1)().ingest({k: on_device(v) if dev else v for k, v in cols.items()})
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]


# ------------------------------------------------------------------------------------------------ streams, lifetimes
def imputed(name):
    """a feature set whose graph only imputes `name` (its columns hold no NaN: every value passes through)"""
    fs = bi.FeatureSet("s")
    fs.graph.to(bs.Imputer(mapping={name: 0.0}))
    return fs


def test_columns_written_on_a_side_stream_just_before_the_call():
    n = 1 << 22
    side = torch.cuda.Stream()
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # keep the side stream busy well past the call's start
        x.copy_(torch.arange(n, dtype=torch.float32, device="cuda") * 0.5)
        out = imputed("x").ingest({"x": x})
    np.testing.assert_array_equal(out["x"].numpy(), np.arange(n, dtype=np.float32) * 0.5)
    # a CUDA-array-interface v3 producer names its stream
    y = torch.empty(n, dtype=torch.float32, device="cuda")
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        y.fill_(3.0)
    out = imputed("y").ingest({"y": CaiOnly(y, stream=side.cuda_stream)})
    assert (out["y"].numpy() == 3.0).all()


def test_results_outlive_the_inputs_and_free_with_the_last_view():
    torch.cuda.synchronize()
    gc.collect()
    before = nat.darray_live()
    cols = {"timestamp": torch.arange(1000, dtype=torch.int64, device="cuda") * 10**12,
            "v": torch.ones(1000, dtype=torch.float32, device="cuda")}
    fs = bi.FeatureSet("s", timestamp_key="timestamp")
    fs.graph.to(bs.DateExtractor(parts=["year"]))
    out = fs.ingest(cols)
    del cols
    torch.cuda.empty_cache()
    keep = torch.from_dlpack(out["timestamp_year"])
    v = out["v"]
    del out
    assert nat.darray_live() > before
    assert (v.numpy() == 1).all() and int(keep.min()) == 1970
    del v, keep
    gc.collect()
    assert nat.darray_live() == before


def test_a_device_batch_is_ingested_again():
    n = 3000
    cols = {"timestamp": (np.arange(n) * 10**9).astype("datetime64[ns]"), "v": np.arange(n, dtype=np.float32)}
    fs = steps_set(lambda api: [api.DateExtractor(parts=["hour"])], timestamp_key="timestamp")()
    first = fs.ingest({k: on_device(v) for k, v in cols.items()})
    again = imputed("v").ingest(first)
    same_batch(again, imputed("v").ingest(dict(first.to_host().columns)))


# -------------------------------------------------------------------------------------------------- C-ABI refusals
def test_new_entry_points_refuse_bad_arguments_with_no_launch():
    lib = nat.load()
    buf = nat.DeviceArray(nat.darray_alloc(4096, zero=True), (4096,), np.uint8)
    p = buf.ptr
    before = nat.launch_count()

    def conv(*ops, n=16, counters=p, n_counters=1):
        arr = (nat.Convert * max(len(ops), 1))(*ops)
        return lib.b2s_cols_convert_device(arr if ops else None, len(ops), n, counters, n_counters, None)

    bad = [conv(n=16),                                                        # no operations
           conv(nat.Convert(p, p, 11, 0)),                                   # unknown kind
           conv(nat.Convert(None, p, nat.CONV_COPY4, 0)),                    # null source
           conv(nat.Convert(p + 2, p, nat.CONV_COPY4, 0)),                   # misaligned source
           conv(nat.Convert(p, p + 4, nat.CONV_COPY8, 0)),                   # misaligned 8-byte destination
           conv(nat.Convert(p, p + 1, nat.CONV_I32_BOOL, 0), n=-1),          # negative n
           conv(nat.Convert(p, None, nat.CONV_CHECK_F32, 1)),                # counter out of range
           conv(nat.Convert(p, None, nat.CONV_CHECK_F32, 0), counters=p + 4)]  # misaligned counters
    keys = nat.DeviceArray(nat.darray_alloc(16 * 8), (16,), np.int64)

    def enc(*cols, n=16, out=keys.ptr):
        arr = (nat.KeyCol * len(cols))(*cols)
        return lib.b2s_keys_encode_device(arr, len(cols), n, out, None)

    bad += [enc(nat.KeyCol(p, 8, 0)),                                        # unsigned 64-bit key
            enc(nat.KeyCol(p, 3, 1)),                                        # bad width
            enc(nat.KeyCol(p, 4, 1), nat.KeyCol(p, 8, 1)),                   # a pair must be two int32
            enc(nat.KeyCol(p + 2, 4, 1)),                                    # misaligned
            enc(nat.KeyCol(None, 4, 1)),                                     # null
            enc(nat.KeyCol(p, 4, 1), out=keys.ptr + 4),                      # misaligned output
            enc(nat.KeyCol(p, 4, 1), nat.KeyCol(p, 4, 1), nat.KeyCol(p, 4, 1))]  # three columns
    h = C.c_void_p()
    bad += [lib.b2s_darray_alloc(-1, 0, C.byref(h)), lib.b2s_darray_view(buf._h, 8, 4096, C.byref(h)),
            lib.b2s_darray_view(buf._h, 4, 8, C.byref(h)), lib.b2s_darray_view(None, 0, 8, C.byref(h))]
    assert bad == [-1] * len(bad)  # B2S_ERR_INVALID
    assert nat.launch_count() == before
