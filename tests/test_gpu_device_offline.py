"""Feature sets registered from CUDA columns and training tensors built from spines and entity rows in HBM, on the H100.
Every case registers the same data twice, once from CUDA columns (torch tensors, CUDA-array-interface producers, a
DeviceColumnBatch) and once from the equal pandas frame, and runs the same queries on both: the registered state, the
tensors of `get_offline_tensors` (bit for bit, NaN where NaN) and the frames of `get_offline_features` must be equal, and
so must every refusal.

Launches, per call (`nat.launch_count()`):
- `register_offline_frame` of CUDA columns: 1 key encode + 1 timestamp profile (with a timestamp key) + 1 convert (when
  a feature is a 1- or 2-byte int or bool) + 53 for the index build (two 24-launch sorts, 5 more).
- `get_offline_tensors` over a spine registered from CUDA columns: 1 timestamp profile and 24 for the sort (with an as-of
  set) + one join launch per joined set + 2 to find the kept rows + 1 pack launch; the spine's keys were encoded at
  registration.
- `get_offline_tensors` with CUDA entity rows: the same, plus 1 timestamp profile (with an as-of set) and 1 key encode
  per distinct entity key of the vector's sets.
- `b2s_ts_profile_device`: 1."""

import ctypes as C
import gc

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import columnar  # noqa: E402
from mlrun_b200.feature_store import ingest as bi  # noqa: E402
from mlrun_b200.feature_store import offline as boff  # noqa: E402
from mlrun_b200.feature_store import steps as bs  # noqa: E402
from mlrun_b200.lowering import LoweringError  # noqa: E402

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
INDEX_LAUNCHES, SORT_LAUNCHES = 53, 24


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


@pytest.fixture(autouse=True)
def _registry(monkeypatch):
    monkeypatch.setattr(boff, "_OFFLINE", {})
    yield
    for src in list(boff._OFFLINE.values()):
        src.close()


class CaiOnly:
    """a producer with a CUDA array interface (v3) and no DLPack, over a torch tensor's memory"""

    def __init__(self, t, typestr=None, stream=None):
        self.t = t
        cai = dict(t.__cuda_array_interface__)
        cai.update(version=3, stream=stream)
        if typestr:
            cai["typestr"] = typestr
        self.__cuda_array_interface__ = cai


def on_device(a, ts=False):
    """a numpy column -> a CUDA column; a datetime64[ns] column becomes int64 nanoseconds when `ts` (the set's or entity
    frame's timestamp), else a CUDA-array-interface column that states datetime64[ns]"""
    a = np.array(a, copy=True, order="C")
    if a.dtype.kind == "M":
        t = torch.from_numpy(a.view(np.int64)).cuda()
        return t if ts else CaiOnly(t, a.dtype.str)
    if a.dtype in (np.uint16, np.uint32):
        return CaiOnly(torch.from_numpy(a.view(a.dtype.str.replace("u", "i"))).cuda(), a.dtype.str)
    return torch.from_numpy(a).cuda()


def to_device(frame, ts=None):
    return {c: on_device(frame[c].to_numpy(), ts=c == ts) for c in frame.columns}


def make_frame(n, seed=0, n_keys=None, key_dtype=np.int64, unit_ns=1, nat_rows=0, negative=False, extra=True):
    rng = np.random.default_rng(seed)
    n_keys = n_keys or max(1, n // 3)
    ids = rng.integers(0, n_keys, n).astype(key_dtype)
    base = -10**18 if negative else 10**17
    ts = (base + rng.integers(0, 10**6, n) * 997 * 10**6 // unit_ns * unit_ns).astype(np.int64)
    ts[:nat_rows] = I64_MIN
    f32 = rng.normal(size=n).astype(np.float32)
    f32[rng.random(n) < 0.2] = np.nan
    cols = {"id": ids, "ts": ts.view("datetime64[ns]"), "f32": f32, "f64": rng.normal(size=n)}
    if extra:
        cols.update({"i8": rng.integers(-128, 128, n).astype(np.int8), "i16": rng.integers(-3000, 3000, n).astype(np.int16),
                     "i32": rng.integers(-10**9, 10**9, n).astype(np.int32), "u8": rng.integers(0, 256, n).astype(np.uint8),
                     "u16": rng.integers(0, 65536, n).astype(np.uint16), "flag": rng.random(n) < 0.5,
                     "when": (10**18 + rng.integers(0, 10**9, n)).view("datetime64[ns]"),
                     "u32": rng.integers(0, 2**32, n).astype(np.uint32), "i64": rng.integers(0, 10, n).astype(np.int64)})
    return pd.DataFrame(cols)


def state(src):
    ix = src.index
    return (src.features, src.key_kind, src.has_nat, src.ts_factor, ix.n_rows, ix.n_keys, ix.longest_run, ix.row_words,
            _cap(ix))


def _cap(ix):
    cap = C.c_int64()
    nat.check(nat.load().b2s_pit_index_info(ix._h, None, None, None, None, C.byref(cap)))
    return cap.value


def fset(name, ts="ts", entities=("id",)):
    return bi.FeatureSet(name, entities=list(entities), timestamp_key=ts)


def tensors_of(t):
    out = {"features": t.features.numpy(), "order": t.order.numpy(), "columns": list(t.columns), "rows": t.rows}
    out["label"] = None if t.label is None else t.label.numpy()
    return out


def assert_same_tensors(a, b):
    assert a["columns"] == b["columns"] and a["rows"] == b["rows"]
    for k in ("features", "order", "label"):
        if a[k] is None:
            assert b[k] is None
            continue
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape
        assert a[k].tobytes() == b[k].tobytes(), k  # bit for bit: NaN where NaN


def assert_same_frames(a, b):
    assert list(a.columns) == list(b.columns) and list(a.dtypes) == list(b.dtypes) and list(a.index.names) == list(b.index.names)
    pd.testing.assert_frame_equal(a, b, check_exact=True)


def run_both(register, query):
    """register (device) -> query -> register (host) -> query: the two results"""
    register(True)
    dev = query()
    register(False)
    host = query()
    return dev, host


@pytest.fixture
def no_host_copies():
    """the Python-level host copies fail while the fixture is active"""
    def fail(*a, **k):
        raise AssertionError("a column crossed to the host")

    patches = [(columnar.DeviceColumn, "numpy"), (nat.DeviceArray, "numpy"), (columnar.DeviceColumnBatch, "to_host")]

    class Guard:
        def __enter__(self):
            self.mp = pytest.MonkeyPatch()
            for obj, name in patches:
                self.mp.setattr(obj, name, fail)

        def __exit__(self, *exc):
            self.mp.undo()

    return Guard()


# ---- registered state ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key_dtype", ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32"])
def test_registered_state_per_key_dtype(key_dtype, no_host_copies):
    frame = make_frame(1000, seed=1, n_keys=100, key_dtype=key_dtype)
    with no_host_copies:
        before = nat.launch_count()
        dev = state(boff.register_offline_frame(fset("s"), to_device(frame, ts="ts")))
        assert nat.launch_count() - before == 1 + 1 + 1 + INDEX_LAUNCHES
    assert dev == state(boff.register_offline_frame(fset("s"), frame))


def test_registered_state_of_an_int32_pair_and_without_a_timestamp():
    rng = np.random.default_rng(2)
    frame = pd.DataFrame({"a": rng.integers(-5, 5, 500).astype(np.int32), "b": rng.integers(-2**31, 2**31, 500).astype(np.int32),
                          "x": rng.normal(size=500).astype(np.float32)})
    fs = bi.FeatureSet("p", entities=["a", "b"])
    before = nat.launch_count()
    dev = state(boff.register_offline_frame(fs, to_device(frame)))
    assert nat.launch_count() - before == 1 + INDEX_LAUNCHES  # no timestamp, nothing to widen
    host = state(boff.register_offline_frame(fs, frame))
    assert dev == host and dev[1] == "pair" and dev[3] == 10**9


def test_registered_from_a_device_batch_equals_its_host_frame(no_host_copies):
    n = 3000
    rng = np.random.default_rng(3)
    cols = {"ts": torch.from_numpy(10**17 + rng.integers(0, 10**12, n)).cuda(), "x": torch.from_numpy(rng.normal(size=n).astype(np.float32)).cuda(),
            "k": torch.from_numpy(rng.integers(0, 50, n).astype(np.int16)).cuda(), "id": torch.from_numpy(rng.integers(0, 300, n)).cuda()}
    fs = fset("b")
    fs.graph.to(bs.Imputer(mapping={"x": 0.0}))
    batch = fs.ingest(cols)
    assert isinstance(batch, columnar.DeviceColumnBatch) and list(batch.index) == ["id"]
    with no_host_copies:
        dev = state(boff.register_offline_frame(fs, batch))
    frame = batch.to_host().to_pandas()
    assert dev == state(boff.register_offline_frame(fs, frame))
    assert list(dev[0]) == [c for c in frame.reset_index().columns if c not in ("id", "ts")]


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
@pytest.mark.parametrize("negative", [False, True])
def test_timestamp_granularity_and_the_entity_unit_refusal(unit, negative):
    f = boff._UNIT_NS[unit]
    frame = make_frame(400, seed=4, n_keys=40, unit_ns=f, negative=negative, extra=False)
    frame.loc[3, "ts"] = frame.loc[3, "ts"] + pd.Timedelta(f, "ns") if f < 10**9 else frame.loc[3, "ts"]
    ent = frame[["id", "ts"]].iloc[::3].reset_index(drop=True)
    fs = fset("g")
    dev_src = boff.register_offline_frame(fs, to_device(frame, ts="ts"))
    dev_state = state(dev_src)
    host_state = state(boff.register_offline_frame(fs, frame))
    assert dev_state == host_state and dev_state[3] == f
    for eunit in ["s", "ms", "us", "ns"]:
        e = ent.assign(ts=pd.Series(ent["ts"].to_numpy().astype(f"datetime64[{eunit}]")))
        vec = boff.FeatureVector("v", ["g.f32", "g.f64"])

        def query():
            try:
                return tensors_of(boff.get_offline_tensors(vec, e, "ts"))
            except LoweringError as err:
                return ("refused", str(err))

        dev, host = run_both(lambda d: boff.register_offline_frame(fs, to_device(frame, ts="ts") if d else frame), query)
        if isinstance(host, tuple):
            assert dev == host and boff._UNIT_NS[eunit] > f
        else:
            assert_same_tensors(dev, host)


def test_nat_in_set_timestamps_is_refused_on_the_right_side():
    frame = make_frame(300, seed=5, nat_rows=4, extra=False)
    fs = fset("n")
    ent = frame[["id"]].assign(ts=pd.Timestamp("2000-01-01")).iloc[:50]
    for src in (to_device(frame, ts="ts"), frame):
        assert boff.register_offline_frame(fs, src).has_nat
        with pytest.raises(ValueError, match="null values on right side"):
            boff.get_offline_tensors(boff.FeatureVector("v", ["n.f32"]), ent, "ts")


@pytest.mark.parametrize("selected,ok", [("f32", True), ("f64", True), ("i8", True), ("i16", True), ("i32", True), ("u8", True),
                                         ("u16", True), ("flag", True), ("when", True), ("u32", False), ("i64", False)])
def test_feature_dtypes_join_alike_and_wide_ints_are_refused(selected, ok):
    frame = make_frame(2000, seed=6, n_keys=150)
    ent = frame[["id", "ts"]].sample(700, random_state=1).reset_index(drop=True)
    ent["ts"] = ent["ts"] + pd.Timedelta(1, "s")
    vec = boff.FeatureVector("v", [f"s.{selected}"])

    def query():
        try:
            return boff.get_offline_features(vec, ent, "ts").to_dataframe()
        except LoweringError as err:
            return str(err)

    dev, host = run_both(lambda d: boff.register_offline_frame(fset("s"), to_device(frame, ts="ts") if d else frame), query)
    if ok:
        assert_same_frames(dev, host)
    else:
        assert dev == host and "has dtype" in dev


# ---- queries ------------------------------------------------------------------------------------------------------------
def three_sets(n=6000, seed=7):
    rng = np.random.default_rng(seed)
    tx = make_frame(n, seed=seed, n_keys=n // 4).drop(columns=["when", "u32", "i64"])  # the columns a matrix cannot hold
    ev = make_frame(n // 2, seed=seed + 1, n_keys=n // 4, extra=False).rename(columns={"f32": "e32", "f64": "e64"})
    lab = make_frame(n // 3, seed=seed + 2, n_keys=n // 4, extra=False)[["id", "ts", "f32"]].rename(columns={"f32": "label"})
    prof = pd.DataFrame({"id": np.arange(n // 4, dtype=np.int64), "age": rng.integers(18, 90, n // 4).astype(np.int16),
                         "score": rng.normal(size=n // 4).astype(np.float32)})
    return {"tx": (tx, fset("tx")), "ev": (ev, fset("ev")), "lab": (lab, fset("lab")), "prof": (prof, fset("prof", ts=None))}


def register_all(sets, device):
    for name, (frame, fs) in sets.items():
        boff.register_offline_frame(fs, to_device(frame, ts=fs.timestamp_key) if device else frame)


VECTORS = [
    ("spine star, label on a set", ["tx.*", "ev.e32", "prof.score"], "lab.label"),
    ("spine features, label on the spine", ["tx.f32", "tx.i8", "tx.flag", "ev.*"], "tx.f64"),
    ("exact-key set and aliases", ["tx.u16 as u", "prof.age", "prof.score as s"], None),
]


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("label,features,label_feature", VECTORS)
def test_entity_less_tensors_and_frames_with_a_device_spine(label, features, label_feature, dtype, no_host_copies):
    sets = three_sets()
    vec = boff.FeatureVector("v", features, label_feature=label_feature)
    register_all(sets, True)
    others = {f.split(".")[0] for f in features + ([label_feature] if label_feature else [])} - {"tx"}
    asof = any(boff._OFFLINE[name].timestamp_key for name in others)
    with no_host_copies:
        before = nat.launch_count()
        t = boff.get_offline_tensors(vec, dtype=dtype)
        assert nat.launch_count() - before == (1 + SORT_LAUNCHES if asof else 0) + max(1, len(others)) + 3
        assert t.stats["h2d_ms"] == 0
    dev = tensors_of(t)
    with no_host_copies:
        t_idx = boff.get_offline_tensors(vec, dtype=dtype, with_indexes=True)
    dev_t_idx = tensors_of(t_idx)
    dev_frame = boff.get_offline_features(vec).to_dataframe()
    dev_idx = boff.get_offline_features(vec, with_indexes=True).to_dataframe()
    register_all(sets, False)
    assert_same_tensors(dev, tensors_of(boff.get_offline_tensors(vec, dtype=dtype)))
    assert_same_tensors(dev_t_idx, tensors_of(boff.get_offline_tensors(vec, dtype=dtype, with_indexes=True)))
    assert_same_frames(dev_frame, boff.get_offline_features(vec).to_dataframe())
    assert_same_frames(dev_idx, boff.get_offline_features(vec, with_indexes=True).to_dataframe())


@pytest.mark.parametrize("n", [1, 255, 256, 257, (2 << 20) + 3])
@pytest.mark.parametrize("device_sets", [True, False])
def test_cuda_entity_rows_equal_the_pandas_entity_frame(n, device_sets, no_host_copies):
    sets = three_sets(n=max(4 * n // 3, 600) if n < 1000 else 1 << 20)
    register_all(sets, device_sets)
    rng = np.random.default_rng(n)
    tx = sets["tx"][0]
    ent = pd.DataFrame({"id": tx["id"].to_numpy()[rng.integers(0, len(tx), n)],
                        "ts": (tx["ts"].to_numpy()[rng.integers(0, len(tx), n)] + np.timedelta64(1, "s")),
                        "w": rng.normal(size=n).astype(np.float32)})
    for features, label_feature in (([f for f in VECTORS[0][1] if f != "tx.*"] + ["tx.f32", "tx.i16"], "lab.label"),
                                    (["tx.*", "prof.age"], None)):
        vec = boff.FeatureVector("v", features, label_feature=label_feature)
        for dtype in ("float32", "float64"):
            cuda = to_device(ent, ts="ts")
            with no_host_copies:
                before = nat.launch_count()
                t = boff.get_offline_tensors(vec, cuda, "ts", dtype=dtype)
                sets_used = {f.split(".")[0] for f in features + ([label_feature] if label_feature else [])}
                assert nat.launch_count() - before == 1 + 1 + SORT_LAUNCHES + len(sets_used) + 3
                assert t.stats["h2d_ms"] == 0
            assert_same_tensors(tensors_of(t), tensors_of(boff.get_offline_tensors(vec, ent, "ts", dtype=dtype)))
            batch = columnar.DeviceColumnBatch({"ts": cuda["ts"], "w": cuda["w"]}, n, index={"id": cuda["id"]})
            assert_same_tensors(tensors_of(boff.get_offline_tensors(vec, batch, "ts", dtype=dtype)), tensors_of(t))
            assert_same_tensors(tensors_of(boff.get_offline_tensors(vec, cuda, "ts", dtype=dtype, with_indexes=True)),
                                tensors_of(boff.get_offline_tensors(vec, ent, "ts", dtype=dtype, with_indexes=True)))


def test_exact_key_sets_with_several_rows_per_key_are_refused_alike():
    frame = make_frame(300, seed=8, n_keys=30, extra=False).drop(columns=["ts"])
    fs = fset("x", ts=None)
    ent = pd.DataFrame({"id": np.arange(10, dtype=np.int64)})
    for src in (to_device(frame), frame):
        boff.register_offline_frame(fs, src)
        with pytest.raises(LoweringError, match="several rows per key"):
            boff.get_offline_tensors(boff.FeatureVector("v", ["x.f32"]), ent)
    with pytest.raises(LoweringError, match="several rows per key"):
        boff.get_offline_tensors(boff.FeatureVector("v", ["x.f32"]), to_device(ent))


def test_cuda_entity_rows_with_nat_are_refused_on_the_left_side():
    frame = make_frame(300, seed=9, extra=False)
    boff.register_offline_frame(fset("s"), to_device(frame, ts="ts"))
    ent = frame[["id", "ts"]].iloc[:20].copy()
    ent.loc[5, "ts"] = pd.NaT
    for rows in (ent, to_device(ent, ts="ts")):
        with pytest.raises(ValueError, match="null values on left side"):
            boff.get_offline_tensors(boff.FeatureVector("v", ["s.f32"]), rows, "ts")


def test_key_kind_mismatch_is_refused_alike():
    frame = make_frame(300, seed=10, extra=False)
    boff.register_offline_frame(fset("s"), to_device(frame, ts="ts"))
    ent = pd.DataFrame({"id": np.arange(5, dtype=np.float32), "ts": frame["ts"].iloc[:5].to_numpy()})
    msgs = []
    for rows in (ent, to_device(ent, ts="ts")):
        with pytest.raises(LoweringError) as err:
            boff.get_offline_tensors(boff.FeatureVector("v", ["s.f32"]), rows, "ts")
        msgs.append(str(err.value))
    assert msgs[0] == msgs[1] and "are not lowered" in msgs[0]


# ---- the timestamp profile ---------------------------------------------------------------------------------------------
def profile(values):
    a = np.asarray(values, dtype=np.int64)
    d = torch.from_numpy(a).cuda()
    counts = np.full(4, -1, dtype=np.int64)
    before = nat.launch_count()
    nat.check(nat.load().b2s_ts_profile_device(d.data_ptr() if len(a) else None, len(a), nat._p(counts, C.c_int64), None))
    assert nat.launch_count() - before == (1 if len(a) else 0)
    return counts.tolist()


def numpy_profile(a):
    a = np.asarray(a, dtype=np.int64)
    real = a[a != I64_MIN]
    return [int((a == I64_MIN).sum())] + [int((real % f != 0).sum()) for f in (10**3, 10**6, 10**9)]


@pytest.mark.parametrize("values", [
    [], [I64_MIN] * 5, [I64_MAX, I64_MIN + 1, 0],
    [u + d for u in (10**3, 10**6, 10**9) for d in (-1, 0, 1)],
    [-u + d for u in (10**3, 10**6, 10**9) for d in (-1, 0, 1)],
    [-(10**18), -(10**18) + 1, -999, -1000, -10**9 * 7, I64_MIN, 5 * 10**8],
])
def test_ts_profile_counts_equal_numpy(values):
    assert profile(values) == numpy_profile(values)


def test_ts_profile_over_many_blocks():
    rng = np.random.default_rng(11)
    a = rng.integers(-10**15, 10**15, (1 << 21) + 5) // 10**3 * 10**3
    a[rng.random(len(a)) < 0.01] = I64_MIN
    a[::7] = a[::7] // 10**9 * 10**9
    assert profile(a) == numpy_profile(a)


# ---- streams, lifetime, ownership ---------------------------------------------------------------------------------------
def test_columns_written_on_a_side_stream_just_before_the_calls():
    n = 1 << 20
    frame = make_frame(n, seed=12, n_keys=1 << 16, extra=False)
    want_state = state(boff.register_offline_frame(fset("s"), frame))
    vec = boff.FeatureVector("v", ["s.f32", "s.f64"])
    want = tensors_of(boff.get_offline_tensors(vec))
    cols = {c: torch.empty(n, dtype=torch.float32 if c == "f32" else torch.float64 if c == "f64" else torch.int64, device="cuda")
            for c in frame.columns}
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    host = to_device(frame, ts="ts")
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # keep the side stream busy well past the call's start
        for c in cols:
            cols[c].copy_(host[c])
        assert state(boff.register_offline_frame(fset("s"), cols)) == want_state
        torch.cuda._sleep(50_000_000)
        cols["f32"].mul_(2.0)
        t = boff.get_offline_tensors(vec)
    got = tensors_of(t)
    want["features"][:, 0] *= 2.0
    # the GPU's multiply gives NaN its canonical bits: equal values, NaN where NaN
    np.testing.assert_array_equal(got["features"], want["features"])
    np.testing.assert_array_equal(got["order"], want["order"])
    assert got["columns"] == want["columns"]


def test_close_and_reregistration_release_everything():
    frame = make_frame(5000, seed=13)
    cols = to_device(frame, ts="ts")
    torch.cuda.synchronize()
    gc.collect()
    before = nat.darray_live()
    src = boff.register_offline_frame(fset("s"), cols)
    assert nat.darray_live() == before + 1  # the encoded keys
    boff.register_offline_frame(fset("s"), cols)
    assert nat.darray_live() == before + 1
    boff._OFFLINE.pop("s").close()
    del src
    gc.collect()
    assert nat.darray_live() == before


def test_overwriting_the_entity_tensor_after_registration_changes_nothing():
    frame = make_frame(4000, seed=14, n_keys=300, extra=False)
    cols = to_device(frame, ts="ts")
    boff.register_offline_frame(fset("s"), cols)
    ent = frame[["id", "ts"]].iloc[::5].reset_index(drop=True)
    ent["ts"] = ent["ts"] + pd.Timedelta(1, "s")
    vec = boff.FeatureVector("v", ["s.f32", "s.f64"])
    first = tensors_of(boff.get_offline_tensors(vec, to_device(ent, ts="ts"), "ts"))
    spine = tensors_of(boff.get_offline_tensors(vec))
    cols["id"].fill_(-7)
    torch.cuda.synchronize()
    assert_same_tensors(tensors_of(boff.get_offline_tensors(vec, to_device(ent, ts="ts"), "ts")), first)
    assert_same_tensors(tensors_of(boff.get_offline_tensors(vec)), spine)
    # the spine's timestamps are read, and checked, where they are: NaT written into them later is refused by a query
    # that joins another set as-of on them
    boff.register_offline_frame(fset("o"), to_device(make_frame(500, seed=15, n_keys=300, extra=False), ts="ts"))
    both = boff.FeatureVector("v", ["s.f32", "o.f64"])
    boff.get_offline_tensors(both)
    cols["ts"][7] = I64_MIN
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="null values on left side"):
        boff.get_offline_tensors(both)


# ---- C-ABI refusals -----------------------------------------------------------------------------------------------------
def test_new_entry_points_refuse_bad_arguments_without_a_launch():
    lib = nat.load()
    n = 64
    d = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d32 = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
    host = np.zeros(n, dtype=np.int64)
    p, hp = d.data_ptr(), host.ctypes.data
    h = C.c_void_p()
    w8 = np.array([8], dtype=np.int32)
    w4 = np.array([4], dtype=np.int32)
    before = nat.launch_count()

    def index(keys, ts, rows, cols, widths):
        ptrs = (C.c_void_p * max(len(cols), 1))(*cols)
        return lib.b2s_pit_index_create_device(keys, ts, rows, ptrs, nat._p(widths, C.c_int32), len(cols), C.byref(h))

    bad = [index(hp, p, n, [], w8), index(p, hp, n, [], w8), index(p + 4, p, n, [], w8), index(p, p + 4, n, [], w8),
           index(p, p, n, [hp], w8), index(p, p, n, [d32.data_ptr() + 2], w4), index(p, p, 0, [], w8),
           index(None, p, n, [], w8), index(p, p, n, [p], np.array([2], dtype=np.int32))]
    assert bad == [-1] * len(bad)  # B2S_ERR_INVALID
    assert nat.launch_count() == before
    counts = np.zeros(4, dtype=np.int64)
    bad += [lib.b2s_ts_profile_device(hp, n, nat._p(counts, C.c_int64), None),
            lib.b2s_ts_profile_device(p + 4, n, nat._p(counts, C.c_int64), None),
            lib.b2s_ts_profile_device(p, n, None, None), lib.b2s_ts_profile_device(None, n, nat._p(counts, C.c_int64), None),
            lib.b2s_ts_profile_device(p, -1, nat._p(counts, C.c_int64), None)]
    assert bad == [-1] * len(bad)
    assert nat.launch_count() == before
    # the pack: a real index, then host and misaligned inputs
    ix = boff.PitIndex(np.arange(n, dtype=np.int64), np.zeros(n, np.int64), [np.zeros(n, np.float32)])
    before = nat.launch_count()

    def pack(ts, keys, col):
        outs = (nat.PitOut * 1)(nat.PitOut(0, 4, 0, None))
        sets = (nat.PitSet * 1)(nat.PitSet(ix._h, keys, 1 if ts else 0, 1, outs, None, None))
        cols = (nat.PitCol * 1)(nat.PitCol(col, None, 8))
        feats = (nat.PitFeat * 1)(nat.PitFeat(0, 0, 4, nat.PIT_FEAT_FLOAT))
        out = nat.PitTensors()
        return lib.b2s_pit_train_pack_device(ts, n, sets, 1, cols, 1, None, feats, 1, None, 4, C.byref(out), None, None)

    bad = [pack(hp, p, p), pack(p, hp, p), pack(p, p, hp), pack(p + 4, p, p), pack(p, p + 4, p), pack(p, p, p + 4)]
    assert bad == [-1] * len(bad)
    assert nat.launch_count() == before
    ix.close()
