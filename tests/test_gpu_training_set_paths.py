"""Training sets on every path of the b2s_pit keep, scan and scatter kernels and of their host staging, against the numpy
reference `train` of tests/pit_reference.py.  Needs an H100: `-m gpu`.

What can serve a training set (csrc/b2s_pit.cu, `b2s_pit_train_*`):
  * the sort and join launches of tests/test_gpu_pit_paths.py, writing every output at full length into scratch;
  * keep_kernel: one row per thread over 1 024-row tiles; a row is kept when every exact-key set matched it and its label
    is present (its set matched; a NAN label is no NaN of its 4- or 8-byte float, a NAT label not INT64_MIN); per set, a warp
    ballot counts the misses among the rows every earlier exact-key set kept, into 64 shared counters flushed once per
    block; each tile's kept rows are counted;
  * scan_tiles_kernel: one block turns the tile counts into exclusive offsets, each of its 1 024 threads owning
    ceil(tiles / 1 024) of them, and writes the total;
  * scatter_kernel: a kept row goes to its tile's offset plus its rank in the tile (the warp counts scanned, then its
    lane's rank in the warp's ballot); 64 arrays per launch;
  * b2s_pit_train_host, which copies back only rows [0, kept) in 1 Mi-row ranges, and b2s_pit_train_device on the library
    stream or a caller's, which overwrites the miss counters and kept.

Every comparison is exact: outputs, timestamps, found flags, the order and the entity columns bit for bit, kept and the misses
as integers.  The label patterns run without timestamps or sets, so the order is the identity and names each kept row, and
each tile's scan offset is read back from it on its own.  Every case asserts its launches, as the library's launch count and
(host calls) as `stats["kernels"]`: 24 for the sort when there are timestamps, max(1, n_sets, ceil(n_cols / 64)) for the
join, 2 for keep and scan and ceil(arrays / 64) for the scatter, where arrays counts each set's outputs, ts_out and found,
the entity columns and the order; none for n = 0.  The last cases go through `get_offline_features`, where the device's
miss counts decide the reference's dtypes.
"""

import ctypes as C
import math

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import ingest as bingest  # noqa: E402
from mlrun_b200.feature_store import offline as boff  # noqa: E402
from tests import pit_reference as ref  # noqa: E402
from tests.golden import diff_training_set  # noqa: E402

RANGE = 1 << 20   # rows per copy-back range of b2s_pit_train_host
TILE = ref.TILE   # rows per block of the keep and scatter kernels
SENT = 0xA5       # byte that fills every output before a run; rows from kept on must keep it
GARBAGE = 0x5A5A5A5A5A5A5A5A


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


# ---------------------------------------------------------------------------------------------------------- helpers
def train_launches(has_ts, n, n_sets, n_cols, arrays):
    if n == 0:
        return 0
    return (24 if has_ts else 0) + max(1, n_sets, math.ceil(n_cols / 64)) + 2 + math.ceil(arrays / 64)


def n_arrays(sets, n_cols, ts_out=True, order=True):
    """the arrays the scatter moves: each set's outputs, ts_out (when asked for) and found, the entity columns, the order"""
    return sum(len(outs) + int(ts_out) + 1 for *_, outs in sets) + n_cols + int(order)


def rows(ts, sets, cols):
    return len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1])


def indexes(sets):
    """one device index per Table of `sets` -> [(index, keys, asof, outs)]"""
    ixs = {}
    for t, *_ in sets:
        if id(t) not in ixs:
            ixs[id(t)] = boff.PitIndex(t.keys, t.ts, t.cols)
    return [(ixs[id(t)], k, a, o) for t, k, a, o in sets]


def run(ts, sets, cols, label):
    """the host training set of (ts, sets over Tables, cols, label) equals `ref.train`, with the launches it should make
    -> the result, with pit_train's stats"""
    n = rows(ts, sets, cols)
    on_device = indexes(sets)
    before = nat.launch_count()
    got = boff.pit_train(ts, on_device, cols, label, with_stats=True)
    want = train_launches(ts is not None, n, len(sets), len(cols), n_arrays(sets, len(cols)))
    assert nat.launch_count() - before == want
    assert got[4]["kernels"] == want and got[4]["rows"] == n
    ref.assert_same_train(got, ref.train(ts, sets, cols, label))
    return got


def sentinel(n, dtype):
    return np.full(n * np.dtype(dtype).itemsize, SENT, np.uint8).view(dtype)


# --------------------------------------------------------------------------------------------------------- keep rule
@pytest.mark.parametrize("kinds", ref.SET_ORDERS, ids=lambda k: f"{len(k)}:{k[:7] or '-'}")
def test_set_orders(kinds):
    """0 to 64 sets in orders of as-of (A) and exact-key (E) joins: keep is the AND of the exact-key sets' found flags, and
    each set's misses are counted among the rows the exact-key sets before it kept"""
    got = run(*ref.train_workload(f"order_{kinds or '-'}"))
    assert len(got[3]) == len(kinds)


@pytest.mark.parametrize("case", ref.LABEL_PLACES)
def test_label_places(case):
    """the label on an as-of or an exact-key set, on a 4- or 8-byte output, with miss bits that are a NaN or are not (then
    only the set's found flag drops a missed row), a FOUND label whose values are NaN, and entity columns of each kind"""
    ts, sets, cols, label = ref.label_place(case, seed=ref.LABEL_PLACES.index(case))
    got = run(ts, sets, cols, label)
    if label[2] == ref.LABEL_FOUND and label[0] >= 0:
        assert np.isnan(got[1][label[0]][0][label[1]]).any()  # NaN labels kept


@pytest.mark.parametrize("case", ref.EDGE_CASES)
def test_label_value_edges(case):
    """every NaN (quiet, signalling, negative, with payload) is dropped; -0.0, infinities, the smallest denormal, the float
    maxima and INT64_MIN + 1 are kept; a FOUND label drops no value"""
    dtype, place, *found = case.split("_")
    ts, sets, cols, label = ref.label_edges(dtype, place, ref.LABEL_FOUND if found else None, seed=ref.EDGE_CASES.index(case))
    got = run(ts, sets, cols, label)
    values = got[1][label[0]][0][label[1]] if label[0] >= 0 else got[2][label[1]]
    edges = {"float32": ref.F32_EDGES, "float64": ref.F64_EDGES, "int64": ref.I64_EDGES}[dtype]
    uint = np.uint32 if edges.dtype.itemsize == 4 else np.uint64
    kept = edges[ref.label_present(edges, label[2])]
    assert set(values.view(uint).tolist()) >= set(kept.view(uint).tolist())


# ------------------------------------------------------------------------------------------------- tiles and the scan
SMALL_N = [1, 31, 32, 33, 1023, 1024, 1025, 2047, 3 * TILE + 5]
LARGE_N = [RANGE - 1,          # 1 024 tiles: one per scan thread
           RANGE,
           RANGE + 1,          # 1 025 tiles: two per thread, threads past 512 idle
           2048 * TILE,        # two per thread, every thread busy
           2048 * TILE + 1]    # 2 049 tiles: three per thread, threads past 682 idle
LARGE_PATTERNS = ["all", "none", "random_50", "tile_in_7"]
TILE_CASES = [(n, p) for n in SMALL_N for p in ref.LABEL_PATTERNS] + [(n, p) for n in LARGE_N for p in LARGE_PATTERNS]


@pytest.mark.parametrize("n, pattern", TILE_CASES)
def test_tiles_and_scan_offsets(n, pattern):
    seed = ref.LABEL_PATTERNS.index(pattern)
    got = run(*ref.label_column(n, pattern, np.float32 if n % 2 == 0 else np.float64, seed=seed))
    keep = ref.keep_pattern(n, pattern, np.random.default_rng(seed))
    n_tiles = math.ceil(n / TILE)
    counts = np.bincount(np.flatnonzero(keep) // TILE, minlength=n_tiles)
    # each tile's offset on its own: where its first row lands (the order is the identity, so it names the rows)
    np.testing.assert_array_equal(np.searchsorted(got[0], np.arange(n_tiles) * TILE), np.cumsum(counts) - counts)
    assert got[4]["kept"] == int(keep.sum())


# ---------------------------------------------------------------------------------------------------- scatter launches
def scatter_case(arrays, n=5000):
    """-> (ts, sets, cols, label) whose training set moves `arrays` arrays: one as-of set over a table of 256 columns (its
    row number, then 4- and 8-byte columns alternating) with the first arrays - 7 of them as outputs, its ts_out and found,
    entity columns of 1, 2, 4 and 8 bytes and the order; the label is the set's last output, a float with 30 % NaNs"""
    rng = np.random.default_rng(arrays)
    universe = np.arange(300, dtype=np.int64) * 11
    keys, ts = ref.query(rng, universe, n)
    t = ref.wide_table(rng, universe[rng.integers(0, 300, size=2000)], rng.integers(-20, 20, size=2000) * 10**9, [4, 8] * 127 + [4])
    n_out = arrays - 7
    col = t.cols[n_out - 1]
    nans = ref.NAN32_BITS if col.dtype.itemsize == 4 else ref.NAN64_BITS
    hit = np.flatnonzero(rng.random(len(col)) < 0.3)
    col.view(nans.dtype)[hit] = nans[hit % 4]
    cols = [ref.random_bits(rng, n, dt) for dt in (np.uint8, np.int16, np.float32, np.int64)]
    return ts, [(t, keys, 1, ref.all_outs(t)[:n_out])], cols, (0, n_out - 1, ref.LABEL_NAN)


@pytest.mark.parametrize("arrays", [63, 64, 65, 128, 129, 263])
def test_scatter_launches(arrays):
    ts, sets, cols, label = scatter_case(arrays)
    assert n_arrays(sets, len(cols)) == arrays
    if arrays == 263:
        assert len(sets[0][3]) == 256 and label[1] == 255
    got = run(ts, sets, cols, label)
    assert got[4]["kernels"] == 24 + 1 + 2 + math.ceil(arrays / 64)
    assert 0 < got[4]["kept"] < len(ts)


# -------------------------------------------------------------------------------------------------- host copy-back
@pytest.mark.parametrize("kept", [0, 1, RANGE - 1, RANGE, RANGE + 1, 2 * RANGE + 3])
def test_host_copy_back_stops_at_kept(kept):
    """b2s_pit_train_host over host arrays filled with a sentinel: rows [0, kept) come back, in 1 Mi-row ranges, and
    every element from kept on still holds the sentinel"""
    n = 2 * RANGE + 1000
    rng = np.random.default_rng(kept)
    keep = np.zeros(n, bool)
    keep[rng.choice(n, kept, replace=False)] = True
    universe = np.arange(1000, dtype=np.int64)
    t = ref.Table(universe, np.zeros(1000, np.int64), [rng.normal(size=1000).astype(np.float32), rng.normal(size=1000)])
    keys = universe[rng.integers(0, 1000, size=n)]  # every key known: the exact-key set keeps every row
    outs = ref.all_outs(t)
    cols = [np.where(keep, rng.normal(size=n), np.nan)] + ref.entity_cols(rng, n, 4)
    label = (-1, 0, ref.LABEL_NAN)
    want = ref.train(None, [(t, keys, 0, outs)], cols, label)

    ix = boff.PitIndex(t.keys, t.ts, t.cols)
    arrays = [sentinel(n, dt) for _w, dt, _m in outs]
    ts_out, found, order = sentinel(n, np.int64), sentinel(n, np.uint8), sentinel(n, np.int64)
    dsts = [sentinel(n, c.dtype) for c in cols]
    descs = (nat.PitOut * len(outs))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, a.ctypes.data) for (w, dt, m), a in zip(outs, arrays)])
    c_s = (nat.PitSet * 1)(nat.PitSet(ix._h, keys.ctypes.data, 0, len(outs), descs, ts_out.ctypes.data, found.ctypes.data))
    cc = (nat.PitCol * len(cols))(*[nat.PitCol(c.ctypes.data, d.ctypes.data, c.dtype.itemsize) for c, d in zip(cols, dsts)])
    miss = np.full(2, GARBAGE, np.uint64)
    k, phase, stats = C.c_int64(-1), (C.c_float * 3)(-1.0, -1.0, -1.0), nat.Stats()
    before = nat.launch_count()
    nat.check(nat.load().b2s_pit_train_host(None, n, c_s, 1, cc, len(cols), C.byref(nat.PitLabel(*label)), order.ctypes.data,
                                            miss.ctypes.data, C.byref(k), phase, C.byref(stats)))
    launches = train_launches(False, n, 1, len(cols), n_arrays([(t, keys, 0, outs)], len(cols)))
    assert nat.launch_count() - before == stats.kernels == launches
    assert stats.rows == n and k.value == kept
    assert all(math.isfinite(p) and p >= 0 for p in phase)
    assert miss[1] == np.uint64(GARBAGE)  # one set: one counter written
    got = (order[:kept], [([a[:kept] for a in arrays], ts_out[:kept], found[:kept].view(bool))], [d[:kept] for d in dsts], miss[:1])
    ref.assert_same_train(got, want)
    for a in [order, ts_out, found, *arrays, *dsts]:
        assert (ref.bits(a)[kept * a.dtype.itemsize:] == SENT).all(), "an element past kept was written"


# ------------------------------------------------------------------------------------------------------ device path
def _device_train(ts, sets, cols, label, stream, with_order=True, with_ts_out=True):
    """b2s_pit_train_device over sentinel-filled buffers of n + 1 elements, with miss and kept preloaded with garbage ->
    (order, [(outputs, ts_out, found)], cols, miss) cut to kept (None for an array not asked for), after checking that
    every array holds its sentinel from kept on, the counter past the sets kept its garbage, and the launches"""
    n = rows(ts, sets, cols)
    bufs = []

    def dev(arr=None, elem=None):
        b = nat.DeviceBuffer((n + 1) * elem).upload(np.full((n + 1) * elem, SENT, np.uint8)) if arr is None else \
            nat.DeviceBuffer(max(np.asarray(arr).nbytes, 8)).upload(arr)
        bufs.append(b)
        return b

    d_ts = dev(np.ascontiguousarray(ts, np.int64)) if ts is not None else None
    descs, layout = [], []
    for ix, keys, asof, outs in sets:
        d_keys = dev(np.ascontiguousarray(keys, np.int64))
        d_outs = [dev(elem=np.dtype(dt).itemsize) for _w, dt, _m in outs]
        d_tsout, d_found = (dev(elem=8) if with_ts_out else None), dev(elem=1)
        descs.append((d_keys, asof, (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, b.ptr)
                                                                         for (w, dt, m), b in zip(outs, d_outs)])))
        layout.append((ix, d_outs, d_tsout, d_found, [dt for _w, dt, _m in outs]))
    c_s = (nat.PitSet * max(len(sets), 1))()
    for s, ((d_keys, asof, o), (ix, d_outs, d_tsout, d_found, _dts)) in enumerate(zip(descs, layout)):
        c_s[s] = nat.PitSet(ix._h, d_keys.ptr, int(asof), len(d_outs), o, None if d_tsout is None else d_tsout.ptr, d_found.ptr)
    d_cols = [(dev(c), dev(elem=c.dtype.itemsize), c.dtype) for c in cols]
    cc = (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(s.ptr, d.ptr, dt.itemsize) for s, d, dt in d_cols])
    d_order = dev(elem=8) if with_order else None
    # garbage in every counter: b2s_pit_train_device overwrites miss and kept (b2s_pit_join_device adds to its miss)
    d_miss = dev(np.full(len(sets) + 1, GARBAGE, np.uint64))
    d_kept = dev(np.full(2, GARBAGE, np.uint64))
    before = nat.launch_count()
    nat.check(nat.load().b2s_pit_train_device(None if d_ts is None else d_ts.ptr, n, c_s, len(sets), cc, len(cols),
                                              None if label is None else C.byref(nat.PitLabel(*label)),
                                              None if d_order is None else d_order.ptr, d_miss.ptr, d_kept.ptr,
                                              None if stream is None else stream.cuda_stream))
    arrays = n_arrays(sets, len(cols), ts_out=with_ts_out, order=with_order)
    assert nat.launch_count() - before == train_launches(ts is not None, n, len(sets), len(cols), arrays)
    if stream is not None:
        stream.synchronize()
    nat.check(nat.load().b2s_device_sync())
    kept_pair = d_kept.download(np.uint64, 2)
    assert kept_pair[1] == np.uint64(GARBAGE)
    kept = int(kept_pair[0])
    assert 0 <= kept <= n

    def back(b, dtype):
        if b is None:
            return None
        size = np.dtype(dtype).itemsize
        raw = b.download(np.uint8, (n + 1) * size)
        assert (raw[kept * size:] == SENT).all(), "an element past kept was written"
        return raw[: kept * size].view(dtype)

    joined = [([back(b, dt) for b, dt in zip(d_outs, dts)], back(d_tsout, np.int64), back(d_found, np.uint8).astype(bool))
              for _ix, d_outs, d_tsout, d_found, dts in layout]
    miss = d_miss.download(np.uint64, len(sets) + 1)
    assert miss[-1] == np.uint64(GARBAGE)
    return back(d_order, np.int64), joined, [back(d, dt) for _s, d, dt in d_cols], miss[:-1]


def _with_missing_from(got, want):
    """`got` with the arrays the call was not asked for (None) taken from `want`, so the rest compare bit for bit"""
    order = want[0] if got[0] is None else got[0]
    joined = [(a, w[1] if t is None else t, f) for (a, t, f), w in zip(got[1], want[1])]
    return order, joined, got[2], got[3]


@pytest.mark.parametrize("nulls", ["none", "order_and_ts_out"])
@pytest.mark.parametrize("stream", ["library", "caller"])
@pytest.mark.parametrize("with_ts", [True, False])
def test_device_path_equals_the_host_run(with_ts, stream, nulls):
    kinds = "EAE" if with_ts else "EEE"
    ts, sets, cols = ref.ordered_sets(kinds, n=6000, seed=len(kinds) + int(with_ts))
    cols = cols + ref.entity_cols(np.random.default_rng(1), 6000, 66)  # 68 entity columns: two join launches
    label = (1, 2, ref.LABEL_NAN)
    host = run(ts, sets, cols, label)
    strm = None
    if stream == "caller":
        import torch

        strm = torch.cuda.Stream(device=0)
    null = nulls == "order_and_ts_out"
    got = _device_train(ts, indexes(sets), cols, label, strm, with_order=not null, with_ts_out=not null)
    assert (got[0] is None) == null and all((t is None) == null for _a, t, _f in got[1])
    ref.assert_same_train(_with_missing_from(got, host), host[:4])
    ref.assert_same_train(_with_missing_from(got, host), ref.train(ts, sets, cols, label))


def test_device_path_with_no_rows_on_a_callers_stream():
    """n = 0 launches nothing and still writes kept = 0 and zero misses over the garbage, on the caller's stream"""
    import torch

    ts, sets, cols = ref.ordered_sets("EAE", n=16, seed=2)
    on_device = indexes(sets)
    strm = torch.cuda.Stream(device=0)
    d_ts = nat.DeviceBuffer(8).upload(np.zeros(1, np.int64))
    d_miss = nat.DeviceBuffer(32).upload(np.full(4, GARBAGE, np.uint64))
    d_kept = nat.DeviceBuffer(8).upload(np.full(1, GARBAGE, np.uint64))
    outs = (nat.PitOut * 1)(nat.PitOut(0, 4, 0, None))  # room for no row: nothing may be written
    c_s = (nat.PitSet * 3)(*[nat.PitSet(ix._h, None, int(a), 1, outs, None, None) for ix, _k, a, _o in on_device])
    before = nat.launch_count()
    nat.check(nat.load().b2s_pit_train_device(d_ts.ptr, 0, c_s, 3, None, 0, C.byref(nat.PitLabel(1, 0, ref.LABEL_FOUND)), None,
                                              d_miss.ptr, d_kept.ptr, strm.cuda_stream))
    assert nat.launch_count() == before
    strm.synchronize()
    assert d_kept.download(np.int64, 1)[0] == 0
    assert d_miss.download(np.uint64, 4).tolist() == [0, 0, 0, GARBAGE]


# ---------------------------------------------------------------------------------------------- through the product
def _frames(cards_has_7, label_nan_on_7):
    """20 cards; an as-of set `txn` with an int32 feature and no row of card 7, an exact-key set `cards` (with or without
    card 7), and a `labels` set at the entity rows' times (NaN on card 7's rows or nowhere); entity rows after every
    txn row"""
    rng = np.random.default_rng(3)
    n, base = 400, 10**18
    card = rng.integers(0, 20, size=n)
    card[:25] = 7
    t = pd.to_datetime(base + (rng.permutation(n) + 10**4) * 10**9)
    others = np.setdiff1d(np.arange(20), [7])
    txn = pd.DataFrame({"card": np.repeat(others, 5), "when": pd.to_datetime(base + rng.permutation(5 * len(others)) * 10**9),
                        "cnt": rng.integers(0, 100, size=5 * len(others)).astype(np.int32)})
    ids = np.arange(20) if cards_has_7 else others
    cards = pd.DataFrame({"card": ids, "tier": rng.integers(0, 4, size=len(ids)).astype(np.int32)})
    label = rng.normal(size=n)
    if label_nan_on_7:
        label[card == 7] = np.nan
    labels = pd.DataFrame({"card": card, "when": t, "label": label})
    frames = {"txn": (["card"], "when", txn), "cards": (["card"], None, cards), "labels": (["card"], "when", labels)}
    return frames, pd.DataFrame({"card": card, "t": t})


@pytest.mark.parametrize("exact_first", [True, False])
@pytest.mark.parametrize("dropped_by", ["exact_key_set", "label"])
def test_dtypes_follow_the_misses_at_each_sets_place(dropped_by, exact_first, monkeypatch):
    """`txn.cnt` misses only card 7's rows.  Removed by the exact-key set before txn joins, they never reach the merged frame
    and cnt stays int32; removed by the exact-key set after txn, or by the label's dropna (which runs after the dtypes are
    set), cnt is float64"""
    monkeypatch.setattr(boff, "_OFFLINE", {})
    frames, entity = _frames(cards_has_7=dropped_by == "label", label_nan_on_7=dropped_by == "label")
    features = ["cards.tier", "txn.cnt"] if exact_first else ["txn.cnt", "cards.tier"]
    args = dict(frames=frames, features=features, label_feature="labels.label", entity_rows=entity, entity_timestamp_column="t",
                with_indexes=False)
    for name, (entities, ts, frame) in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)
    got = boff.get_offline_features(boff.FeatureVector("v", features, label_feature="labels.label"), entity, "t").to_dataframe()
    pd.testing.assert_frame_equal(got, diff_training_set.oracle_training_set(**args), check_exact=True)
    assert got["cnt"].dtype == (np.int32 if exact_first and dropped_by == "exact_key_set" else np.float64)
    assert len(got) == int((entity["card"] != 7).sum())
