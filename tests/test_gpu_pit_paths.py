"""Point-in-time joins on every path of the b2s_pit sort, index and join kernels, against the numpy sweep of
tests/pit_reference.py.  Needs an H100: `-m gpu`.

What can serve a join (csrc/b2s_pit.{cuh,cu}):
  * the stable LSD radix sort: 8 passes of histogram, one-block scan over 256 x n_blocks counters and a `__match_any_sync`
    scatter, over tiles of 4 096 keys; the entity rows are sorted by timestamp when there are timestamps, else kept in order;
  * the index build: a sort by timestamp, a stable sort by key, the row layout of 4- and 8-byte columns, the run count and
    the slot insert (capacity 16, doubling while below twice the keys);
  * pit_join_kernel: per set, probe the key's run, binary-search it (as-of) or take its only row (exact key), gather the
    selected words, write ts_out / found when given; one set per launch, and entity columns 64 to a launch, only the first
    launch writing `order`;
  * b2s_pit_join_host, pipelined in 1 Mi-row ranges, and b2s_pit_join_device on the library stream or the caller's.

Every comparison is exact: outputs, timestamps, found flags, the order and the permuted entity columns bit for bit, misses as
integers.  Every feature set carries its input row number as column 0, so a wrong pick names the row it took.  Every case
asserts the launches it made: 53 per index build, and per join 24 for the sort when there are timestamps plus
max(1, n_sets, ceil(n_cols / 64)) per 1 Mi-row range, which b2s_pit_join_host also reports in `stats["kernels"]`.
"""

import ctypes as C
import math

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import offline as boff  # noqa: E402
from oracle import offline as oo  # noqa: E402
from tests import offline_fixtures as fx  # noqa: E402
from tests import pit_reference as ref  # noqa: E402
from tests import table_hash  # noqa: E402

RANGE = 1 << 20  # rows per range of b2s_pit_join_host
TILE = 4096      # keys per radix-sort block
INDEX_LAUNCHES = 53
INVALID = -1     # B2S_ERR_INVALID
SENT = 0xA5      # byte that fills device outputs before a run; the element past n must keep it


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


# ---------------------------------------------------------------------------------------------------------- helpers
def join_launches(has_ts, n, n_sets, n_cols):
    if n == 0:
        return 0
    return (24 if has_ts else 0) + math.ceil(n / RANGE) * max(1, n_sets, math.ceil(n_cols / 64))


def make_index(table):
    before = nat.launch_count()
    ix = boff.PitIndex(table.keys, table.ts, table.cols)
    assert nat.launch_count() - before == INDEX_LAUNCHES
    return ix


def index_info(ix):
    v = [C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32(), C.c_int64()]
    nat.check(nat.load().b2s_pit_index_info(ix._h, *[C.byref(x) for x in v]))
    return dict(zip(["n_rows", "n_keys", "longest_run", "row_words", "capacity"], [x.value for x in v]))


def run(ts, sets, cols):
    """the host join of (ts, sets over Tables, cols) equals the sweep, with the launches it should make -> the result"""
    indexes = {}
    for t, *_ in sets:
        if id(t) not in indexes:
            indexes[id(t)] = make_index(t)
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1])
    before = nat.launch_count()
    got = boff.pit_join(ts, [(indexes[id(t)], k, a, o) for t, k, a, o in sets], cols, with_stats=True)
    want = join_launches(ts is not None, n, len(sets), len(cols))
    assert nat.launch_count() - before == want
    assert got[4]["kernels"] == want and got[4]["rows"] == n
    ref.assert_same(got, ref.join(ts, sets, cols))
    return got


def c_sets(descs):
    """[(index, keys ptr, asof, [(src_word, bytes, miss, out ptr)], ts_out ptr, found ptr)] -> (PitSet array, what it points into)"""
    arr, keep = (nat.PitSet * max(len(descs), 1))(), []
    for i, (ix, kp, asof, outs, tsp, fp) in enumerate(descs):
        o = (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, b, m, p) for w, b, m, p in outs])
        keep.append(o)
        arr[i] = nat.PitSet(ix._h, kp, asof, len(outs), o, tsp, fp)
    return arr, keep


def c_cols(cols):
    """[(src ptr, dst ptr, bytes)] -> PitCol array"""
    return (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(s, d, b) for s, d, b in cols])


# ---------------------------------------------------------------------------------------------------------------- sort
SORT_SIZES = [1, 2, 31, 33, TILE - 1, TILE, TILE + 1, 3 * TILE + 1,
              4 * TILE,          # 1 024 scan counters: one per scan thread
              5 * TILE,          # 1 280 counters: the last scan threads idle
              257 * TILE + 5]    # 258 tiles over two host ranges


def sort_keys(kind, n, rng):
    return {"all_equal": np.full(n, -5, np.int64), "reversed": np.arange(n, 0, -1, dtype=np.int64) * -(10**9),
            "random": rng.integers(ref.I64_MIN, ref.I64_MAX, size=n, dtype=np.int64, endpoint=True),
            "extremes": rng.choice(ref.EXTREME_KEYS, size=n)}[kind]


@pytest.mark.parametrize("kind", ["all_equal", "reversed", "random", "extremes"])
@pytest.mark.parametrize("n", SORT_SIZES)
def test_sort_is_a_stable_argsort(n, kind):
    ts = sort_keys(kind, n, np.random.default_rng(n))
    order = run(ts, [], [])[0]
    np.testing.assert_array_equal(order, np.argsort(ts, kind="stable"))


# --------------------------------------------------------------------------------------------------------------- index
def index_case(name, rng):
    """-> (Table, query keys, query timestamps)"""
    if name == "one_key_2^20":
        m = 1 << 20
        t = ref.Table(np.full(m, 42, np.int64), rng.integers(0, m // 4, size=m))
        return t, np.r_[np.full(20000, 42), [41, 43]], rng.integers(-1, m // 4 + 1, size=20002)
    if name == "all_distinct":
        keys = rng.permutation(np.arange(-50000, 50000, dtype=np.int64) * 7919)
        t = ref.wide_table(rng, keys, rng.integers(-5, 5, size=len(keys)) * 10**9, [8])
    elif name in ("keys_8", "keys_9"):
        k = int(name[-1])
        t = ref.wide_table(rng, np.repeat(np.arange(k, dtype=np.int64) * 1000 - 3, 11), rng.integers(0, 4, size=11 * k), [4])
    elif name == "extreme_keys":
        t = ref.wide_table(rng, np.tile(ref.EXTREME_KEYS, 40), rng.integers(-3, 3, size=200) * 10**9, [8, 4])
    elif name == "wrapped_chain":
        t, qk, qt = ref.asof_edges(rng, n_keys=12)
        return t, qk, qt
    elif name == "no_columns":
        t = ref.Table(rng.integers(0, 30, size=500), rng.integers(0, 10, size=500), rowid=False)
    elif name == "interleaved_4_8":
        t = ref.wide_table(rng, rng.integers(0, 40, size=800), rng.integers(0, 10, size=800), [8, 4, 8, 4, 4, 8, 8, 4, 8])
    elif name == "columns_256":
        t = ref.wide_table(rng, rng.integers(0, 200, size=3000), rng.integers(0, 10, size=3000), [8] * 255)
    else:
        raise ValueError(name)
    known = np.unique(t.keys)
    qk = np.concatenate([known, known, rng.integers(10**15, 10**16, size=64)])
    qt = np.concatenate([np.full(len(known), ref.I64_MAX), rng.choice(np.unique(t.ts), size=len(known)), rng.integers(-10, 10, 64)])
    return t, qk, qt


INDEX_CASES = ["one_key_2^20", "all_distinct", "keys_8", "keys_9", "extreme_keys", "wrapped_chain", "no_columns", "interleaved_4_8",
               "columns_256"]


@pytest.mark.parametrize("name", INDEX_CASES)
def test_index_build(name):
    rng = np.random.default_rng(INDEX_CASES.index(name))
    t, qk, qt = index_case(name, rng)
    ix = make_index(t)
    _u, counts = np.unique(t.keys, return_counts=True)
    assert index_info(ix) == dict(n_rows=len(t.keys), n_keys=len(counts), longest_run=int(counts.max()), row_words=t.row_words,
                                  capacity=table_hash.capacity(len(counts)))
    ix.close()
    if name == "columns_256":
        assert len(t.cols) == 256 and t.row_words == 511
    if name == "interleaved_4_8":
        assert any(t.word[c] % 2 for c in range(len(t.cols)) if t.cols[c].dtype.itemsize == 8)
    run(qt, [(t, qk, 1, ref.all_outs(t))], [])


# ------------------------------------------------------------------------------------------------------ as-of edges
@pytest.mark.parametrize("dup", [2, 3, 40])
def test_asof_edges(dup):
    rng = np.random.default_rng(dup)
    t, qk, qt = ref.asof_edges(rng, dup=dup)
    got = run(qt, [(t, qk, 1, ref.all_outs(t))], ref.entity_cols(rng, len(qk), 4))
    rows, found = got[1][0][0][0], got[1][0][2]  # the row-number output and the found flags
    pairs, counts = np.unique(np.stack([t.keys, t.ts], 1), axis=0, return_counts=True)
    dup = {tuple(p) for p in pairs[counts > 1].tolist()}
    assert any((int(t.keys[r]), int(t.ts[r])) in dup for r in rows[found])  # some query landed on a duplicated (key, ts)


# -------------------------------------------------------------------------------------------------------------- sets
@pytest.mark.parametrize("n_sets", [1, 2, 3, 4, 5])
def test_sets_mixed_asof_and_exact(n_sets):
    run(*ref.mixed_sets(np.random.default_rng(n_sets), n_sets, 3000))


@pytest.mark.parametrize("n_sets", [1, 3])
def test_exact_sets_without_timestamps(n_sets):
    ts, sets, cols = ref.mixed_sets(np.random.default_rng(10 + n_sets), n_sets, 3000, with_ts=False)
    got = run(ts, sets, cols)
    np.testing.assert_array_equal(got[0], np.arange(3000))


def test_sets_with_no_output_and_with_256_outputs():
    rng = np.random.default_rng(7)
    universe = np.arange(100, dtype=np.int64) * 13
    keys, ts = ref.query(rng, universe, 4000)
    wide = ref.wide_table(rng, universe[rng.integers(0, 100, size=2000)], rng.integers(-20, 20, size=2000) * 10**9,
                          [4, 8] * 127 + [4])
    bare = ref.keyed_table(rng, universe, 500)
    assert len(ref.all_outs(wide)) == 256
    run(ts, [(bare, keys, 1, []), (wide, keys, 1, ref.all_outs(wide)), (bare, keys, 1, ref.all_outs(bare))], [])


@pytest.mark.parametrize("miss", [ref.MISS_NAN32, ref.MISS_NAN64, ref.MISS_NAT, ref.MISS_ZERO, ref.MISS_BITS])
def test_miss_bits(miss):
    rng = np.random.default_rng(3)
    e, qk, qt = ref.asof_edges(rng)
    t = ref.wide_table(rng, e.keys, e.ts, [4, 8])
    got = run(qt, [(t, qk, 1, [t.out(0, miss), (0, np.int64, miss), t.out(1, miss), t.out(2, miss)])], [])
    # (0, int64) spans the row number and the float32 after it; a miss stores all 64 bits, a 4-byte one the low 32
    outs, found = got[1][0][0], got[1][0][2]
    assert not found.all()
    assert (outs[1][~found].view(np.uint64) == np.uint64(miss)).all()
    assert (outs[0][~found].view(np.uint32) == np.uint32(miss & 0xFFFFFFFF)).all()


def test_null_found_ts_out_and_order():
    """the NULL forms of the optional outputs: set 0 without ts_out, set 1 without found, set 2 without both, and no order"""
    rng = np.random.default_rng(5)
    ts, sets, cols = ref.mixed_sets(rng, 3, 2500)
    want = ref.join(ts, sets, cols)
    n = len(ts)
    ixs = [make_index(t) for t, *_ in sets]
    keep, descs, results = [], [], []
    for s, ((t, keys, asof, outs), ix) in enumerate(zip(sets, ixs)):
        keys = np.ascontiguousarray(keys, np.int64)
        arrays = [np.empty(n, np.dtype(dt)) for _w, dt, _m in outs]
        ts_out = np.empty(n, np.int64) if s == 1 else None
        found = np.empty(n, np.uint8) if s == 0 else None
        keep += [keys, arrays, ts_out, found]
        descs.append((ix, keys.ctypes.data, int(asof), [(w, np.dtype(dt).itemsize, m, a.ctypes.data) for (w, dt, m), a in zip(outs, arrays)],
                      None if ts_out is None else ts_out.ctypes.data, None if found is None else found.ctypes.data))
        results.append((arrays, ts_out, found))
    c_s, k2 = c_sets(descs)
    dsts = [np.empty_like(c) for c in cols]
    cc = c_cols([(s.ctypes.data, d.ctypes.data, s.dtype.itemsize) for s, d in zip(cols, dsts)])
    miss, stats = np.zeros(3, np.uint64), nat.Stats()
    tsa = np.ascontiguousarray(ts, np.int64)
    before = nat.launch_count()
    nat.check(nat.load().b2s_pit_join_host(tsa.ctypes.data, n, c_s, 3, cc, len(cols), None, miss.ctypes.data, C.byref(stats)))
    assert nat.launch_count() - before == stats.kernels == join_launches(True, n, 3, len(cols))
    for s, (arrays, ts_out, found) in enumerate(results):
        w_arrays, w_ts, w_found = want[1][s]
        for g, w in zip(arrays, w_arrays):
            np.testing.assert_array_equal(ref.bits(g), ref.bits(w))
        if ts_out is not None:
            np.testing.assert_array_equal(ts_out, w_ts)
        if found is not None:
            np.testing.assert_array_equal(found.astype(bool), w_found)
    for g, w in zip(dsts, want[2]):
        np.testing.assert_array_equal(ref.bits(g), ref.bits(w))
    np.testing.assert_array_equal(miss, want[3])


# ---------------------------------------------------------------------------------------------------- entity columns
@pytest.mark.parametrize("n_sets", [0, 1, 2])
@pytest.mark.parametrize("n_cols", [0, 1, 64, 65, 130])
def test_entity_columns(n_cols, n_sets):
    rng = np.random.default_rng(n_cols * 3 + n_sets)
    n = 5000
    ts, sets, _c = ref.mixed_sets(rng, n_sets, n) if n_sets else (rng.integers(-30, 30, size=n) * 10**9, [], [])
    run(ts, sets, ref.entity_cols(rng, n, n_cols))


def test_entity_columns_without_timestamps_keep_input_order():
    rng = np.random.default_rng(9)
    got = run(None, [], ref.entity_cols(rng, 5000, 130))
    np.testing.assert_array_equal(got[0], np.arange(5000))


# ------------------------------------------------------------------------------------------------------ host ranges
@pytest.mark.parametrize("n", [1, RANGE - 1, RANGE, RANGE + 1, 2 * RANGE + 3])
def test_host_ranges(n):
    """1-byte (found, an entity column), 2-, 4- and 8-byte results copied back per range, the last range partial"""
    rng = np.random.default_rng(n)
    universe = np.arange(-500, 500, dtype=np.int64)
    t = ref.keyed_table(rng, universe, 20000, widths=(8,))
    keys, ts = ref.query(rng, universe, n)
    outs = [t.out(0, ref.MISS_BITS), t.out(1, ref.MISS_NAT)]
    run(ts, [(t, keys, 1, outs)], ref.entity_cols(rng, n, 4))


# ------------------------------------------------------------------------------------------------------ device path
def _device_join(ts, sets, cols, stream, preload):
    """b2s_pit_join_device over sentinel-filled buffers of n + 1 elements -> (order, [(outs, ts_out, found)], cols, miss),
    after checking every sentinel and the launches"""
    n = len(ts) if ts is not None else len(sets[0][1])
    bufs = []

    def dev(arr=None, elem=None):
        if arr is None:
            b = nat.DeviceBuffer((n + 1) * elem).upload(np.full((n + 1) * elem, SENT, np.uint8))
        else:
            b = nat.DeviceBuffer(np.asarray(arr).nbytes).upload(arr)
        bufs.append(b)
        return b

    def back(b, dtype):
        raw = b.download(np.uint8, (n + 1) * np.dtype(dtype).itemsize)
        assert (raw[n * np.dtype(dtype).itemsize:] == SENT).all(), "the element past n was written"
        return raw[: n * np.dtype(dtype).itemsize].view(dtype)

    d_ts = dev(np.ascontiguousarray(ts, np.int64)) if ts is not None else None
    descs, layout = [], []
    for ix, keys, asof, outs in sets:
        d_keys = dev(np.ascontiguousarray(keys, np.int64))
        d_outs = [dev(elem=np.dtype(dt).itemsize) for _w, dt, _m in outs]
        d_tsout, d_found = dev(elem=8), dev(elem=1)
        descs.append((ix, d_keys.ptr, int(asof), [(w, np.dtype(dt).itemsize, m, b.ptr) for (w, dt, m), b in zip(outs, d_outs)],
                      d_tsout.ptr, d_found.ptr))
        layout.append((d_outs, d_tsout, d_found, [dt for _w, dt, _m in outs]))
    c_s, keep = c_sets(descs)
    d_cols = [(dev(c), dev(elem=c.dtype.itemsize), c.dtype) for c in cols]
    cc = c_cols([(s.ptr, d.ptr, dt.itemsize) for s, d, dt in d_cols])
    d_order = dev(elem=8)
    d_miss = dev(np.append(preload, np.uint64(0xA5A5A5A5A5A5A5A5)))
    before = nat.launch_count()
    handle = None if stream is None else stream.cuda_stream
    nat.check(nat.load().b2s_pit_join_device(None if d_ts is None else d_ts.ptr, n, c_s, len(sets), cc, len(cols), d_order.ptr,
                                             d_miss.ptr, handle))
    assert nat.launch_count() - before == join_launches(ts is not None, n, len(sets), len(cols))
    if stream is not None:
        stream.synchronize()
    nat.check(nat.load().b2s_device_sync())
    joined = [([back(b, dt) for b, dt in zip(d_outs, dts)], back(d_tsout, np.int64), back(d_found, np.uint8).astype(bool))
              for d_outs, d_tsout, d_found, dts in layout]
    miss = d_miss.download(np.uint64, len(preload) + 1)
    assert miss[-1] == np.uint64(0xA5A5A5A5A5A5A5A5)
    return back(d_order, np.int64), joined, [back(d, dt) for _s, d, dt in d_cols], miss[:-1] - preload


@pytest.mark.parametrize("stream", ["default", "caller"])
@pytest.mark.parametrize("with_ts", [True, False])
def test_device_path_equals_the_host_run(with_ts, stream):
    rng = np.random.default_rng(int(with_ts))
    ts, sets, cols = ref.mixed_sets(rng, 3, 6000, with_ts=with_ts)
    cols = cols + ref.entity_cols(rng, 6000, 66)
    host = run(ts, sets, cols)
    ixs = {id(t): make_index(t) for t, *_ in sets}
    strm = None
    if stream == "caller":
        import torch

        strm = torch.cuda.Stream(device=0)
    preload = np.array([1000, 7, (1 << 40) + 3], np.uint64)
    got = _device_join(ts, [(ixs[id(t)], k, a, o) for t, k, a, o in sets], cols, strm, preload)
    ref.assert_same(got, host)


# --------------------------------------------------------------------------------------------------------- refusals
def test_refusals_launch_nothing():
    rng = np.random.default_rng(1)
    lib = nat.load()
    t = ref.wide_table(rng, rng.integers(0, 8, size=64), rng.integers(0, 5, size=64), [8])
    ix = make_index(t)
    exact = make_index(ref.Table(np.arange(8, dtype=np.int64), np.zeros(8, np.int64)))
    n = 64
    bufs = [nat.DeviceBuffer(8 * (n + 2)).upload(np.zeros(n + 2, np.int64)) for _ in range(9)]
    d_ts, d_keys, d_out4, d_out8, d_tsout, d_found, d_order, d_miss, d_col = [b.ptr for b in bufs]

    def call(ts=d_ts, keys=d_keys, asof=1, outs=None, ts_out=d_tsout, cols=None, order=d_order, miss=d_miss, index=ix):
        """-> the return code, or "launched" when a call that should be refused launched a kernel"""
        outs = [(0, 4, 0, d_out4), (1, 8, 0, d_out8)] if outs is None else outs
        c_s, keep = c_sets([(index, keys, asof, outs, ts_out, d_found)])
        cc = c_cols(cols or [])
        before = nat.launch_count()
        rc = lib.b2s_pit_join_device(ts, n, c_s, 1, cc, len(cols or []), order, miss, None)
        nat.check(lib.b2s_device_sync())
        return "launched" if rc != 0 and nat.launch_count() != before else rc

    # the baseline and an exact-key join on a one-row-per-key index are valid
    assert call() == 0 and call(index=exact, asof=0, outs=[(0, 4, 0, d_out4)]) == 0
    refused = {
        "asof_without_ts": call(ts=None),
        "exact_on_repeated_keys": call(asof=0),
        "ts_misaligned": call(ts=d_ts + 4),
        "keys_misaligned": call(keys=d_keys + 4),
        "ts_out_misaligned": call(ts_out=d_tsout + 4),
        "out4_misaligned": call(outs=[(0, 4, 0, d_out4 + 2)]),
        "out8_misaligned": call(outs=[(1, 8, 0, d_out8 + 4)]),
        "order_misaligned": call(order=d_order + 4),
        "miss_misaligned": call(miss=d_miss + 4),
        "word_past_row": call(outs=[(t.row_words, 4, 0, d_out4)]),
        "pair_past_row": call(outs=[(t.row_words - 1, 8, 0, d_out8)]),
        "negative_word": call(outs=[(-1, 4, 0, d_out4)]),
        "bytes_2": call(outs=[(0, 2, 0, d_out4)]),
        "n_out_257": call(outs=[(0, 4, 0, d_out4)] * 257),
        "col_bytes_3": call(cols=[(d_col, d_out8, 3)]),
        "col_misaligned": call(cols=[(d_col + 2, d_out8, 4)]),
        "null_miss": call(miss=None),
    }
    assert {k: v for k, v in refused.items() if v != INVALID} == {}
    # the host entry point shares the checks
    h_ts, h_keys = np.zeros(n, np.int64), np.zeros(n, np.int64)
    c_s, keep = c_sets([(ix, h_keys.ctypes.data, 1, [], None, None)])
    before = nat.launch_count()
    assert lib.b2s_pit_join_host(None, n, c_s, 1, c_cols([]), 0, None, np.zeros(1, np.uint64).ctypes.data, None) == INVALID
    assert lib.b2s_pit_join_host(h_ts.ctypes.data, n, c_s, 1, c_cols([]), 0, None, None, None) == INVALID
    assert nat.launch_count() == before


@pytest.mark.parametrize("case", ["n_rows_0", "n_rows_2^31", "n_cols_257", "col_bytes_2", "null_column"])
def test_index_create_refusals(case):
    lib = nat.load()
    m = 4
    keys, ts = np.arange(m, dtype=np.int64), np.zeros(m, np.int64)
    col = np.zeros(m, np.float32)
    n_cols = 257 if case == "n_cols_257" else 1
    ptrs = (C.c_void_p * n_cols)(*([None if case == "null_column" else col.ctypes.data] * n_cols))
    widths = np.full(n_cols, 2 if case == "col_bytes_2" else 4, np.int32)
    n_rows = {"n_rows_0": 0, "n_rows_2^31": 1 << 31}.get(case, m)
    out = C.c_void_p()
    before = nat.launch_count()
    rc = lib.b2s_pit_index_create(keys.ctypes.data, ts.ctypes.data, n_rows, ptrs, nat._p(widths, C.c_int32), n_cols, C.byref(out))
    assert rc == INVALID and not out.value
    assert nat.launch_count() == before


# ---------------------------------------------------------------------------------------------- through the product
def _check_product(fsets, frames, feats, entity, ts):
    fx.register(fsets, frames)
    want = oo.get_offline_features(frames, feats, entity, ts)
    n_dev = sum(entity[c].dtype.kind in "iufMb" for c in entity.columns)
    before = nat.launch_count()
    got = boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts).to_dataframe()
    assert nat.launch_count() - before == join_launches(True, len(entity), len(fsets), n_dev)
    pd.testing.assert_frame_equal(got, want, check_exact=True)
    return got


def test_offline_datetime_features_in_s_and_ns():
    got = _check_product(*fx.workload(21, n_sets=3, exact_sets=(1,), dates=("s", "ns")))
    assert str(got["s0ds"].dtype) == "datetime64[s]" and str(got["s0dns"].dtype) == "datetime64[ns]"
    assert got["s0ds"].isna().any() and got["s0ds"].notna().any()


def test_offline_entity_frame_with_seventy_numeric_columns():
    fsets, frames, feats, entity, ts = fx.workload(22, n_sets=2, n_entity=3000)
    rng = np.random.default_rng(0)
    dts = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.float32, np.float64, bool]
    for c in range(70):
        dt = dts[c % len(dts)]
        entity[f"e{c:02d}"] = rng.random(len(entity)) < 0.5 if dt is bool else ref.random_bits(rng, len(entity), dt)
        if dt in (np.float32, np.float64):
            entity[f"e{c:02d}"] = rng.normal(size=len(entity)).astype(dt)
    _check_product(fsets, frames, feats, entity, ts)
