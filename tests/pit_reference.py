"""A point-in-time (as-of) join in plain numpy, and the crafted workloads the b2s_pit kernels are held to.

The reference shares no algorithm with csrc/b2s_pit.cu (radix sort, slot array, per-run binary search) nor with
tests/emulated_pit.py (sorted index, per-run bisection).  It is a sweep: the feature rows and the queries are concatenated,
lexsorted by (key, timestamp, feature rows before queries, input position), and each query takes the last feature row seen
since its key's group began.  So a query takes the set's last row with timestamp <= its own, of equal (key, timestamp) rows the
last in input order, and an exact-key query (timestamp INT64_MAX) the key's only row.  The outputs are gathered from the input
columns by input row number; every Table carries an int32 "input row number" column first, so an output of it names the exact
row a join took.

`join(ts, sets, cols)` takes the arguments of `mlrun_b200.feature_store.offline.pit_join` with `Table`s in place of indexes and
returns what it returns: (order, [(outputs, ts_out, found)] per set, permuted entity columns, misses per set).
"""

import numpy as np

from tests import table_hash

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
NAT = I64_MIN
EXTREME_KEYS = np.array([I64_MIN, -1, 0, 1, I64_MAX], dtype=np.int64)
# bits stored for a row without a match: a float32 / float64 NaN, NaT, zero and an arbitrary 64-bit pattern
MISS_NAN32, MISS_NAN64, MISS_NAT, MISS_ZERO, MISS_BITS = 0x7FC00000, 0x7FF8000000000000, 1 << 63, 0, 0xDEADBEEFCAFEF00D


class Table:
    """a feature set's rows: int64 keys, int64 nanosecond timestamps and 4- / 8-byte columns, the first of them (unless
    `rowid=False`) the int32 input row number"""

    def __init__(self, keys, ts, cols=(), rowid=True):
        self.keys = np.ascontiguousarray(keys, dtype=np.int64)
        self.ts = np.ascontiguousarray(ts, dtype=np.int64)
        assert len(self.keys) == len(self.ts)
        self.cols = ([np.arange(len(self.keys), dtype=np.int32)] if rowid else []) + [np.ascontiguousarray(c) for c in cols]
        assert all(c.dtype.itemsize in (4, 8) and len(c) == len(self.keys) for c in self.cols)
        self.word = list(np.cumsum([0] + [c.dtype.itemsize // 4 for c in self.cols]))  # first word of each column
        self.row_words = int(self.word[-1])

    def out(self, c, miss=MISS_ZERO):
        """the output descriptor (src_word, dtype, miss bits) of column c whole"""
        return (int(self.word[c]), self.cols[c].dtype, miss)

    def words(self):
        """[n_rows, row_words] uint32: row r's columns in column order, in input order"""
        w = [c.view(np.uint32).reshape(len(self.keys), -1) for c in self.cols]
        return np.concatenate(w, axis=1) if w else np.zeros((len(self.keys), 0), np.uint32)


def asof_rows(f_keys, f_ts, q_keys, q_ts):
    """for each query, the input row of the feature set it takes, or -1 (the sweep)"""
    f_keys, f_ts = np.asarray(f_keys, np.int64), np.asarray(f_ts, np.int64)
    q_keys, q_ts = np.asarray(q_keys, np.int64), np.asarray(q_ts, np.int64)
    m, n = len(f_keys), len(q_keys)
    keys, ts = np.concatenate([f_keys, q_keys]), np.concatenate([f_ts, q_ts])
    is_q = np.concatenate([np.zeros(m, bool), np.ones(n, bool)])
    pos = np.concatenate([np.arange(m), np.arange(n)])
    s = np.lexsort((pos, is_q, ts, keys))
    k, at = keys[s], np.arange(m + n)
    group = np.maximum.accumulate(np.where(np.concatenate([[True], k[1:] != k[:-1]]), at, 0))
    last = np.maximum.accumulate(np.where(is_q[s], -1, at))  # sweep position of the last feature row seen
    took = np.where(last >= group, pos[s][np.maximum(last, 0)], -1)
    out = np.full(n, -1, np.int64)
    out[pos[s][is_q[s]]] = took[is_q[s]]
    return out


def join(ts, sets, cols):
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    order = np.argsort(np.asarray(ts, np.int64), kind="stable") if ts is not None else np.arange(n)
    joined, misses = [], []
    for table, keys, asof, outs in sets:
        q_ts = np.asarray(ts, np.int64) if asof else np.full(n, I64_MAX, np.int64)
        row = asof_rows(table.keys, table.ts, keys, q_ts)[order]
        found = row >= 0
        safe = np.maximum(row, 0)
        words = table.words()
        arrays = []
        for w, dt, miss in outs:
            dt = np.dtype(dt)
            if dt.itemsize == 4:
                v = np.where(found, words[safe, w], np.uint32(miss & 0xFFFFFFFF))
            else:
                v = words[safe, w].astype(np.uint64) | (words[safe, w + 1].astype(np.uint64) << np.uint64(32))
                v = np.where(found, v, np.uint64(miss))
            arrays.append(np.ascontiguousarray(v).view(dt))
        joined.append((arrays, np.where(found, table.ts[safe], NAT), found))
        misses.append(int((~found).sum()))
    return order.astype(np.int64), joined, [np.asarray(c)[order] for c in cols], np.array(misses, np.uint64)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def assert_same(got, want):
    """two results of `join` / pit_join are equal bit for bit (NaN payloads included)"""
    (g_order, g_sets, g_cols, g_miss), (w_order, w_sets, w_cols, w_miss) = got[:4], want[:4]
    np.testing.assert_array_equal(g_order, w_order)
    assert len(g_sets) == len(w_sets) and len(g_cols) == len(w_cols)
    for s, ((ga, gt, gf), (wa, wt, wf)) in enumerate(zip(g_sets, w_sets)):
        assert len(ga) == len(wa)
        np.testing.assert_array_equal(np.asarray(gf, bool), wf, err_msg=f"set {s} found")
        np.testing.assert_array_equal(gt, wt, err_msg=f"set {s} ts_out")
        for j, (g, w) in enumerate(zip(ga, wa)):
            assert g.dtype.itemsize == w.dtype.itemsize
            np.testing.assert_array_equal(bits(g), bits(w), err_msg=f"set {s} output {j}")
    for c, (g, w) in enumerate(zip(g_cols, w_cols)):
        np.testing.assert_array_equal(bits(g), bits(w), err_msg=f"entity column {c}")
    np.testing.assert_array_equal(np.asarray(g_miss, np.uint64), w_miss)


# ------------------------------------------------------------------------------------------------------ crafted workloads
def random_bits(rng, n, dtype):
    """n values of `dtype` with uniformly random bits (NaN payloads, denormals and -0.0 included for floats)"""
    size = np.dtype(dtype).itemsize
    return rng.integers(0, 256, size=n * size, dtype=np.uint8).view(dtype)


def entity_cols(rng, n, n_cols):
    """n_cols entity columns of widths 1, 2, 4, 8, 1, 2, ... with random bits"""
    return [random_bits(rng, n, (np.uint8, np.int16, np.float32, np.int64)[c % 4]) for c in range(n_cols)]


def wide_table(rng, keys, ts, widths):
    """a Table over (keys, ts) whose columns after the row number have the given widths (4 or 8) and random bits: after the
    row number's one word, an 8-byte column preceded by an even number of 4-byte columns starts at an odd word"""
    return Table(keys, ts, [random_bits(rng, len(keys), np.float32 if w == 4 else np.float64) for w in widths])


def all_outs(table, misses=(MISS_NAN32, MISS_NAN64, MISS_NAT, MISS_ZERO, MISS_BITS)):
    """every column of `table` as one output, the miss bits cycling through `misses`"""
    return [table.out(c, misses[c % len(misses)]) for c in range(len(table.cols))]


def asof_edges(rng, n_keys=8, dup=3):
    """-> (Table, query keys, query timestamps): for each key of a run with a `dup`-fold duplicated (key, ts) in the middle,
    queries before its first timestamp, at it, between two timestamps, on the duplicate, at its last timestamp, after it,
    at INT64_MIN + 1 and at INT64_MAX; the same times for unknown keys whose probe walks a chain that wraps past the last
    slot.  One key's run starts at INT64_MIN + 1 and another's ends at INT64_MAX.  Rows and queries are in random order."""
    cap = table_hash.capacity(n_keys)
    homes = [cap - 1] * 3 + [cap - 2] + [int(h) for h in rng.integers(0, cap, size=max(n_keys - 4, 0))]
    keys = table_hash.keys_with_home_slots(homes[:n_keys], cap, rng, exclude=EXTREME_KEYS)
    f_keys, f_ts, q_keys, q_ts = [], [], [], []
    for i, k in enumerate(keys):
        t = np.sort(rng.choice(np.arange(-50, 50) * 10**9, size=6, replace=False))
        if i == 0:
            t[0] = I64_MIN + 1
        if i == 1:
            t[-1] = I64_MAX
        run = np.concatenate([t[:3], np.repeat(t[3], dup), t[4:]])
        f_keys += [k] * len(run)
        f_ts += run.tolist()
        between = t[1] + (t[2] - t[1]) // 2
        q = [t[0] - 1 if t[0] > I64_MIN + 1 else t[0], t[0], between, t[3], t[-1], t[-1] + 1 if t[-1] < I64_MAX else t[-1],
             I64_MIN + 1, I64_MAX]
        q_keys += [k] * len(q)
        q_ts += q
    unknown = table_hash.keys_with_home_slots([cap - 1, cap - 2, cap - 1], cap, rng, exclude=np.concatenate([keys, EXTREME_KEYS]))
    for k in unknown:
        q_keys += [k] * 4
        q_ts += [I64_MIN + 1, 0, f_ts[len(f_ts) // 2], I64_MAX]
    p, s = rng.permutation(len(f_keys)), rng.permutation(len(q_keys))
    return (Table(np.array(f_keys)[p], np.array(f_ts, np.int64)[p]), np.array(q_keys, np.int64)[s], np.array(q_ts, np.int64)[s])


def keyed_table(rng, universe, n_rows, exact=False, widths=(8, 4)):
    """a Table over keys drawn from `universe` (every key once when `exact`) with timestamps from a small range, so that
    (key, ts) pairs repeat"""
    keys = rng.permutation(universe) if exact else universe[rng.integers(0, len(universe), size=n_rows)]
    ts = rng.integers(-20, 20, size=len(keys)) * 10**9
    return wide_table(rng, keys, ts, widths)


def query(rng, universe, n, unknown=0.25):
    """n entity keys drawn from `universe`, a share of them unknown, and timestamps over the feature sets' range and past
    it, with ties"""
    keys = universe[rng.integers(0, len(universe), size=n)]
    unk = rng.random(n) < unknown
    keys[unk] = rng.integers(10**15, 10**16, size=int(unk.sum()))
    return keys, rng.integers(-25, 25, size=n) * 10**9


def mixed_sets(rng, n_sets, n, with_ts=True):
    """-> (ts, sets, cols): n_sets sets over one key universe, as-of and exact-key alternating (exact only without `with_ts`),
    each with every column as an output; two entity columns"""
    universe = np.unique(np.concatenate([EXTREME_KEYS, rng.integers(-10**6, 10**6, size=40)]))
    keys, ts = query(rng, universe, n)
    sets = []
    for s in range(n_sets):
        asof = with_ts and s % 2 == 0
        t = keyed_table(rng, universe, 300, exact=not asof, widths=[(4, 8), (8,), (8, 8, 4)][s % 3])
        sets.append((t, keys, asof, all_outs(t)))
    return (ts if with_ts else None), sets, entity_cols(rng, n, 2)


def workloads():
    """name -> (ts, sets, cols) of the crafted workloads at small sizes (the CPU pins run them all)"""
    rng = np.random.default_rng(20)
    out = {}
    t, qk, qt = asof_edges(rng)
    out["asof_edges"] = (qt, [(t, qk, 1, all_outs(t))], [])
    t = Table(np.repeat(EXTREME_KEYS, 7), rng.integers(-3, 3, size=35) * 10**9)
    qk = np.concatenate([EXTREME_KEYS, EXTREME_KEYS, [2, -2]])
    out["extreme_keys"] = (rng.integers(-4, 4, size=12) * 10**9, [(t, qk, 1, all_outs(t))], entity_cols(rng, 12, 4))
    t = Table(np.full(5000, 7, np.int64), rng.integers(0, 50, size=5000))
    out["one_key"] = (rng.integers(-1, 52, size=300), [(t, np.full(300, 7, np.int64), 1, all_outs(t))], [])
    t = wide_table(rng, np.arange(64, dtype=np.int64) * 3, np.zeros(64, np.int64), [4, 4, 8, 4, 8, 8, 4, 8])
    out["interleaved_widths"] = (None, [(t, np.arange(100, dtype=np.int64) - 10, 0, all_outs(t))], [])
    t = wide_table(rng, rng.integers(0, 50, size=400), rng.integers(0, 9, size=400), [8] * 255)
    out["n_out_256"] = (rng.integers(0, 10, size=200), [(t, rng.integers(0, 60, size=200), 1, all_outs(t))], [])
    for n_sets in (1, 2, 5):
        out[f"mixed_{n_sets}_sets"] = mixed_sets(rng, n_sets, 500)
    out["exact_without_ts"] = mixed_sets(rng, 3, 500, with_ts=False)
    out["cols_130"] = (rng.integers(0, 5, size=300), [], entity_cols(rng, 300, 130))
    out["sort_only"] = (rng.choice(EXTREME_KEYS, size=999), [], [])
    return out
