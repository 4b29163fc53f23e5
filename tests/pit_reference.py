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

`train(ts, sets, cols, label)` takes the arguments of `offline.pit_train` the same way and returns what it returns: the join,
cut to the rows a training set keeps, with the misses each set makes at its place in the merge.  It restates the contract of
`b2s_pit_train_*` (include/b200serve.h) on the sweep's result and shares no code with tests/emulated_train.py.
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


# ---------------------------------------------------------------------------------------------------------- training sets
LABEL_FOUND, LABEL_NAN, LABEL_NAT = 0, 1, 2  # B2S_PIT_LABEL_*


def label_present(values, kind):
    """per row: the label value passes its kind's test (NAN: not a NaN of its 4- or 8-byte float; NAT: not INT64_MIN)"""
    values = np.ascontiguousarray(values)
    if kind == LABEL_NAN:
        return ~np.isnan(values.view(np.float32 if values.dtype.itemsize == 4 else np.float64))
    if kind == LABEL_NAT:
        return values.view(np.int64) != NAT
    return np.ones(len(values), bool)


def train(ts, sets, cols, label):
    """the rows of `join` a training set keeps: those every exact-key set matched and, with label = (set, output, kind) or
    (-1, entity column, kind), whose label is present -- its set matched (set >= 0) and its value passes `label_present`.
    miss[s] counts the rows set s misses among those every exact-key set before s matched."""
    order, joined, permuted, _miss = join(ts, sets, cols)
    n = len(order)
    exact_found = [found for (_t, _k, asof, _o), (_a, _t_out, found) in zip(sets, joined) if not asof]
    keep = np.logical_and.reduce(exact_found) if exact_found else np.ones(n, bool)
    miss = []
    for s, (_arrays, _t_out, found) in enumerate(joined):
        before = [joined[e][2] for e in range(s) if not sets[e][2]]
        earlier = np.logical_and.reduce(before) if before else np.ones(n, bool)
        miss.append(int((earlier & ~found).sum()))
    if label is not None:
        s, j, kind = label
        if s >= 0:
            keep = keep & joined[s][2] & label_present(joined[s][0][j], kind)
        else:
            keep = keep & label_present(permuted[j], kind)
    return (order[keep], [([a[keep] for a in arrays], t[keep], f[keep]) for arrays, t, f in joined], [p[keep] for p in permuted],
            np.array(miss, np.uint64))


def assert_same_train(got, want):
    """two results of `train` / pit_train are equal bit for bit, every array holding exactly the kept rows; with pit_train's
    stats (a fifth element), its `kept` too"""
    kept = len(want[0])
    assert len(got[0]) == kept
    for arrays, t, f in got[1]:
        assert len(t) == len(f) == kept and all(len(a) == kept for a in arrays)
    assert all(len(c) == kept for c in got[2])
    if len(got) > 4:
        assert got[4]["kept"] == kept
    assert_same(got, want)


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


# ------------------------------------------------------------------------------------------- crafted training-set workloads
TILE = 1024  # rows per block of the keep and scatter kernels: one row per thread, 32 warps
# the NaNs `isnan` must catch: quiet, signalling, negative and with payload bits
NAN32_BITS = np.array([0x7FC00000, 0x7F800001, 0xFFC00000, 0x7FC12345], np.uint32)
NAN64_BITS = np.array([0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FF8000000012345], np.uint64)
# label values at the edges of their type: the four NaNs, then what no test may drop: -0.0, +inf, -inf, the smallest
# denormal, +max, -max and 1.5; for int64 NaT (INT64_MIN) and the values next to it and at the other end
F32_EDGES = np.concatenate([NAN32_BITS, np.array([0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x7F7FFFFF, 0xFF7FFFFF,
                                                  0x3FC00000], np.uint32)]).view(np.float32)
F64_EDGES = np.concatenate([NAN64_BITS, np.array([0x8000000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 1,
                                                  0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x3FF8000000000000],
                                                 np.uint64)]).view(np.float64)
I64_EDGES = np.array([I64_MIN, I64_MIN + 1, 0, I64_MAX], np.int64)

# the rows `label_column` keeps, by position in the 1 024-row tiles and 32-row warps of the keep and scatter kernels
LABEL_PATTERNS = ["all", "none", "tile_first", "tile_last", "lane_31", "warp_empty", "alt_tiles", "tile_in_7", "random_50",
                  "random_1", "random_99.9"]


def keep_pattern(n, pattern, rng):
    """[n] bool: the rows of `pattern`.  warp_empty: every row but one whole warp per tile (warp tile % 32); alt_tiles:
    every other tile empty; tile_in_7: only tiles 3, 10, 17, ..., so a one-block scan over up to 3 tiles per thread has
    threads whose tiles are all empty; random_p: each row with probability p %"""
    q = np.arange(n)
    if pattern in ("all", "none"):
        return np.full(n, pattern == "all")
    if pattern == "tile_first":
        return q % TILE == 0
    if pattern == "tile_last":
        return q % TILE == TILE - 1
    if pattern == "lane_31":
        return q % 32 == 31
    if pattern == "warp_empty":
        return (q % TILE) // 32 != (q // TILE) % 32
    if pattern == "alt_tiles":
        return (q // TILE) % 2 == 0
    if pattern == "tile_in_7":
        return (q // TILE) % 7 == 3
    if pattern.startswith("random_"):
        return rng.random(n) < float(pattern[len("random_"):]) / 100
    raise ValueError(pattern)


def label_column(n, pattern, dtype=np.float32, seed=0):
    """-> (ts, sets, cols, label) without timestamps or sets, so the order is the identity and the kept rows are exactly
    `keep_pattern(n, pattern)`: the one entity column is the label (NAN kind), a kept row holding its row number and a
    dropped one one of the four NaNs"""
    keep = keep_pattern(n, pattern, np.random.default_rng(seed))
    dtype = np.dtype(dtype)
    nans, uint = (NAN32_BITS, np.uint32) if dtype.itemsize == 4 else (NAN64_BITS, np.uint64)
    col = np.where(keep, np.arange(n, dtype=dtype).view(uint), nans[np.arange(n) % 4]).view(dtype)
    return None, [], [col], (-1, 0, LABEL_NAN)


def ordered_sets(kinds, n=3000, seed=0):
    """-> (ts, sets, cols): one set per letter of `kinds` ("A" as-of, "E" exact key), in that order, over one universe of
    256 keys, each with its row number, a float32 and a float64 output.  An as-of set lacks 32 random keys and misses
    entity rows before a key's first row; the j-th exact set lacks keys 2j, 2j + 1 and 2j + 2, one of them shared with the
    exact set before it; a tenth of the entity rows have keys no set holds.  So past the first exact set every set's misses
    at its place in the merge are fewer than its misses.  No timestamps when no set is as-of (the order is then the
    identity); two entity columns."""
    rng = np.random.default_rng(seed)
    universe = np.arange(256, dtype=np.int64) * 7919 - 10**6
    keys, ts = query(rng, universe, n, unknown=0.1)
    sets, j = [], 0
    for kind in kinds:
        if kind == "A":
            t = keyed_table(rng, rng.permutation(universe)[32:], 600, widths=(4, 8))
        else:
            t = keyed_table(rng, np.delete(universe, np.arange(2 * j, 2 * j + 3)), 0, exact=True, widths=(4, 8))
            j += 1
        sets.append((t, keys, int(kind == "A"), all_outs(t)))
    return (ts if "A" in kinds else None), sets, entity_cols(rng, n, 2)


# set orders from 0 to 64 sets (the most one training-set call joins)
SET_ORDERS = ["", "A", "E", "AE", "EA", "EE", "EAEAE", "AAEEA", "EEEEE", "AAE" * 21, "EA" * 31 + "E", "A" * 64, "E" * 64,
              "EA" * 32]

# where the label sits (over ordered_sets("EAEA"): set 1 is as-of, set 2 exact): <set>_<output>_<miss bits> with the miss
# bits a NaN (the value test would drop a missed row too) or zero / arbitrary bits (only the found flag drops it), "found"
# a FOUND label on a float64 output holding NaNs (kept); entity_<kind>_<bytes> an entity column
LABEL_PLACES = ["asof_f32_nan", "asof_f64_nan", "asof_f32_zero", "asof_f64_bits", "exact_f32_nan", "exact_f64_zero",
                "asof_f64_found", "exact_f32_found", "entity_found_1", "entity_found_2", "entity_found_8", "entity_nan_4",
                "entity_nan_8", "entity_nat_8"]


def label_place(case, n=3000, seed=0):
    """-> (ts, sets, cols, label) of a LABEL_PLACES case; a third of every float value of every set is one of the four NaNs,
    and of the label column a third is NaN (NAN and FOUND kinds) or NaT"""
    rng = np.random.default_rng(seed)
    ts, sets, cols = ordered_sets("EAEA", n, seed)
    for t, *_ in sets:
        for c, nans in ((1, NAN32_BITS), (2, NAN64_BITS)):
            hit = np.flatnonzero(rng.random(len(t.keys)) < 0.3)
            t.cols[c].view(nans.dtype)[hit] = nans[hit % 4]
    where, what, last = case.split("_")
    if where == "entity":
        kind = {"found": LABEL_FOUND, "nan": LABEL_NAN, "nat": LABEL_NAT}[what]
        dtype = {1: np.uint8, 2: np.int16, 4: np.float32, 8: np.int64 if kind == LABEL_NAT else np.float64}[int(last)]
        col = random_bits(rng, n, dtype)
        hit = np.flatnonzero(rng.random(n) < 0.3)
        if kind == LABEL_NAT:
            col[hit] = NAT
        elif col.dtype.kind == "f":
            nans = NAN32_BITS if col.dtype.itemsize == 4 else NAN64_BITS
            col.view(nans.dtype)[hit] = nans[hit % 4]
        return ts, sets, cols + [col], (-1, len(cols), kind)
    s, j = (1 if where == "asof" else 2), (1 if what == "f32" else 2)
    miss = {"nan": MISS_NAN32 if j == 1 else MISS_NAN64, "zero": MISS_ZERO, "bits": MISS_BITS, "found": MISS_NAN64}[last]
    t, keys, asof, outs = sets[s]
    sets[s] = (t, keys, asof, outs[:j] + [t.out(j, miss)] + outs[j + 1:])
    return ts, sets, cols, (s, j, LABEL_FOUND if last == "found" else LABEL_NAN)


def label_edges(dtype, place, kind=None, n=3000, seed=0):
    """-> (ts, sets, cols, label): an exact-key set holding every key of a 64-key universe, then an as-of set over it; the
    label cycles through the edges of `dtype` (F32_EDGES, F64_EDGES or I64_EDGES) in the exact set ("exact"), the as-of set
    ("asof") or an entity column ("entity"); kind defaults to NAN for floats and NAT for int64"""
    rng = np.random.default_rng(seed)
    edges = {"float32": F32_EDGES, "float64": F64_EDGES, "int64": I64_EDGES}[np.dtype(dtype).name]
    kind = (LABEL_NAT if edges is I64_EDGES else LABEL_NAN) if kind is None else kind
    universe = np.arange(64, dtype=np.int64) * 31 + 5
    keys, ts = query(rng, universe, n, unknown=0.05)
    exact = Table(rng.permutation(universe), np.zeros(64, np.int64), [edges[np.arange(64) % len(edges)]])
    m = 800
    asof = Table(universe[rng.integers(0, 64, size=m)], rng.integers(-20, 20, size=m) * 10**9, [edges[np.arange(m) % len(edges)]])
    sets = [(exact, keys, 0, all_outs(exact)), (asof, keys, 1, all_outs(asof))]
    cols = [edges[np.arange(n) % len(edges)]] + entity_cols(rng, n, 2)
    return ts, sets, cols, {"exact": (0, 1, kind), "asof": (1, 1, kind), "entity": (-1, 0, kind)}[place]


EDGE_CASES = [f"{d}_{p}" for d in ("float32", "float64", "int64") for p in ("asof", "exact", "entity")] + ["float64_asof_found",
                                                                                                          "int64_entity_found"]

TRAIN_WORKLOADS = ([f"pattern_{p}" for p in LABEL_PATTERNS] + [f"order_{k or '-'}" for k in SET_ORDERS]
                   + [f"place_{c}" for c in LABEL_PLACES] + [f"edges_{c}" for c in EDGE_CASES])


def train_workload(name):
    """-> (ts, sets, cols, label) of the crafted training-set workload `name` (of TRAIN_WORKLOADS) at a small size"""
    group, case = name.split("_", 1)
    if group == "pattern":
        i = LABEL_PATTERNS.index(case)
        return label_column(5 * TILE + 37, case, np.float32 if i % 2 else np.float64, seed=i)
    if group == "order":
        return ordered_sets(case.strip("-"), seed=len(case)) + (None,)
    if group == "place":
        return label_place(case, seed=LABEL_PLACES.index(case))
    dtype, place, *found = case.split("_")
    return label_edges(dtype, place, LABEL_FOUND if found else None, seed=EDGE_CASES.index(case))
