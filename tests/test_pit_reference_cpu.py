"""The point-in-time reference of tests/pit_reference.py pinned on the CPU: its sweep equals a brute-force scan of every feature
row for every query, and the numpy emulation of the b2s_pit join that the CPU suite runs the product over
(tests/emulated_pit.py) equals the sweep on every crafted workload the GPU suite (tests/test_gpu_pit_paths.py) uses.  Its
training-set rule `train` equals the header's contract applied row by row, and the CPU suite's emulation of
b2s_pit_train_host (tests/emulated_train.py) equals it on every crafted training-set workload of
tests/test_gpu_training_set_paths.py."""

import math
import struct

import numpy as np
import pytest

from tests import emulated_pit
from tests import emulated_train
from tests import pit_reference as ref


def brute_rows(f_keys, f_ts, q_keys, q_ts):
    """per query: of the rows with its key and timestamp <= its own, the one with the largest (timestamp, input row)"""
    out = np.full(len(q_keys), -1, np.int64)
    for i, (k, t) in enumerate(zip(q_keys.tolist(), q_ts.tolist())):
        cand = np.flatnonzero((f_keys == k) & (f_ts <= t))
        if len(cand):
            out[i] = cand[np.lexsort((cand, f_ts[cand]))[-1]]
    return out


@pytest.mark.parametrize("seed", range(40))
def test_sweep_equals_a_brute_force_scan(seed):
    rng = np.random.default_rng(seed)
    m, n = int(rng.integers(1, 60)), int(rng.integers(1, 80))
    universe = np.concatenate([ref.EXTREME_KEYS, rng.integers(-5, 5, size=3)])[: int(rng.integers(1, 9))]
    f_keys = universe[rng.integers(0, len(universe), size=m)]
    times = np.array([ref.I64_MIN + 1, -3, -1, 0, 1, 2, 5, ref.I64_MAX], np.int64)  # few values: (key, ts) pairs repeat
    f_ts = times[rng.integers(0, len(times), size=m)]
    q_keys = np.concatenate([universe, [77]])[rng.integers(0, len(universe) + 1, size=n)]
    q_ts = np.concatenate([times, [ref.I64_MIN, 3]])[rng.integers(0, len(times) + 2, size=n)]
    np.testing.assert_array_equal(ref.asof_rows(f_keys, f_ts, q_keys, q_ts), brute_rows(f_keys, f_ts, q_keys, q_ts))


def test_sweep_takes_the_last_duplicate_in_input_order():
    f_keys = np.array([5, 5, 5, 5, 9], np.int64)
    f_ts = np.array([10, 20, 10, 20, 10], np.int64)
    got = ref.asof_rows(f_keys, f_ts, np.array([5, 5, 5, 9, 4]), np.array([9, 10, 25, 10, 10]))
    np.testing.assert_array_equal(got, [-1, 2, 3, 4, -1])


def test_asof_edges_reach_every_edge():
    """the edge workload holds what its docstring promises: duplicates, both int64 ends and a wrapped probe chain"""
    from tests import table_hash

    rng = np.random.default_rng(0)
    t, qk, qt = ref.asof_edges(rng)
    rows = ref.asof_rows(t.keys, t.ts, qk, qt)
    assert (rows == -1).any() and (rows >= 0).any()
    assert ref.I64_MAX in t.ts and ref.I64_MIN + 1 in t.ts
    pairs = np.stack([t.keys, t.ts], 1)
    assert len(np.unique(pairs, axis=0)) < len(pairs)
    cap = table_hash.capacity(len(np.unique(t.keys)))
    homes = table_hash.home_slot(np.unique(t.keys), cap)
    assert (homes == cap - 1).sum() >= 3  # the chain from the last slot wraps to slot 0 and on
    unknown = np.setdiff1d(qk, t.keys)
    assert len(unknown) and (table_hash.home_slot(unknown, cap) >= cap - 2).all()


def _emulated(ts, sets, cols):
    return emulated_pit.pit_join(None if ts is None else np.asarray(ts, np.int64),
                                 [(emulated_pit.EmulatedPitIndex(t.keys, t.ts, t.cols), k, a, o) for t, k, a, o in sets], cols)


@pytest.mark.parametrize("name", sorted(ref.workloads()))
def test_emulated_join_equals_the_sweep(name):
    ts, sets, cols = ref.workloads()[name]
    ref.assert_same(_emulated(ts, sets, cols), ref.join(ts, sets, cols))


# ------------------------------------------------------------------------------------------------------ training sets
def brute_train(ts, sets, cols, label):
    """the training-set contract applied row by row to the sweep's join: a row is kept when every exact-key set matched it
    and its label is present (its set matched it; NAN: the value, read as a 4- or 8-byte IEEE float, is not NaN; NAT: the
    value, read as a signed 64-bit integer, is not INT64_MIN); miss[s] counts the rows set s misses among those every
    exact-key set before s matched"""
    order, joined, permuted, _miss = ref.join(ts, sets, cols)
    exact = [not asof for _t, _k, asof, _o in sets]
    miss, kept = [0] * len(sets), []
    for q in range(len(order)):
        found = [bool(f[q]) for _a, _t, f in joined]
        for s in range(len(sets)):
            if all(found[e] for e in range(s) if exact[e]) and not found[s]:
                miss[s] += 1
        keep = all(found[e] for e in range(len(sets)) if exact[e])
        if keep and label is not None:
            s, j, kind = label
            raw = (joined[s][0][j] if s >= 0 else permuted[j])[q].tobytes()
            if s >= 0 and not found[s]:
                keep = False
            elif kind == ref.LABEL_NAN:
                keep = not math.isnan(struct.unpack("<f" if len(raw) == 4 else "<d", raw)[0])
            elif kind == ref.LABEL_NAT:
                keep = int.from_bytes(raw, "little", signed=True) != -(2**63)
        if keep:
            kept.append(q)
    k = np.array(kept, np.int64)
    return (order[k], [([a[k] for a in arrays], t[k], f[k]) for arrays, t, f in joined], [p[k] for p in permuted],
            np.array(miss, np.uint64))


def _mixed(rng, m, edges):
    """m values of the edges' dtype: two in five an edge, the rest random normals"""
    normal = rng.normal(size=m).astype(edges.dtype) if edges.dtype.kind == "f" else rng.integers(-9, 9, size=m)
    return np.where(rng.random(m) < 0.4, edges[rng.integers(0, len(edges), size=m)], normal).astype(edges.dtype)


def random_train_case(seed):
    """-> (ts, sets, cols, label): 0 to 5 sets in a random order of as-of and exact-key, each with its row number, a float32,
    a float64 and an int64 column whose values are often label edges (NaNs of every kind, NaT); entity columns of 1 to 8
    bytes and such float / int64 columns; the label on a random output or entity column, with a kind its width allows"""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(1, 90))
    universe = np.arange(10, dtype=np.int64) * 5 - 20
    keys, ts = ref.query(rng, universe, n, unknown=0.2)
    sets = []
    for _ in range(int(rng.integers(0, 6))):
        asof = bool(rng.random() < 0.5)
        known = universe[rng.random(len(universe)) < 0.8]
        m = int(rng.integers(1, 40)) if asof else len(known)
        t_keys = known[rng.integers(0, len(known), size=m)] if asof and len(known) else rng.permutation(known)
        m = len(t_keys)
        t = ref.Table(t_keys, rng.integers(-25, 25, size=m) * 10**9,
                      [_mixed(rng, m, ref.F32_EDGES), _mixed(rng, m, ref.F64_EDGES), _mixed(rng, m, ref.I64_EDGES)])
        misses = [ref.MISS_NAN32, ref.MISS_NAN64, ref.MISS_NAT, ref.MISS_ZERO, ref.MISS_BITS]
        sets.append((t, keys, int(asof), [t.out(c, misses[int(rng.integers(0, 5))]) for c in range(4)]))
    if not any(a for _t, _k, a, _o in sets) and rng.random() < 0.5:
        ts = None
    cols = ref.entity_cols(rng, n, int(rng.integers(0, 4))) + [_mixed(rng, n, e) for e in (ref.F32_EDGES, ref.F64_EDGES, ref.I64_EDGES)]
    kinds = {np.dtype(np.float32): [ref.LABEL_NAN, ref.LABEL_FOUND], np.dtype(np.float64): [ref.LABEL_NAN, ref.LABEL_FOUND],
             np.dtype(np.int64): [ref.LABEL_NAT, ref.LABEL_NAN, ref.LABEL_FOUND]}
    on_sets = [(s, j, dt) for s, (t, _k, _a, outs) in enumerate(sets) for j, (_w, dt, _m) in enumerate(outs)]
    places = on_sets if on_sets and rng.random() < 0.5 else [(-1, c, col.dtype) for c, col in enumerate(cols)]
    label = None
    if rng.random() < 0.85:
        s, j, dt = places[int(rng.integers(0, len(places)))]
        options = kinds.get(np.dtype(dt), [ref.LABEL_FOUND])
        label = (s, j, options[int(rng.integers(0, len(options)))])
    if seed % 5 == 4:  # NAT labels: the int64 entity column, or the last set's int64 output
        label = (len(sets) - 1, 3, ref.LABEL_NAT) if sets and seed % 2 else (-1, len(cols) - 1, ref.LABEL_NAT)
    return ts, sets, cols, label


@pytest.mark.parametrize("seed", range(40))
def test_train_equals_a_per_row_loop(seed):
    case = random_train_case(seed)
    ref.assert_same_train(ref.train(*case), brute_train(*case))


def test_random_train_cases_cover_the_contract():
    """the 40 cases hold every order of up to 5 sets, labels of every kind on sets and entity columns, and drop rows by a
    missed exact-key set, a missed label set, a NaN and a NaT"""
    seen = set()
    for seed in range(40):
        ts, sets, cols, label = random_train_case(seed)
        order, joined, permuted, _m = ref.join(ts, sets, cols)
        seen.add(f"sets_{len(sets)}")
        seen.add("no_ts" if ts is None else "ts")
        if any(not a for _t, _k, a, _o in sets) and not all(joined[s][2].all() for s in range(len(sets)) if not sets[s][2]):
            seen.add("exact_drops")
        if label is not None:
            s, j, kind = label
            seen.add(f"label_{'set' if s >= 0 else 'entity'}_{kind}")
            values = joined[s][0][j] if s >= 0 else permuted[j]
            present = ref.label_present(values, kind)
            if s >= 0 and not joined[s][2].all():
                seen.add("label_set_missed")
            if not present.all():
                seen.add(f"value_drops_{kind}")
    want = {f"sets_{k}" for k in range(6)} | {"ts", "no_ts", "exact_drops", "label_set_missed", "value_drops_1", "value_drops_2"}
    want |= {f"label_{w}_{k}" for w in ("set", "entity") for k in (0, 1, 2)}
    assert want <= seen, want - seen


def _emulated_train(ts, sets, cols, label):
    return emulated_train.pit_train(None if ts is None else np.asarray(ts, np.int64),
                                    [(emulated_pit.EmulatedPitIndex(t.keys, t.ts, t.cols), k, a, o) for t, k, a, o in sets], cols, label)


@pytest.mark.parametrize("name", ref.TRAIN_WORKLOADS)
def test_emulated_train_equals_train(name):
    w = ref.train_workload(name)
    ref.assert_same_train(_emulated_train(*w), ref.train(*w))


def test_crafted_train_workloads_reach_their_edges():
    """the label patterns keep what they name; past the first exact-key set every set's misses at its place are fewer than
    its plain misses; every label edge reaches the label of found rows, and only NaNs / NaT are dropped for their value"""
    n = 3 * ref.TILE + 5
    rng = np.random.default_rng(0)
    q = np.arange(n)
    assert (np.flatnonzero(ref.keep_pattern(n, "tile_first", rng)) == [0, 1024, 2048, 3072]).all()
    assert (np.flatnonzero(ref.keep_pattern(n, "tile_last", rng)) == [1023, 2047, 3071]).all()
    assert (ref.keep_pattern(n, "lane_31", rng) == (q % 32 == 31)).all()
    empty = ~ref.keep_pattern(n, "warp_empty", rng)
    assert [np.unique(q[empty & (q // 1024 == t)] // 32 % 32).tolist() for t in range(3)] == [[0], [1], [2]]
    for kinds in ref.SET_ORDERS:
        ts, sets, cols = ref.ordered_sets(kinds, seed=len(kinds))
        assert len(sets) == len(kinds) <= 64
        got, plain = ref.train(ts, sets, cols, None)[3], ref.join(ts, sets, cols)[3]
        first = kinds.find("E")
        for s in range(len(kinds)):
            assert (got[s] < plain[s]) if 0 <= first < s else (got[s] == plain[s]), (kinds, s)
    edges = {"float32": ref.F32_EDGES, "float64": ref.F64_EDGES, "int64": ref.I64_EDGES}
    assert ref.label_present(ref.F32_EDGES, ref.LABEL_NAN).tolist() == [False] * 4 + [True] * 7
    assert ref.label_present(ref.F64_EDGES, ref.LABEL_NAN).tolist() == [False] * 4 + [True] * 7
    assert ref.label_present(ref.I64_EDGES, ref.LABEL_NAT).tolist() == [False, True, True, True]
    for case in ref.EDGE_CASES:
        dtype, place = case.split("_")[:2]
        ts, sets, cols, (s, j, _kind) = ref.label_edges(dtype, place)
        _order, joined, permuted, _m = ref.join(ts, sets, cols)
        values = joined[s][0][j][joined[s][2]] if s >= 0 else permuted[j]
        uint = np.uint32 if values.dtype.itemsize == 4 else np.uint64
        assert set(values.view(uint).tolist()) >= set(edges[dtype].view(uint).tolist()), case
