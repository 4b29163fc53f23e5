"""The point-in-time reference of tests/pit_reference.py pinned on the CPU: its sweep equals a brute-force scan of every feature
row for every query, and the numpy emulation of the b2s_pit join that the CPU suite runs the product over
(tests/emulated_pit.py) equals the sweep on every crafted workload the GPU suite (tests/test_gpu_pit_paths.py) uses."""

import numpy as np
import pytest

from tests import emulated_pit
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
