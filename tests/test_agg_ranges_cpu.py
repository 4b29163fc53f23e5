"""What tests/test_gpu_aggregate_paths.py and the variance bound of tests/test_gpu_aggregate.py rest on, checked without a GPU:
the bound passes the pairwise and sequential (count, mean, M2) combines and rejects sum x^2 - (sum x)^2 / n; on the exact
workload the integer prefix-difference references equal math.fsum and the oracle; the restated walk of range_reduce
(tests/agg_ranges.py) covers every range exactly once and the GPU levels case reaches every shape of it; and the oracle and the
numpy emulation count a 1 ns period's window at 1677 without overflowing."""

import math

import numpy as np
import pytest

from mlrun_b200 import _native as nat
from oracle import aggregate as oa
from tests import agg_ranges as ar
from tests import emulated_agg
from tests.test_gpu_aggregate_paths import LEVEL_SIZES, LEVEL_WINDOWS, MEAN, grid

EPS = 2.0**-53
K = 128
I64_MIN = -(1 << 63)


def _bound(x, m2):
    """tests/test_gpu_aggregate.py's stdvar bound with the exact sums: K eps sqrt(sum x^2 M2) / (n - 1)"""
    return K * EPS * math.sqrt(math.fsum(v * v for v in x) * m2) / (len(x) - 1)


def _m2(x):
    mean = math.fsum(x) / len(x)
    return math.fsum((v - mean) ** 2 for v in x)


def _combine(a, b):
    """the kernel's combine of (count, mean, M2)"""
    c = a[0] + b[0]
    d = b[1] - a[1]
    return c, a[1] + d * (b[0] / c), a[2] + b[2] + d * d * (a[0] * b[0] / c)


def _pairwise(x):
    if len(x) == 1:
        return 1.0, x[0], 0.0
    h = len(x) // 2
    return _combine(_pairwise(x[:h]), _pairwise(x[h:]))


def _sequential(x):
    acc = (1.0, x[0], 0.0)
    for v in x[1:]:
        acc = _combine(acc, (1.0, v, 0.0))
    return acc


@pytest.mark.parametrize("mean", [1e3, 1e5, 1e6, 3e7])
@pytest.mark.parametrize("n", [2, 33, 1000, 30000])
def test_the_variance_bound_passes_chan_and_rejects_the_cancelling_formula(mean, n):
    rng = np.random.default_rng(n)
    x = (mean + rng.normal(size=n)).astype(np.float32).astype(np.float64).tolist()
    m2 = _m2(x)
    ref, tol = m2 / (n - 1), _bound(x, m2)
    for name, combine in (("pairwise", _pairwise), ("sequential", _sequential)):
        got = combine(x)[2] / (n - 1)
        assert abs(got - ref) <= tol, (name, abs(got - ref), tol)
    xs = np.asarray(x)
    naive = (np.sum(xs * xs) - np.sum(xs) ** 2 / n) / (n - 1)  # numpy's pairwise sums
    if mean >= 1e5 and n >= 1000:
        assert abs(naive - ref) > tol, (abs(naive - ref), tol)


@pytest.mark.parametrize("mean", [0.0, MEAN])
def test_the_exact_workload_sums_exactly_at_the_largest_size(mean):
    """every sequential fp64 partial sum of the grid equals the integer prefix sum; windows equal math.fsum and the oracle"""
    n = max(n for n, _m in LEVEL_SIZES)
    rng = np.random.default_rng(1)
    x = grid(rng, n, mean).astype(np.float64)
    u = np.rint((x - mean) * 1024).astype(np.int64)
    pu, pq = np.r_[0, np.cumsum(u)], np.r_[0, np.cumsum(u * u)]
    c = np.arange(n + 1)
    np.testing.assert_array_equal(np.r_[0.0, np.cumsum(x)], (c * int(mean * 1024) + pu) / 1024)
    if not mean:
        np.testing.assert_array_equal(np.r_[0.0, np.cumsum(x * x)], pq / 2.0**20)
    windows = [(0, n - 1), (1, n - 2), (n // 3, n // 3 + 2**20)] + [tuple(sorted(rng.integers(0, n, 2).tolist())) for _ in range(5)]
    for lo, hi in windows:
        s = ((hi - lo + 1) * int(mean * 1024) + int(pu[hi + 1] - pu[lo])) / 1024
        assert s == math.fsum(x[lo:hi + 1])
        if not mean:
            assert pq[hi + 1] - pq[lo] < 2**53 and (pq[hi + 1] - pq[lo]) / 2.0**20 == math.fsum(x[lo:hi + 1] ** 2)
    for lo in (0, 12345, n - 3000):  # the oracle's reduce on windows it can afford
        w = x[lo:lo + 3000]
        s = (3000 * int(mean * 1024) + int(pu[lo + 3000] - pu[lo])) / 1024
        assert oa.reduce(w, "sum") == s and oa.reduce(w, "avg") == s / 3000
        if not mean:
            assert oa.reduce(w, "sqr") == (pq[lo + 3000] - pq[lo]) / 2.0**20


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 64, 65, 96, 97, 98, 1023, 1024, 1025, 1056, 1057, 1089, 1100])
def test_the_walk_covers_every_range_exactly_once_and_possible_lists_its_shapes(n):
    lo, hi = np.triu_indices(n)
    ok, shapes = ar.walk(lo, hi, n)
    assert ok.all()
    assert shapes == ar.possible(n)


@pytest.mark.parametrize("n", [n for n, _m in LEVEL_SIZES])
def test_the_walk_covers_sampled_ranges_at_the_gpu_sizes(n):
    rng = np.random.default_rng(n)
    a, b = rng.integers(0, n, 200_000), rng.integers(0, n, 200_000)
    ok, _s = ar.walk(np.minimum(a, b), np.maximum(a, b), n)
    assert ok.all()


@pytest.mark.parametrize("n", [n for n, _m in LEVEL_SIZES])
def test_the_gpu_levels_case_reaches_every_shape(n):
    """the rows of test_gpu_aggregate_paths.py::test_levels_every_row_every_window take every shape of the walk that
    exists at n, at every level from 0 to n_levels"""
    n_levels, _m = ar.levels(n)
    i = np.arange(n, dtype=np.int64)
    reached = set()
    for w in LEVEL_WINDOWS:
        ok, shapes = ar.walk(np.maximum(0, i - w + 1), i, n)
        assert ok.all()
        reached |= shapes
    assert reached == ar.possible(n)
    # the fourth stored level (pre / suf[3]) is built from 2^20 + 1 rows, but there its 33 elements leave no range to split
    # across two of its blocks; ranges read it from 2^21 + 37 on
    assert n_levels == (3 if n < 2**20 else 4)
    assert (("stop", 3) in reached) == (n > 2**21)


def test_one_ns_period_window_start_below_int64_min():
    """timestamps at 1677, window 2^62 or INT64_MAX, period 1: every earlier row of the key is in the window"""
    ts = np.array([I64_MIN + 1, I64_MIN + 5, I64_MIN + 10], np.int64)
    keys = np.zeros(3, np.int64)
    x = np.array([1, 2, 3], np.float32)
    for window in (1 << 62, (1 << 63) - 1):
        aggs = [dict(name="p", column="x", operations=["count"], windows=[window], period=1)]
        assert oa.aggregate(keys, ts, {"x": x}, aggs)[f"p_count_{window}"].tolist() == [1, 2, 3]
        out = np.full(3, np.nan)
        emulated_agg.aggregate_host(keys, ts, [(x, nat.COL_F32, nat.AGG_OPS["count"], 1, [window], [out])], 3)
        assert out.tolist() == [1, 2, 3]
