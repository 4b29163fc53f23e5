"""The exhaustive timestamp set the DateExtractor tests run (tests/test_ingest_dates_cpu.py on a host build of
csrc/b2s_dates.cuh, tests/test_gpu_ingest_paths.py on columns_kernel), and its calendar fields from pandas."""

import numpy as np
import pandas as pd

from mlrun_b200 import _native as nat

NS_S, NS_H, NS_D = 1_000_000_000, 3_600_000_000_000, 86_400_000_000_000
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
# part id -> the pd.Series.dt attribute it restates (DP_WEEK: ISO week, Series.dt.isocalendar().week)
PARTS = {v: k for k, v in reversed(list(nat.DATE_PARTS.items()))}
assert sorted(PARTS) == list(range(18)) and PARTS[17] == "week" and PARTS[6] == "day_of_week"
# offsets inside a day: both sides of every second, hour and day boundary the floor divisions meet
DAY_OFFSETS = np.array([0, 1, NS_S - 1, NS_S, NS_H - 1, 12 * NS_H + 7, NS_D - NS_S, NS_D - 1], dtype=np.int64)
# the ends of datetime64[ns] (INT64_MIN is NaT) and -1 s +- 1 ns, where truncating division goes wrong (-1 ns and -1 s
# are on the day grid already)
EXTRAS = np.array([I64_MIN + 1, I64_MAX, -NS_S - 1, -NS_S + 1], dtype=np.int64)


def exhaustive_timestamps():
    """every day from 1677-09-22 to 2262-04-10 at each of DAY_OFFSETS, then EXTRAS (int64 nanoseconds, no NaT)"""
    first = (np.datetime64("1677-09-22", "D") - np.datetime64("1970-01-01", "D")).astype(np.int64)
    last = (np.datetime64("2262-04-10", "D") - np.datetime64("1970-01-01", "D")).astype(np.int64)
    days = np.arange(first, last + 1, dtype=np.int64)
    return np.concatenate([(days[:, None] * NS_D + DAY_OFFSETS[None, :]).reshape(-1), EXTRAS])


def pandas_part(ts, part):
    """int64 calendar field `part` (an id of nat.DATE_PARTS) of int64 nanosecond timestamps without NaT"""
    s = pd.Series(ts.view("datetime64[ns]"))
    v = s.dt.isocalendar().week if part == nat.DATE_PARTS["week"] else getattr(s.dt, PARTS[part])
    return v.to_numpy().astype(np.int64)
