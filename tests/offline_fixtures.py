"""Seeded point-in-time workloads shared by the offline-retrieval tests: feature-set frames, entity frames and vectors.

Timestamps are distinct within each frame unless `ties` asks otherwise, so the row order of the reference (pandas'
unstable sort) is defined and can be compared exactly."""

import numpy as np
import pandas as pd

from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff

EXTREME_KEYS = np.array([0, -1, np.iinfo(np.int64).min, np.iinfo(np.int64).max], dtype=np.int64)


def _distinct_ts(rng, n, lo, hi):
    """n distinct int64 nanosecond timestamps in [lo, hi)"""
    span = hi - lo
    vals = set()
    while len(vals) < n:
        vals.update((lo + rng.integers(0, span, size=2 * (n - len(vals)) + 4)).tolist())
    return np.array(list(vals)[:n], dtype=np.int64)


def _keys(rng, kind, n_keys):
    if kind == "int64":
        base = rng.choice(np.arange(-10 * n_keys, 10 * n_keys), size=max(n_keys - 4, 1), replace=False).astype(np.int64)
        return np.unique(np.concatenate([EXTREME_KEYS, base]))[:n_keys] if n_keys >= 4 else base[:n_keys]
    if kind == "int32":
        return rng.choice(np.arange(-5 * n_keys, 5 * n_keys), size=n_keys, replace=False).astype(np.int32)
    if kind == "str":
        return np.array([f"user-{i}" for i in rng.choice(10 * n_keys, size=n_keys, replace=False)], dtype=object)
    raise ValueError(kind)


def _key_columns(kind, names, chosen):
    if kind == "pair":
        return {names[0]: (chosen // 7).astype(np.int32), names[1]: (chosen % 7 - 3).astype(np.int32)}
    col = chosen.astype(object) if kind == "str" else chosen
    return {names[0]: pd.array(col, dtype="str") if kind == "str" else col}


def workload(seed, n_sets=2, n_rows=200, n_keys=16, n_entity=120, key_kind="int64", unit="ns", exact_sets=(), unknown=0.2,
             before_1970=True, ties=False, n_float=3, ints=True, dates=()):
    """-> (featuresets, {name: (entities, ts, frame)}, features, entity frame, entity timestamp column); `dates`: units of
    datetime64 feature columns to add to every set (values before and after 1970, a tenth of them NaT)"""
    rng = np.random.default_rng(seed)
    span = (-(10**12) if before_1970 else 10**12, 3 * 10**12)
    f = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}[unit]
    kind = "int32" if key_kind == "pair" else key_kind
    universe = _keys(rng, "int64" if kind == "int64" else kind, n_keys) if kind != "int32" else \
        rng.choice(np.arange(0, 7 * n_keys), size=n_keys, replace=False).astype(np.int64)
    names = ["a", "b"] if key_kind == "pair" else ["id"]
    fsets, frames, features = [], {}, []
    for s in range(n_sets):
        name = f"fs{s}"
        exact = s in exact_sets
        rows = n_keys if exact else n_rows
        chosen = rng.permutation(universe)[:rows] if exact else universe[rng.integers(0, len(universe), size=rows)]
        cols = _key_columns(key_kind, names, chosen)
        ts = None
        if not exact:
            raw = _distinct_ts(rng, rows, span[0] // f, span[1] // f) if not ties else rng.integers(0, 6, size=rows) * 10**6
            cols["when"] = pd.to_datetime(raw, unit=unit).as_unit(unit) if not ties else pd.to_datetime(raw).as_unit(unit)
            ts = "when"
        for j in range(n_float):
            v = rng.normal(size=rows).astype(np.float32)
            v[rng.random(rows) < 0.1] = np.nan
            cols[f"s{s}x{j}"] = v
        if ints:
            cols[f"s{s}count"] = rng.integers(-1000, 1000, size=rows).astype(np.int32)
            cols[f"s{s}small"] = rng.integers(-100, 100, size=rows).astype(np.int8)
            cols[f"s{s}flag"] = rng.random(rows) < 0.5
        for u in dates:
            d = rng.integers(-(10**9), 4 * 10**9, size=rows) * (10**9 // {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}[u])
            d[rng.random(rows) < 0.1] = np.iinfo(np.int64).min
            cols[f"s{s}d{u}"] = d.view(f"datetime64[{u}]")
        frame = pd.DataFrame(cols)
        fs = bingest.FeatureSet(name, entities=names, timestamp_key=ts)
        fsets.append(fs)
        frames[name] = (names, ts, frame)
        picked = [f"s{s}x{j}" for j in range(1, n_float)] + ([f"s{s}count", f"s{s}small", f"s{s}flag"] if ints else [])
        picked += [f"s{s}d{u}" for u in dates]
        features += [f"{name}.s{s}x0 as first{s}"] + [f"{name}.{c}" for c in picked] if s % 2 == 0 else [f"{name}.*"]
    # entity rows: known keys, unknown keys, times before / between / after the feature rows
    n_unknown = int(n_entity * unknown)
    ekeys = universe[rng.integers(0, len(universe), size=n_entity)]
    if n_unknown and key_kind != "str":
        ekeys[:n_unknown] = universe.max() // 2 + 7919 if key_kind == "pair" else rng.integers(10**15, 10**16, size=n_unknown)
    ecols = _key_columns(key_kind, names, ekeys)
    if n_unknown and key_kind == "str":
        ecols["id"] = pd.array([f"nobody-{i}" if i < n_unknown else v for i, v in enumerate(ecols["id"])], dtype="str")
    if ties:
        raw = rng.integers(0, 6, size=n_entity) * 10**6
    else:  # a quarter of the entity times equal a feature row's time (the exact-match edge), all distinct
        exact_part = frames["fs0"][2]["when"].to_numpy().view(np.int64)[:n_entity // 4] if frames["fs0"][1] else np.zeros(0, np.int64)
        rest = _distinct_ts(rng, 2 * n_entity + 8, span[0] // f - 1000, span[1] // f + 1000)
        rest = rest[~np.isin(rest, exact_part)][:n_entity - len(exact_part)]
        raw = rng.permutation(np.concatenate([exact_part, rest]))
    ecols["t"] = pd.to_datetime(raw, unit=unit).as_unit(unit) if not ties else pd.to_datetime(raw).as_unit(unit)
    ecols["label"] = rng.normal(size=n_entity)
    ecols["weight"] = rng.integers(0, 5, size=n_entity).astype(np.int16)
    entity = pd.DataFrame(ecols)
    return fsets, frames, features, entity, "t"


def register(fsets, frames):
    for fs in fsets:
        boff.register_offline_frame(fs, frames[fs.name][2])
