"""Goldens of the offline merge: the REAL LocalFeatureMerger.merge (mlrun/feature_store/retrieval/base.py:412-468 with
local_merger.py:29-104) over stub feature sets (metadata.name, spec.timestamp_key) on seeded workloads, stored in
ref_offline.pkl.xz: merged frame, drop columns and the resulting timestamp column per workload.

    python -m tests.golden.gen_offline      # needs the reference sources importable (tests/golden/_refshim.py)

`merge_inputs(seed)` rebuilds a workload's inputs; tests/test_offline_cpu.py runs oracle/offline.py's merge on them.
"""
import lzma
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_offline.pkl.xz")
N_GOLDEN = 48


def merge_inputs(seed):
    """-> (entity frame, entity timestamp column or None, [(set name, timestamp key or None, engine frame, keys)])"""
    rng = np.random.default_rng(seed)
    unit = ["ns", "us", "ms", "s"][seed % 4]
    fs_unit = ["ns", unit][seed % 3 == 0]
    f = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}
    n_keys = int(rng.integers(1, 12))
    key_kind = ["int64", "int32", "str", "pair"][seed % 4 if seed % 5 else 0]
    names = ["a", "b"] if key_kind == "pair" else ["id"]
    universe = rng.choice(np.arange(-50, 50), size=n_keys, replace=False)

    def keycols(vals):
        if key_kind == "pair":
            return {"a": (vals // 7).astype(np.int32), "b": (vals % 7).astype(np.int32)}
        if key_kind == "str":
            return {"id": pd.array([f"k{v}" for v in vals], dtype="str")}
        return {"id": vals.astype(np.int64 if key_kind == "int64" else np.int32)}

    def distinct(n, lo, hi):
        return rng.choice(np.arange(lo, hi), size=n, replace=False).astype(np.int64)

    sets = []
    ts_entity = None if seed % 7 == 6 else "t"
    for s in range(int(rng.integers(1, 4))):
        name = f"fs{s}"
        exact = ts_entity is None or rng.random() < 0.2
        rows = n_keys if exact else int(rng.integers(1, 40))
        vals = rng.permutation(universe)[:rows] if exact else universe[rng.integers(0, n_keys, size=rows)]
        cols = keycols(vals)
        ts = None
        if not exact or rng.random() < 0.5:
            ts = f"when{s}" if rng.random() < 0.7 else "t"
            cols[ts] = pd.to_datetime(distinct(rows, -500, 500) * f[unit], unit=fs_unit).as_unit(fs_unit) if fs_unit == unit else \
                pd.to_datetime(distinct(rows, -500, 500) * f[unit]).as_unit(fs_unit)
        cols[f"x_{name}"] = rng.normal(size=rows).astype(np.float32)
        cols[f"n_{name}"] = rng.integers(-9, 9, size=rows).astype(["int32", "int8", "int16"][s % 3])
        if rng.random() < 0.4:
            cols[f"b_{name}"] = rng.random(rows) < 0.5
        if rng.random() < 0.3:
            cols["label"] = rng.normal(size=rows).astype(np.float32)  # collides with the entity frame: suffixed, dropped
        sets.append((name, ts if not exact or ts_entity is None else None, pd.DataFrame(cols), names))
    n = int(rng.integers(1, 30))
    ecols = keycols(np.concatenate([universe, [97, 98]])[rng.integers(0, n_keys + 2, size=n)])
    ecols["t"] = pd.to_datetime(distinct(n, -520, 520) * f[unit], unit="ns").as_unit(unit)
    ecols["label"] = rng.normal(size=n)
    return pd.DataFrame(ecols), ts_entity, sets


def run_merge(merge_fn, seed):
    """merge_fn(entity, entity_ts, stubs, dfs, keys) -> (frame, drop, ts)"""
    from oracle.offline import FeatureSetStub

    entity, ts, sets = merge_inputs(seed)
    stubs = [FeatureSetStub(name, t) for name, t, _df, _k in sets]
    dfs = [df.drop(columns=[c for c in df.columns if c.startswith("when") or c == "t"]) if t is None else df for _n, t, df, _k in sets]
    try:
        return merge_fn(entity, ts, stubs, dfs, [(k, k) for *_x, k in sets])
    except Exception as exc:  # noqa: BLE001
        return {"raised": type(exc).__name__, "message": str(exc).splitlines()[0] if str(exc) else ""}


def reference_merge(entity, ts, stubs, dfs, keys):
    from mlrun.feature_store.retrieval.local_merger import LocalFeatureMerger

    merger = LocalFeatureMerger(vector=None)
    merger.merge(ts, [None] + stubs, [entity.copy()] + [d.copy() for d in dfs], [[[], []]] + [list(map(list, k)) for k in keys],
                 [None] + [["default_join", False]] * len(stubs))
    return merger._result_df, list(merger._drop_columns), ts or next((s.spec.timestamp_key for s in stubs if s.spec.timestamp_key), None)


def main():
    from tests.golden import _refshim

    _refshim.install()
    outs = [run_merge(reference_merge, seed) for seed in range(N_GOLDEN)]
    with lzma.open(GOLDEN, "wb") as f:
        pickle.dump(outs, f)
    print("recorded", len(outs), "reference merges")


if __name__ == "__main__":
    main()
