"""Goldens of training sets: the REAL BaseMerger.start -> _generate_offline_vector (mlrun/feature_store/retrieval/base.py:
78-368) on the local engine, over the reference's own FeatureVector and FeatureSet classes whose `to_dataframe` returns the
registered frame (the entities, the timestamp key, then the asked columns, as FeatureSet.to_dataframe asks its target for
them), stored in ref_training_set.pkl.xz: the frame `to_dataframe()` returns, or the exception, per workload.

    python -m tests.golden.gen_training_set     # needs the reference sources importable (tests/golden/_refshim.py)

`training_inputs(seed)` rebuilds a workload: entity-less and entity vectors, 1 to 4 feature sets, as-of and exact-key
sets, labels of every kind in every position, with_indexes on and off, string / int32-pair / int64 keys, float64 columns.
tests/test_training_set_cpu.py runs tests/training_oracle.py on them.
"""
import lzma
import os
import pickle
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_training_set.pkl.xz")
N_GOLDEN = 64
LABEL_DTYPES = ["float32", "float64", "int32", "int8", "bool"]


def training_inputs(seed):
    """-> dict(frames={set: (entities, timestamp key or None, frame)}, features, label_feature, entity_rows or None,
    entity_timestamp_column, with_indexes)"""
    rng = np.random.default_rng(seed)
    key_kind = ["int64", "str", "pair", "int32"][seed % 4]
    names = ["a", "b"] if key_kind == "pair" else ["id"]
    n_keys = int(rng.integers(1, 10))
    universe = rng.choice(np.arange(-40, 40), size=n_keys, replace=False)

    def keycols(vals):
        if key_kind == "pair":
            return {"a": (vals // 7).astype(np.int32), "b": (vals % 7).astype(np.int32)}
        if key_kind == "str":
            return {"id": pd.array([f"k{v}" for v in vals], dtype="str")}
        return {"id": vals.astype(np.int64 if key_kind == "int64" else np.int32)}

    def distinct(n):
        return rng.choice(np.arange(-10**4, 10**4), size=n, replace=False).astype(np.int64) * 10**9

    entity_less = seed % 3 != 2
    n_sets = int(rng.integers(1, 5))
    frames, features = {}, []
    spine_ts = entity_less and rng.random() < 0.8
    label_set = int(rng.integers(0, n_sets)) if rng.random() < 0.85 else None
    for s in range(n_sets):
        name = f"fs{s}"
        # the spine (entity-less) may lack a timestamp key; later sets are as-of unless exact-key
        exact = (s == 0 and entity_less and not spine_ts) or rng.random() < 0.25 or (entity_less and not spine_ts)
        rows = n_keys if exact else int(rng.integers(1, 30))
        if s == 0 and entity_less:
            rows = int(rng.integers(1, 30)) if spine_ts else n_keys
        vals = rng.permutation(universe)[:rows] if rows <= n_keys and exact else universe[rng.integers(0, n_keys, size=rows)]
        cols = keycols(vals)
        ts = None
        if not exact or (s == 0 and spine_ts):
            ts = "when" if rng.random() < 0.5 else f"when{s}"
            cols[ts] = pd.to_datetime(distinct(rows)).as_unit("ns")
        x = rng.normal(size=rows).astype(np.float32)
        x[rng.random(rows) < 0.2] = np.nan
        cols[f"x{s}"] = x
        agg = rng.normal(size=rows) * 10.0 ** rng.integers(-300, 300, size=rows)
        agg[rng.random(rows) < 0.2] = np.nan
        cols[f"agg{s}_sum_1h"] = agg
        cols[f"n{s}"] = rng.integers(-9, 9, size=rows).astype(["int32", "int16", "int8"][s % 3])
        if s == label_set:
            kind = LABEL_DTYPES[int(rng.integers(0, len(LABEL_DTYPES)))]
            lab = rng.integers(0, 2, size=rows).astype(kind) if kind != "bool" else rng.random(rows) < 0.5
            if kind.startswith("float"):
                lab = rng.normal(size=rows).astype(kind)
                lab[rng.random(rows) < float(rng.choice([0.0, 0.3, 1.0]))] = np.nan
            cols["label"] = lab
        frames[name] = (names, ts, pd.DataFrame(cols))
        if rng.random() < 0.4:
            features.append(f"{name}.*")
        else:
            picked = [c for c in cols if c not in names and c != ts and c != "label" and rng.random() < 0.7] or [f"x{s}"]
            features += [f"{name}.{c}" + (f" as {c}_{s}a" if rng.random() < 0.2 else "") for c in picked]
    label_feature = f"fs{label_set}.label" if label_set is not None else None
    entity_rows = entity_ts = None
    if not entity_less:
        n = int(rng.integers(1, 25))
        ecols = keycols(np.concatenate([universe, [97]])[rng.integers(0, n_keys + 1, size=n)])
        ecols["t"] = pd.to_datetime(distinct(n)).as_unit("ns")
        ecols["w"] = rng.normal(size=n)
        entity_rows, entity_ts = pd.DataFrame(ecols), "t"
    elif seed % 17 == 5:
        entity_ts = "t"  # the reference's error: a timestamp column without entity rows
    return dict(frames=frames, features=features, label_feature=label_feature, entity_rows=entity_rows,
                entity_timestamp_column=entity_ts, with_indexes=bool(seed % 2))


def run(fn, seed):
    """fn(**training_inputs(seed)) -> its frame, or {"raised": type name, "message": first line}"""
    try:
        return fn(**training_inputs(seed))
    except Exception as exc:  # noqa: BLE001 -- the outcome is what is recorded
        return {"raised": type(exc).__name__, "message": str(exc).splitlines()[0] if str(exc) else ""}


def reference_training_set(frames, features, label_feature, entity_rows, entity_timestamp_column, with_indexes):
    import mlrun.feature_store as fs
    from mlrun.feature_store.retrieval.local_merger import LocalFeatureMerger
    from mlrun.features import Entity, Feature

    objects = {}
    for name, (entities, ts, frame) in frames.items():
        fset = fs.FeatureSet(name, entities=[Entity(e) for e in entities], timestamp_key=ts)
        for c in frame.columns:
            if c not in entities:
                fset[c] = Feature(name=c)

        def to_dataframe(columns=None, frame=frame, head=list(entities) + ([ts] if ts else []), **_kw):
            return frame[head + [c for c in columns if c not in head]].copy()

        fset.to_dataframe = to_dataframe
        objects[name] = fset
    vector = fs.FeatureVector("v", list(features), label_feature=label_feature, with_indexes=with_indexes)
    vector.feature_set_objects = objects
    vector.save = lambda *a, **k: None
    if entity_rows is None and entity_timestamp_column is not None:
        from mlrun.feature_store.api import _get_offline_features

        _get_offline_features(vector, None, entity_timestamp_column)
    merger = LocalFeatureMerger(vector)
    resp = merger.start(entity_rows=None if entity_rows is None else entity_rows.copy(), entity_timestamp_column=entity_timestamp_column,
                        with_indexes=with_indexes)
    return resp.to_dataframe()


def main():
    from tests.golden import _refshim

    _refshim.install()
    import logging

    logging.disable(logging.WARNING)
    outs = [run(reference_training_set, seed) for seed in range(N_GOLDEN)]
    with lzma.open(GOLDEN, "wb") as f:
        pickle.dump(outs, f)
    print("recorded", len(outs), "reference training sets;", sum(isinstance(o, dict) for o in outs), "raised")


if __name__ == "__main__":
    main()
