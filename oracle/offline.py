"""Point-in-time training sets: the local engine's offline merge restated (pandas, no mlrun).

`merge` is BaseMerger.merge (mlrun/feature_store/retrieval/base.py:412-468) with LocalFeatureMerger's `_asof_join` /
`_join` (retrieval/local_merger.py:29-104): feature-set frames are merged onto the entity frame in order, as-of (pandas
merge_asof, backward, exact matches allowed, `by` the keys) when the set has a timestamp key and an entity timestamp
column is known, else on the keys (pd.merge, inner).  It is pinned against the real classes by
tests/golden/ref_offline.pkl.xz.

`get_offline_features` restates the column handling of BaseMerger.start / _generate_offline_vector (base.py:78-368) around
it for a vector whose feature sets all join on the entity frame: feature columns renamed `<feature>_<set>` for the merge,
then to their alias (or name); entity keys, timestamps and `_<set>_` suffix columns dropped unless `with_indexes`, where
the keys become the index.  A feature set's engine frame holds its entity columns, its timestamp key, then the selected
features in vector order.
"""

import re

import pandas as pd


class FeatureSetStub:
    """what merge() reads of a feature set: metadata.name, spec.timestamp_key"""

    def __init__(self, name, timestamp_key=None):
        import types

        self.metadata = types.SimpleNamespace(name=name)
        self.spec = types.SimpleNamespace(timestamp_key=timestamp_key)


def _normalize_timestamp_column(entity_ts, entity_df, fs_ts, fs_df):
    """base.py:389-410: the feature set's timestamps take the entity column's datetime64 unit"""
    want = entity_df[entity_ts].dtype.name
    if want != fs_df[fs_ts].dtype.name:
        fs_df[fs_ts] = fs_df[fs_ts].astype(want)
    return fs_df


def _asof_join(entity_df, entity_ts, name, fs_ts, fs_df, left_keys, right_keys, drop):
    index_not_in_entity = "index" not in entity_df.columns
    index_not_in_fs = "index" not in fs_df.columns
    entity_df = entity_df.copy()
    fs_df = fs_df.copy()
    entity_df[entity_ts] = pd.to_datetime(entity_df[entity_ts])
    fs_df[fs_ts] = pd.to_datetime(fs_df[fs_ts])
    entity_df.sort_values(by=entity_ts, inplace=True)
    fs_df.sort_values(by=fs_ts, inplace=True)
    fs_df = _normalize_timestamp_column(entity_ts, entity_df, fs_ts, fs_df)
    merged = pd.merge_asof(entity_df, fs_df, left_on=entity_ts, right_on=fs_ts, left_by=left_keys or None,
                           right_by=right_keys or None, suffixes=("", f"_{name}_"))
    for col in merged.columns:
        if re.findall(f"_{name}_$", col) and col not in drop:
            drop.append(col)
    if ("index" not in left_keys and "index" not in right_keys and index_not_in_entity and index_not_in_fs
            and "index" in merged.columns):
        merged.drop(columns="index", inplace=True)
    return merged


def _join(entity_df, name, fs_df, left_keys, right_keys, how, drop):
    merged = pd.merge(entity_df, fs_df, how=how, left_on=left_keys, right_on=right_keys, suffixes=("", f"_{name}_"))
    for col in merged.columns:
        if re.findall(f"_{name}_$", col) and col not in drop:
            drop.append(col)
    return merged


def merge(entity_df, entity_timestamp_column, featuresets, featureset_dfs, keys, join_type="inner"):
    """-> (merged frame, drop columns the merge added, the timestamp column the result carries)"""
    drop = []
    merged = entity_df
    for fs, fs_df, (left_keys, right_keys) in zip(featuresets, featureset_dfs, keys):
        ts = fs.spec.timestamp_key
        if ts and entity_timestamp_column:
            merged = _asof_join(merged, entity_timestamp_column, fs.metadata.name, ts, fs_df, left_keys, right_keys, drop)
        else:
            merged = _join(merged, fs.metadata.name, fs_df, left_keys, right_keys, join_type, drop)
        entity_timestamp_column = entity_timestamp_column or ts
    return merged, drop, entity_timestamp_column


def parse_features(features, frames):
    """["set.feature", "set.feature as alias", "set.*"] -> {set: [(feature, alias or None)]} in vector order"""
    fields = {}
    for spec in features:
        spec, alias = (spec.split(" as ", 1) + [None])[:2] if " as " in spec else (spec, None)
        name, feat = spec.strip().split(".", 1)
        entities, ts, frame = frames[name]
        cols = [c for c in frame.columns if c not in entities and c != ts] if feat == "*" else [feat]
        fields.setdefault(name, []).extend((c, alias.strip() if alias else None) for c in cols)
    return fields


def get_offline_features(frames, features, entity_rows, entity_timestamp_column=None, with_indexes=False):
    """frames: {set: (entity column names, timestamp key or None, offline frame)} -> the training frame"""
    drop_indexes = not with_indexes
    drop, index_columns, alias = [], [], {}

    def append_drop(key):
        if key and key not in drop:
            drop.append(key)

    fields = parse_features(features, frames)
    if drop_indexes and entity_timestamp_column:
        append_drop(entity_timestamp_column)
    for name in fields:
        entities, ts, _frame = frames[name]
        if drop_indexes:
            append_drop(ts)
        for key in entities:
            if key not in index_columns:
                index_columns.append(key)
            if drop_indexes:
                append_drop(key)
    if entity_rows.index.names[0]:
        entity_rows = entity_rows.reset_index()
    featuresets, dfs, keys = [], [], []
    for name, columns in fields.items():
        entities, ts, frame = frames[name]
        if drop_indexes:
            append_drop(ts)
        if frame.index.names[0]:
            frame = frame.reset_index()
        head = list(entities) + ([ts] if ts else [])
        df = frame[head + [c for c, _ in columns]].copy()
        df.columns = head + [f"{c}_{name}" for c, _ in columns]
        featuresets.append(FeatureSetStub(name, ts))
        dfs.append(df)
        keys.append((list(entities), list(entities)))
        new = [(c, c) for c in head] if not drop_indexes else []
        new += [(f"{c}_{name}", a or c) for c, a in columns]
        alias.update(dict(new))
    result, merge_drop, result_ts = merge(entity_rows, entity_timestamp_column, featuresets, dfs, keys)
    for col in merge_drop:
        append_drop(col)
    if not drop_indexes and result_ts and result_ts not in alias.values():
        alias[result_ts] = result_ts
    result = result.rename(columns=alias)
    result = result.drop(columns=drop, errors="ignore")
    if index_columns and not drop_indexes:
        if all(k in result.columns for k in index_columns):
            result = result.set_index(index_columns)
    else:
        result = result.reset_index(drop=True)
    return result
