"""Training sets restated (pandas, no mlrun, tests only): BaseMerger.start / _generate_offline_vector
(mlrun/feature_store/retrieval/base.py:78-368) for a vector with a label feature and / or without entity rows, around the
merge of oracle/offline.py.  Pinned against the real merger by tests/golden/ref_training_set.pkl.xz and
tests/golden/diff_training_set.py.

* the label feature is appended to the vector's features, and a "*" over the label's own set skips it
  (feature_vector.py:645-681);
* without entity rows, the first set's frame is the one the others are merged onto (base.py:202-216, merge at :427-428),
  and its timestamp key is their as-of column;
* `dropna(subset=[label])` runs after the merge, the renames and the drops (base.py:343-346).
"""

from oracle.offline import FeatureSetStub, merge


def parse_features(features, frames, label_feature=None):
    """["set.feature", "set.feature as alias", "set.*"], then the label feature -> {set: [(feature, alias or None)]} in
    vector order; "*" skips the timestamp key and, in the label's set, the label"""
    fields = {}
    label = tuple(label_feature.split(" as ", 1)[0].strip().split(".", 1)) if label_feature else None
    for spec in list(features) + ([label_feature] if label_feature else []):
        spec, alias = (spec.split(" as ", 1) + [None])[:2] if " as " in spec else (spec, None)
        name, feat = spec.strip().split(".", 1)
        entities, ts, frame = frames[name]
        cols = [c for c in frame.columns if c not in entities and c != ts and (name, c) != label] if feat == "*" else [feat]
        fields.setdefault(name, []).extend((c, alias.strip() if alias else None) for c in cols)
    return fields


def get_offline_features(frames, features, entity_rows, entity_timestamp_column=None, with_indexes=False, label_feature=None):
    """frames: {set: (entity column names, timestamp key or None, offline frame)} -> the training frame"""
    if entity_rows is None and entity_timestamp_column is not None:  # api.py:228-232
        raise ValueError("entity_timestamp_column param can not be specified without entity_rows param")
    drop_indexes = not with_indexes
    drop, index_columns, alias = [], [], {}

    def append_drop(key):
        if key and key not in drop:
            drop.append(key)

    fields = parse_features(features, frames, label_feature)
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
    if entity_rows is not None and entity_rows.index.names[0]:
        entity_rows = entity_rows.reset_index()
    featuresets, dfs, keys = [], [], []
    for name, columns in fields.items():
        entities, ts, frame = frames[name]
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
    if entity_rows is None:
        entity_rows, entity_timestamp_column = dfs.pop(0), featuresets.pop(0).spec.timestamp_key
        keys.pop(0)
    result, merge_drop, result_ts = merge(entity_rows, entity_timestamp_column, featuresets, dfs, keys)
    for col in merge_drop:
        append_drop(col)
    if not drop_indexes and result_ts and result_ts not in alias.values():
        alias[result_ts] = result_ts
    result = result.rename(columns=alias)
    result = result.drop(columns=drop, errors="ignore")
    if label_feature:
        result = result.dropna(subset=[label_feature.split(" as ", 1)[0].strip().split(".", 1)[1]])
    if index_columns and not drop_indexes:
        if all(k in result.columns for k in index_columns):
            result = result.set_index(index_columns)
    else:
        result = result.reset_index(drop=True)
    return result
