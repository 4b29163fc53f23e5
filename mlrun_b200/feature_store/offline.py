"""Point-in-time correct training sets on the device: `get_offline_features` as one as-of join per feature set.

Plugin-API mirror of mlrun.feature_store.get_offline_features (feature_store/api.py:99, feature_vector.py:727) on the local
engine, whose BaseMerger.merge (retrieval/base.py:412-468) merges each feature set of the vector onto the entity frame with
pandas.merge_asof (retrieval/local_merger.py:29-81).  Storage is out of scope, as for the online table: a feature set's offline
frame is registered beside its `FeatureSet` mirror (`register_offline_frame`), which builds the set's device index once
(`b2s_pit_index_*`, include/b200serve.h).  A query sorts the entity rows by timestamp and joins every feature set in one
`b2s_pit_join_host` call; the host only assembles the columns the reference's frame has, with its names and dtypes.  A
vector with a `label_feature`, or a query without entity rows (the first feature set's own rows are then the frame the
others join), runs `b2s_pit_train_host` instead: the same join, then the rows the reference's merge and label `dropna`
keep are compacted on the device, and only those cross back.

Divergences (DESIGN.md §2): entity rows with equal timestamps keep their input order (pandas' quicksort may reorder them), and
of feature-set rows with equal (key, timestamp) the last in input order is taken.
"""

import ctypes as C

import numpy as np

from .. import _native as nat
from ..lowering import LoweringError
from ..serving.resolve import MLRunInvalidArgumentError
from .ingest import _INT_DTYPES
from .keys import _NAT, _UNIT_NS, _encode_keys, _key_kind, _ns

_OFFLINE = {}  # feature-set name -> OfflineSource
_NAN32 = 0x7FC00000
_NAN64 = 0x7FF8000000000000


class PitIndex:
    """b2s_pit index of one feature set: int64 keys, int64 nanosecond timestamps, 4- / 8-byte feature columns"""

    def __init__(self, keys, ts_ns, cols):
        nat.init()
        self._lib = nat.load()
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        ts_ns = np.ascontiguousarray(ts_ns, dtype=np.int64)
        cols = [np.ascontiguousarray(c) for c in cols]
        ptrs = (C.c_void_p * max(len(cols), 1))(*[c.ctypes.data for c in cols])
        widths = np.array([c.dtype.itemsize for c in cols] or [0], dtype=np.int32)
        self._h = C.c_void_p()
        nat.check(self._lib.b2s_pit_index_create(keys.ctypes.data, ts_ns.ctypes.data, len(keys), ptrs, nat._p(widths, C.c_int32),
                                                 len(cols), C.byref(self._h)))
        n_rows, n_keys, longest, cap = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        words = C.c_int32()
        nat.check(self._lib.b2s_pit_index_info(self._h, C.byref(n_rows), C.byref(n_keys), C.byref(longest), C.byref(words),
                                               C.byref(cap)))
        self.n_rows, self.n_keys, self.longest_run, self.row_words = n_rows.value, n_keys.value, longest.value, words.value

    def close(self):
        if self._h:
            self._lib.b2s_pit_index_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def pit_join(ts, sets, cols, with_stats=False):
    """ts: int64 ns [n] or None (input order kept); sets: [(PitIndex, int64 keys [n], asof, [(src_word, dtype, miss bits)])];
    cols: entity arrays [n] (1, 2, 4 or 8 bytes) -> (order int64 [n], [(outputs, ts_out, found bool)] per set, permuted cols,
    misses per set)"""
    lib = nat.init()
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.int64)
    keep = []  # arrays the descriptors point into
    c_sets = (nat.PitSet * max(len(sets), 1))()
    results = []
    for i, (index, keys, asof, outs) in enumerate(sets):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        arrays = [np.empty(n, dtype=dt) for _w, dt, _m in outs]
        ts_out, found = np.empty(n, dtype=np.int64), np.empty(n, dtype=np.uint8)
        descs = (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, a.ctypes.data)
                                                   for (w, dt, m), a in zip(outs, arrays)])
        keep += [keys, descs]
        c_sets[i] = nat.PitSet(index._h, keys.ctypes.data, int(asof), len(outs), descs, ts_out.ctypes.data, found.ctypes.data)
        results.append((arrays, ts_out, found))
    srcs = [np.ascontiguousarray(c) for c in cols]
    dsts = [np.empty_like(c) for c in srcs]
    c_cols = (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(s.ctypes.data, d.ctypes.data, s.dtype.itemsize) for s, d in zip(srcs, dsts)])
    order = np.empty(n, dtype=np.int64)
    miss = np.zeros(max(len(sets), 1), dtype=np.uint64)
    stats = nat.Stats()
    nat.check(lib.b2s_pit_join_host(None if ts is None else ts.ctypes.data, n, c_sets, len(sets), c_cols, len(cols), order.ctypes.data,
                                    miss.ctypes.data, C.byref(stats)))
    res = (order, [(a, t, f.view(bool)) for a, t, f in results], dsts, miss[:len(sets)])
    return res + (stats.as_dict(),) if with_stats else res


def pit_train(ts, sets, cols, label, with_stats=False):
    """pit_join, keeping only the rows of a training set (b2s_pit_train_host): those every exact-key set matched and, with
    label = (set index, or -1 for an entity column; output or column index; nat.PIT_LABEL_*), those with a label ->
    (order, [(outputs, ts_out, found)] per set, permuted cols, misses per set among the rows the exact-key sets before it
    matched), every array holding the kept rows; with_stats adds {sort_ms, join_ms, compact_ms, kept, **stats}"""
    lib = nat.init()
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.int64)
    keep = []  # arrays the descriptors point into
    c_sets = (nat.PitSet * max(len(sets), 1))()
    results = []
    for i, (index, keys, asof, outs) in enumerate(sets):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        arrays = [np.empty(n, dtype=dt) for _w, dt, _m in outs]
        ts_out, found = np.empty(n, dtype=np.int64), np.empty(n, dtype=np.uint8)
        descs = (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, a.ctypes.data)
                                                   for (w, dt, m), a in zip(outs, arrays)])
        keep += [keys, descs]
        c_sets[i] = nat.PitSet(index._h, keys.ctypes.data, int(asof), len(outs), descs, ts_out.ctypes.data, found.ctypes.data)
        results.append((arrays, ts_out, found))
    srcs = [np.ascontiguousarray(c) for c in cols]
    dsts = [np.empty_like(c) for c in srcs]
    c_cols = (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(s.ctypes.data, d.ctypes.data, s.dtype.itemsize) for s, d in zip(srcs, dsts)])
    c_label = None if label is None else C.byref(nat.PitLabel(*label))
    order = np.empty(n, dtype=np.int64)
    miss = np.zeros(max(len(sets), 1), dtype=np.uint64)
    kept = C.c_int64()
    phase = (C.c_float * 3)()
    stats = nat.Stats()
    nat.check(lib.b2s_pit_train_host(None if ts is None else ts.ctypes.data, n, c_sets, len(sets), c_cols, len(cols), c_label,
                                     order.ctypes.data, miss.ctypes.data, C.byref(kept), phase, C.byref(stats)))
    k = kept.value
    res = (order[:k], [([a[:k] for a in arr], t[:k], f[:k].view(bool)) for arr, t, f in results], [d[:k] for d in dsts],
           miss[:len(sets)])
    return res + (dict(sort_ms=phase[0], join_ms=phase[1], compact_ms=phase[2], kept=k, **stats.as_dict()),) if with_stats else res


def pit_train_pack(ts, sets, cols, label, feats, label_vec, dtype):
    """pit_train's rows packed on the device (b2s_pit_train_pack): feats [(set index or -1, output or column index,
    bytes, nat.PIT_FEAT_*)] are the matrix columns, label_vec the label vector's source (or None), dtype float32 /
    float64 -> (features [kept, F], label [kept] or None, order [kept]: nat.DeviceArray, {sort_ms, join_ms, compact_ms,
    pack_ms, kept, **stats})"""
    lib = nat.init()
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.int64)
    keep = []  # arrays the descriptors point into
    c_sets = (nat.PitSet * max(len(sets), 1))()
    for i, (index, keys, asof, outs) in enumerate(sets):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        descs = (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, None) for w, dt, m in outs])
        keep += [keys, descs]
        c_sets[i] = nat.PitSet(index._h, keys.ctypes.data, int(asof), len(outs), descs, None, None)
    srcs = [np.ascontiguousarray(c) for c in cols]
    c_cols = (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(s.ctypes.data, None, s.dtype.itemsize) for s in srcs])
    c_label = None if label is None else C.byref(nat.PitLabel(*label))
    c_feats = (nat.PitFeat * max(len(feats), 1))(*[nat.PitFeat(*f) for f in feats])
    c_vec = None if label_vec is None else C.byref(nat.PitFeat(*label_vec))
    out = nat.PitTensors()
    phase = (C.c_float * 4)()
    stats = nat.Stats()
    nat.check(lib.b2s_pit_train_pack(None if ts is None else ts.ctypes.data, n, c_sets, len(sets), c_cols, len(cols), c_label,
                                     c_feats, len(feats), c_vec, np.dtype(dtype).itemsize, C.byref(out), phase, C.byref(stats)))
    k = out.kept
    features = nat.DeviceArray(out.features, (k, len(feats)), dtype)
    order = nat.DeviceArray(out.order, (k,), np.int64)
    y = None if label_vec is None else nat.DeviceArray(out.label, (k,), _label_dtype(label_vec))
    return features, y, order, dict(sort_ms=phase[0], join_ms=phase[1], compact_ms=phase[2], pack_ms=phase[3], kept=k,
                                    **stats.as_dict())


def _label_dtype(label_vec):
    """the label vector's dtype for its source (set, output, bytes, kind): floats keep their width, ints become int64"""
    _s, _o, width, kind = label_vec
    return {nat.PIT_FEAT_FLOAT: np.float32 if width == 4 else np.float64, nat.PIT_FEAT_BOOL: np.bool_}.get(kind, np.int64)


class TrainingTensors:
    """a training set where the device built it: `features` [rows, F] (C order) and `label` [rows] (None without a label
    feature) as device arrays that any CUDA framework takes without a copy (`__cuda_array_interface__`, `__dlpack__`),
    `order` [rows] the entity-frame row of each, `columns` the F feature names; `rows` and `stats` are the launch's"""

    def __init__(self, features, label, order, columns, rows, stats):
        self.features, self.label, self.order = features, label, order
        self.columns, self.rows, self.stats = list(columns), rows, stats


class OfflineSource:
    """one feature set's offline frame, registered with its device index (built once)"""

    def __init__(self, featureset, frame):
        self.featureset = featureset
        self.name = featureset.name
        self.entities = [e.name for e in featureset.entities]
        self.timestamp_key = featureset.timestamp_key
        if frame.index.names[0]:
            frame = frame.reset_index()
        missing = [k for k in self.entities + ([self.timestamp_key] if self.timestamp_key else []) if k not in frame.columns]
        if missing:
            raise MLRunInvalidArgumentError(f"feature set {self.name}: the offline frame has no column {missing[0]!r}")
        if not self.entities:
            raise LoweringError(f"feature set {self.name} has no entities: only keyed feature sets are joined on the device")
        self.frame = frame
        self.key_kind = _key_kind(frame, self.entities, f"feature set {self.name}")
        keys = _encode_keys(frame, self.entities, self.key_kind, f"feature set {self.name}")
        if self.key_kind == "str":
            strings = frame[self.entities[0]].to_numpy()
            if len(np.unique(keys)) != len(set(strings.tolist())):
                raise MLRunInvalidArgumentError(f"feature set {self.name}: two entity keys share a 64-bit hash")
        if self.timestamp_key:
            ts_ns, _unit = _ns(frame[self.timestamp_key], f"feature set {self.name} timestamp {self.timestamp_key!r}")
            self.has_nat = bool((ts_ns == _NAT).any())
            # the coarsest unit every timestamp is a whole number of: a query whose timestamps are coarser would round them
            self.ts_factor = max((f for f in _UNIT_NS.values() if not (ts_ns[ts_ns != _NAT] % f).any()), default=1)
        else:
            ts_ns, self.has_nat, self.ts_factor = np.zeros(len(frame), dtype=np.int64), False, 10**9
        self.features, cols, word = {}, [], 0
        for name in frame.columns:
            if name in self.entities or name == self.timestamp_key:
                continue
            a = frame[name].to_numpy()
            s = str(frame[name].dtype)
            if s == "float32":
                stored, miss = a, _NAN32
            elif s == "float64":
                stored, miss = a, _NAN64
            elif s in _INT_DTYPES:
                stored, miss = a.astype(np.int32), 0
            elif s.startswith("datetime64") and getattr(frame[name].dtype, "tz", None) is None:
                stored, miss = a.view(np.int64), _NAT
            else:
                self.features[name] = (None, s, None)  # refused when a vector selects it
                continue
            self.features[name] = (word, s, miss)
            cols.append(stored)
            word += stored.dtype.itemsize // 4
        self.index = PitIndex(keys, ts_ns, cols)

    def close(self):
        self.index.close()


def register_offline_frame(featureset, frame):
    """hand over a feature set's offline rows (the frame its targets would hold); the device index is built here"""
    old = _OFFLINE.pop(featureset.name, None)
    if old is not None:
        old.close()
    src = OfflineSource(featureset, frame)
    _OFFLINE[featureset.name] = src
    return src


class FeatureVector:
    """mlrun.feature_store.FeatureVector (feature_vector.py): a name and features "set.feature [as alias]" / "set.*\""""

    def __init__(self, name=None, features=None, label_feature=None, description=None, with_indexes=None, join_graph=None,
                 relations=None):
        self.name = name
        self.features = list(features or [])
        self.label_feature = label_feature
        self.description = description
        self.with_indexes = with_indexes
        self.join_graph = join_graph
        self.relations = relations


class OfflineVectorResponse:
    """feature_vector.py OfflineVectorResponse: the training set as ordered columns (`columns`, in the frame's row order)"""

    def __init__(self, columns, index_columns):
        self.columns = columns
        self._index_columns = index_columns

    @property
    def status(self):
        return "completed"

    def to_dataframe(self, to_pandas=True):
        import pandas as pd

        frame = pd.DataFrame(dict(self.columns), copy=False)
        if self._index_columns:
            frame = frame.set_index(self._index_columns)
        return frame


def _parse(vector, label=None):
    """features, then the label feature (set, feature) -> {set: [(feature, alias)]} in vector order; a set's "*" skips its
    label (feature_vector.py:645-681)"""
    fields = {}
    for spec in vector.features + ([f"{label[0]}.{label[1]}"] if label else []):
        spec, alias = spec.split(" as ", 1) if " as " in spec else (spec, None)
        if "." not in spec:
            raise MLRunInvalidArgumentError(f"feature {spec!r} must be named <feature set>.<feature>")
        name, feat = spec.strip().split(".", 1)
        if name not in _OFFLINE:
            raise MLRunInvalidArgumentError(f"feature set {name!r} has no registered offline frame (register_offline_frame)")
        src = _OFFLINE[name]
        feats = [f for f in src.features if not (label and (name, f) == label)] if feat == "*" else [feat]
        for f in feats:
            if f not in src.features:
                raise MLRunInvalidArgumentError(f"feature {f!r} is not in feature set {name}")
            if src.features[f][0] is None:
                raise LoweringError(f"feature {name}.{f} has dtype {src.features[f][1]}: the device joins float32, float64, (u)int8/16/32, "
                                    "bool and datetime64 features")
            fields.setdefault(name, []).append((f, alias.strip() if alias else None))
    if not fields:
        raise MLRunInvalidArgumentError("No features in vector. Make sure to infer the schema on all the feature sets first")
    return fields


def _restore(values, dtype, found, missed):
    """a gathered column in the reference's dtype: unchanged when `found` is None or the set missed no row of the merged
    frame (`missed` False: rows an earlier inner join removed do not count); with a miss, ints become float64 and bool
    object, with NaN where `found` is False (float32, float64 and datetime64 columns carry NaN / NaT already)"""
    if dtype.startswith("datetime64"):
        return values.view(dtype)
    if dtype in ("float32", "float64"):
        return values
    if found is None or not missed:
        return values.astype(dtype)
    out = values.astype(bool).astype(object) if dtype == "bool" else values.astype(np.float64)
    out[~found] = np.nan
    return out


class _Query:
    """a vector's query, planned (`_plan_query`): what the device is asked and what the host names"""


def _plan_query(vector, entity_rows=None, entity_timestamp_column=None, target=None, run_config=None, drop_columns=None,
                start_time=None, end_time=None, with_indexes=False, update_stats=False, engine=None, engine_args=None, query=None,
                order_by=None, spark_service=None, timestamp_for_filtering=None, additional_filters=None):
    """the one planner of `get_offline_features` and `get_offline_tensors`: refusals, the parsed fields and label, the
    entity-less spine, the join of each set, the entity timestamps and the device descriptors"""
    if entity_rows is None and entity_timestamp_column is not None:  # api.py:228-232
        raise MLRunInvalidArgumentError("entity_timestamp_column param can not be specified without entity_rows param")
    if engine not in (None, "local"):
        raise LoweringError(f"engine {engine!r}: only the local engine's merge runs on the device")
    if start_time is not None or end_time is not None or timestamp_for_filtering is not None:
        raise LoweringError("start_time / end_time / timestamp_for_filtering are storage filters: not lowered")
    if query is not None or order_by is not None or additional_filters is not None:
        raise LoweringError("query / order_by / additional_filters are not lowered")
    if target is not None:
        raise LoweringError("targets are storage (out of scope): the training set is returned")
    if drop_columns is not None or update_stats or run_config is not None or spark_service is not None:
        raise LoweringError("drop_columns / update_stats / run_config / spark_service are not lowered")
    if getattr(vector, "join_graph", None) is not None or getattr(vector, "relations", None):
        raise LoweringError("join graphs and relations between feature sets are not lowered: every set joins the entity frame")
    label = None
    if getattr(vector, "label_feature", None):
        spec = vector.label_feature.split(" as ", 1)[0].strip()
        if "." not in spec:
            raise MLRunInvalidArgumentError(f"label feature {spec!r} must be named <feature set>.<feature>")
        label = tuple(spec.split(".", 1))
    drop_indexes = not (vector.with_indexes or with_indexes)
    fields = _parse(vector, label)
    spine_alias, spine_features = {}, []
    entity_less = entity_rows is None
    if entity_less:
        # the first set's own rows are the frame the others join (base.py:202-216, 268-285, 427-428): its entities, its
        # timestamp key and its selected features renamed <feature>_<set>
        spine_name = next(iter(fields))
        spine = _OFFLINE[spine_name]
        for name in fields:
            if set(_OFFLINE[name].entities) != set(spine.entities):
                raise LoweringError(f"feature set {name} is keyed by {_OFFLINE[name].entities}, the first set by {spine.entities}: "
                                    "relations between differently keyed feature sets are not lowered")
        head = spine.entities + ([spine.timestamp_key] if spine.timestamp_key else [])
        entity_rows = spine.frame[head + [f for f, _a in fields[spine_name]]].copy(deep=False)
        spine_features = [f"{f}_{spine_name}" for f, _a in fields[spine_name]]
        entity_rows.columns = head + spine_features
        entity_rows = entity_rows.reset_index(drop=True)
        entity_timestamp_column = spine.timestamp_key
        spine_alias = dict(([(c, c) for c in head] if not drop_indexes else []) +
                           [(f"{f}_{spine_name}", a or f) for f, a in fields.pop(spine_name)])
        index_columns = list(spine.entities)
    else:
        index_columns = []
        if entity_rows.index.names[0]:
            entity_rows = entity_rows.reset_index()
    n = len(entity_rows)
    names = [str(c) for c in entity_rows.columns]
    if len(set(names)) != len(names):
        raise LoweringError("duplicate column names in the entity frame")

    # the join of each set (base.py:430-460): as-of when it has a timestamp key and an entity timestamp column is known
    entity_ts = entity_timestamp_column
    plan, ts_col = [], entity_ts
    for name in fields:
        src = _OFFLINE[name]
        missing = [k for k in src.entities if k not in entity_rows.columns]
        if missing:
            raise LoweringError(f"feature set {name}: the entity frame has no key column {missing[0]!r} (relations between "
                                "differently keyed feature sets are not lowered)")
        asof = bool(src.timestamp_key and ts_col)
        if asof and ts_col != entity_ts:
            raise LoweringError(f"feature set {name} would join as-of on another feature set's timestamp {ts_col!r}: pass "
                                "entity_timestamp_column")
        if not asof and src.index.longest_run > 1:
            raise LoweringError(f"feature set {name} joins on its keys alone and has several rows per key: not lowered")
        plan.append((name, src, asof))
        ts_col = ts_col or src.timestamp_key
    any_asof = any(a for _n, _s, a in plan)
    ts_ns = unit = None
    if any_asof:
        if entity_ts not in entity_rows.columns:
            raise KeyError(entity_ts)
        ts_ns, unit = _ns(entity_rows[entity_ts], f"entity timestamp {entity_ts!r}")
        if (ts_ns == _NAT).any():
            raise ValueError("Merge keys contain null values on left side")
        for name, src, asof in plan:
            if asof and src.has_nat:
                raise ValueError("Merge keys contain null values on right side")
            if asof and src.ts_factor < _UNIT_NS[unit]:
                raise LoweringError(f"feature set {name}: timestamps finer than the entity column's unit {unit!r} would be "
                                    "rounded by the reference's cast: not lowered")

    # device call: every set's selected words, its timestamps and found flags; numeric entity columns permuted alongside
    sets = []
    for name, src, asof in plan:
        kind = _key_kind(entity_rows, src.entities, f"entity keys of {name}")
        if kind != src.key_kind:
            raise LoweringError(f"feature set {name}: entity keys are {kind}, the set's are {src.key_kind}")
        keys = _encode_keys(entity_rows, src.entities, kind, f"entity keys of {name}")
        outs = []
        for f, _a in fields[name]:
            word, s, miss = src.features[f]
            outs.append((word, np.int64 if s.startswith("datetime64") else np.float64 if s == "float64" else np.float32 if s == "float32"
                         else np.int32, miss))
        sets.append((src.index, keys, asof, outs))
    dev_cols = [c for c in entity_rows.columns if entity_rows[c].dtype.kind in "iufMb" and getattr(entity_rows[c].dtype, "tz", None) is None
                and isinstance(entity_rows[c].dtype, np.dtype)]
    arrays = [entity_rows[c].to_numpy() for c in dev_cols]
    dev_label = None
    if label is not None:  # the label's place on the device: an output of its set, or the spine's own column
        lname, lfeat = label
        ldtype = _OFFLINE[lname].features[lfeat][1]
        kind = nat.PIT_LABEL_NAN if ldtype.startswith("float") else nat.PIT_LABEL_NAT if ldtype.startswith("datetime64") else \
            nat.PIT_LABEL_FOUND
        if lname in fields:
            s_i = [name for name, _s, _a in plan].index(lname)
            dev_label = (s_i, max(j for j, (f, _a) in enumerate(fields[lname]) if f == lfeat), kind)
        else:
            dev_label = (-1, dev_cols.index(f"{lfeat}_{lname}"), kind)
    q = _Query()
    q.fields, q.label, q.dev_label, q.plan, q.sets = fields, label, dev_label, plan, sets
    q.entity_rows, q.entity_ts, q.ts_col, q.ts_ns, q.unit, q.n = entity_rows, entity_ts, ts_col, ts_ns, unit, n
    q.dev_cols, q.arrays, q.spine_alias, q.spine_features = dev_cols, arrays, spine_alias, spine_features
    q.index_columns, q.entity_less, q.drop_indexes = index_columns, entity_less, drop_indexes
    q.train = label is not None or entity_less
    return q


def _layout(q):
    """the training frame's columns by name alone -> ([(name, source)] in frame order, index columns); a source is
    ("entity", entity column), ("ts", set) or ("out", set, output)"""
    # the merged frame, set by set (local_merger.py:58-66 / 93-100): right columns after the left ones, the keys and an
    # equally named timestamp once, colliding names suffixed `_<set>_` (then dropped)
    cols = {c: ("entity", c) for c in q.entity_rows.columns}
    merge_drop = []
    alias = dict(q.spine_alias)
    for s_i, (name, src, asof) in enumerate(q.plan):
        head = src.entities + ([src.timestamp_key] if src.timestamp_key else [])
        right = {}
        if src.timestamp_key and not (asof and src.timestamp_key == q.entity_ts):
            right[src.timestamp_key] = ("ts", s_i)
        for j, (f, _a) in enumerate(q.fields[name]):
            right[f"{f}_{name}"] = ("out", s_i, j)
        for c, v in right.items():
            out_name = c
            if c in cols:
                out_name = f"{c}_{name}_"
                if out_name not in merge_drop:
                    merge_drop.append(out_name)
            cols[out_name] = v
        new = [(c, c) for c in head] if not q.drop_indexes else []
        new += [(f"{f}_{name}", a or f) for f, a in q.fields[name]]
        alias.update(dict(new))

    # base.py:113-120, 253-254, 325-341: drop keys / timestamps unless with_indexes, rename to aliases
    index_columns = list(q.index_columns)
    drop = []
    for c in ([q.entity_ts] if q.drop_indexes and q.entity_ts else []):
        drop.append(c)
    if q.entity_less and q.drop_indexes:
        drop += index_columns
    for name, src, _asof in q.plan:
        if q.drop_indexes and src.timestamp_key:
            drop.append(src.timestamp_key)
        for k in src.entities:
            if k not in index_columns:
                index_columns.append(k)
            if q.drop_indexes:
                drop.append(k)
    drop += merge_drop
    if not q.drop_indexes and q.ts_col and q.ts_col not in alias.values():
        alias[q.ts_col] = q.ts_col
    result, names = [], set()
    for c, v in cols.items():
        new = alias.get(c, c)
        if new in drop:
            continue
        if new in names:
            raise LoweringError(f"two columns of the training set are named {new!r}")
        result.append((new, v))
        names.add(new)
    if q.drop_indexes or not all(k in names for k in index_columns):
        index_columns = []
    return result, index_columns


def get_offline_features(feature_vector, entity_rows=None, entity_timestamp_column=None, target=None, run_config=None,
                         drop_columns=None, start_time=None, end_time=None, with_indexes=False, update_stats=False, engine=None,
                         engine_args=None, query=None, order_by=None, spark_service=None, timestamp_for_filtering=None,
                         additional_filters=None):
    """feature_store/api.py:99 on the local engine: the training frame of `feature_vector` for `entity_rows`, point-in-time
    correct per feature set.  What the device does not run is refused with LoweringError (there is no pandas fallback)."""
    q = _plan_query(feature_vector, entity_rows, entity_timestamp_column, target=target, run_config=run_config,
                    drop_columns=drop_columns, start_time=start_time, end_time=end_time, with_indexes=with_indexes,
                    update_stats=update_stats, engine=engine, engine_args=engine_args, query=query, order_by=order_by,
                    spark_service=spark_service, timestamp_for_filtering=timestamp_for_filtering,
                    additional_filters=additional_filters)
    sets, arrays = q.sets, q.arrays
    if not q.n:
        order, joined, permuted, miss = (
            np.zeros(0, np.int64), [([np.zeros(0, dt) for _w, dt, _m in s[3]], np.zeros(0, np.int64), np.zeros(0, bool)) for s in sets],
            [a[:0] for a in arrays], np.zeros(len(sets), np.uint64))
    elif q.train:
        order, joined, permuted, miss = pit_train(q.ts_ns, sets, arrays, q.dev_label)
    else:
        order, joined, permuted, _miss = pit_join(q.ts_ns, sets, arrays)
    moved = dict(zip(q.dev_cols, permuted))
    layout, index_columns = _layout(q)

    # the rows every exact-key set matched; per set, whether it missed a row of the merged frame at its place in the merge
    alive = np.ones(len(order), dtype=bool)
    missed = []
    for s_i, ((_name, _src, asof), (_vals, _ts_out, found)) in enumerate(zip(q.plan, joined)):
        missed.append(miss[s_i] > 0 if q.train else not found[alive].all())
        if not asof:
            alive &= found
    result = {}
    for new, source in layout:
        if source[0] == "entity":
            c = source[1]
            if c in moved:
                v = moved[c]
                v = v.view(q.entity_rows[c].dtype) if v.dtype != q.entity_rows[c].dtype else v
            else:  # strings, categories, objects: permuted on the host in the device's order
                v = q.entity_rows[c].take(order).reset_index(drop=True).array
        elif source[0] == "ts":
            name, src, asof = q.plan[source[1]]
            ts_out = joined[source[1]][1]
            # as-of: cast to the entity column's unit (base.py:389-410); exact: the set's own unit
            tdt = np.dtype(f"datetime64[{q.unit}]") if asof else src.frame[src.timestamp_key].dtype
            v = np.where(ts_out == _NAT, _NAT, ts_out // _UNIT_NS[np.datetime_data(tdt)[0]]).view(tdt)
        else:
            s_i, j = source[1], source[2]
            name, src, asof = q.plan[s_i]
            vals, _ts_out, found = joined[s_i]
            v = _restore(vals[j], src.features[q.fields[name][j][0]][1], found if asof else None, missed[s_i])
        result[new] = v[alive] if not alive.all() else v
    return OfflineVectorResponse(result, index_columns)


def _feat_kind(dtype):
    """a device source's dtype -> (bytes, nat.PIT_FEAT_*) as the device holds it"""
    dtype = np.dtype(dtype)
    kind = {"f": nat.PIT_FEAT_FLOAT, "i": nat.PIT_FEAT_INT, "u": nat.PIT_FEAT_UINT, "b": nat.PIT_FEAT_BOOL}[dtype.kind]
    return dtype.itemsize, kind


def get_offline_tensors(feature_vector, entity_rows=None, entity_timestamp_column=None, dtype="float32", **options):
    """the training set of `get_offline_features(feature_vector, entity_rows, entity_timestamp_column, **options)` left in
    device memory: row i of `features`, `label` and `order` is row i of that call's `to_dataframe()`; the features are its
    columns without the label, the entity frame's own columns, the keys and the timestamps, converted as
    `to_numpy(dtype)` converts them (a missing value is NaN, bool 0 / 1).  Refuses what `get_offline_features` refuses,
    with the same messages, and datetime features, which a matrix of numbers cannot hold."""
    if np.dtype(dtype) not in (np.float32, np.float64):
        raise ValueError(f"dtype {dtype!r}: the feature matrix is float32 or float64")
    dtype = np.dtype(dtype)
    q = _plan_query(feature_vector, entity_rows, entity_timestamp_column, **options)
    layout, _index_columns = _layout(q)
    label_source = None
    if q.dev_label is not None:
        s_i, j, _kind = q.dev_label
        label_source = ("out", s_i, j) if s_i >= 0 else ("entity", q.dev_cols[j])
    spine = set(q.spine_features)
    picked = [(name, source) for name, source in layout if source != label_source and
              (source[0] == "out" or (source[0] == "entity" and source[1] in spine))]

    # each matrix column's source on the device: a set's output as the index stores it, or a spine column as the frame has it
    used = [c for c in q.dev_cols if c in spine or (label_source is not None and ("entity", c) == label_source)]
    arrays = [q.arrays[q.dev_cols.index(c)] for c in used]

    def device_source(name, source, what):
        if source[0] == "out":
            s_i, j = source[1], source[2]
            pname, src, _asof = q.plan[s_i]
            stored = src.features[q.fields[pname][j][0]][1]
            if stored.startswith("datetime64"):
                raise LoweringError(f"{what} {name!r} is a {stored} column: a matrix of numbers has no place for it (drop it from "
                                    "the vector)")
            width, kind = _feat_kind(stored if stored in ("float32", "float64") else np.int32)
            return (s_i, j, width, nat.PIT_FEAT_BOOL if stored == "bool" else kind)
        col = q.entity_rows[source[1]]
        if col.dtype.kind == "M":
            raise LoweringError(f"{what} {name!r} is a {col.dtype} column: a matrix of numbers has no place for it (drop it from "
                                "the vector)")
        return (-1, used.index(source[1])) + _feat_kind(col.dtype)

    feats = [device_source(name, source, "feature") for name, source in picked]
    label_vec = None
    if label_source is not None:
        label_vec = device_source(f"{q.label[0]}.{q.label[1]}", label_source, "label")
    dev_label = q.dev_label
    if dev_label is not None and dev_label[0] < 0:
        dev_label = (-1, used.index(label_source[1]), dev_label[2])
    features, label, order, stats = pit_train_pack(q.ts_ns, q.sets, arrays, dev_label, feats, label_vec, dtype)
    return TrainingTensors(features, label, order, [name for name, _s in picked], stats["kept"], stats)
