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
from . import columnar
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
        self._info()

    @classmethod
    def device(cls, d_keys, d_ts, n, cols):
        """the index of n rows whose keys, timestamps and columns [(address, 4 or 8 bytes)] are in device memory
        (b2s_pit_index_create_device): nothing crosses to the host"""
        self = cls.__new__(cls)
        self._lib = nat.init()
        ptrs = (C.c_void_p * max(len(cols), 1))(*[a for a, _w in cols])
        widths = np.array([w for _a, w in cols] or [0], dtype=np.int32)
        self._h = C.c_void_p()
        nat.check(self._lib.b2s_pit_index_create_device(d_keys, d_ts, n, ptrs, nat._p(widths, C.c_int32), len(cols), C.byref(self._h)))
        self._info()
        return self

    def _info(self):
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
    n = len(ts) if ts is not None else len(cols[0]) if cols else len(sets[0][1]) if sets else 0
    ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.int64)
    keys = [np.ascontiguousarray(k, dtype=np.int64) for _ix, k, _a, _o in sets]
    srcs = [np.ascontiguousarray(c) for c in cols]
    return _train_pack("b2s_pit_train_pack", None if ts is None else ts.ctypes.data, n,
                       [(ix, k.ctypes.data, asof, outs) for (ix, _k, asof, outs), k in zip(sets, keys)],
                       [(c.ctypes.data, c.dtype.itemsize) for c in srcs], label, feats, label_vec, dtype)


def pit_train_pack_device(d_ts, n, sets, cols, label, feats, label_vec, dtype):
    """pit_train_pack over inputs in device memory (b2s_pit_train_pack_device): d_ts an address or None, each set's keys
    an address, cols [(address, bytes)]; nothing is uploaded"""
    return _train_pack("b2s_pit_train_pack_device", d_ts, n, sets, cols, label, feats, label_vec, dtype)


def _train_pack(entry, ts, n, sets, cols, label, feats, label_vec, dtype):
    """one b2s_pit_train_pack* call: ts, keys and column sources are addresses the entry point reads"""
    lib = nat.init()
    keep = []  # arrays the descriptors point into
    c_sets = (nat.PitSet * max(len(sets), 1))()
    for i, (index, keys, asof, outs) in enumerate(sets):
        descs = (nat.PitOut * max(len(outs), 1))(*[nat.PitOut(w, np.dtype(dt).itemsize, m, None) for w, dt, m in outs])
        keep.append(descs)
        c_sets[i] = nat.PitSet(index._h, keys, int(asof), len(outs), descs, None, None)
    c_cols = (nat.PitCol * max(len(cols), 1))(*[nat.PitCol(a, None, w) for a, w in cols])
    c_label = None if label is None else C.byref(nat.PitLabel(*label))
    c_feats = (nat.PitFeat * max(len(feats), 1))(*[nat.PitFeat(*f) for f in feats])
    c_vec = None if label_vec is None else C.byref(nat.PitFeat(*label_vec))
    out = nat.PitTensors()
    phase = (C.c_float * 4)()
    stats = nat.Stats()
    nat.check(getattr(lib, entry)(ts, n, c_sets, len(sets), c_cols, len(cols), c_label, c_feats, len(feats), c_vec,
                                  np.dtype(dtype).itemsize, C.byref(out), phase, C.byref(stats)))
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


class _Columns:
    """the columns of an entity frame or offline frame as the planner and the registration read them, filled from a pandas
    frame or from CUDA columns: `columns` (names in order), `dtypes` {name: dtype}, `n`, and each column's data -- the
    frame's (`frame`), or an acquirable `columnar.DeviceColumn` (`device`).  Keys are encoded and timestamps checked with
    numpy on the host side and by the kernels on the device side; what is refused is refused alike."""

    def __init__(self, columns, dtypes, n, frame=None, device=None):
        self.columns, self.dtypes, self.n = list(columns), dict(dtypes), int(n)
        self.frame, self.device = frame, device
        self.keys = {}  # (names, kind) -> encoded keys of a device frame
        self.profiles = {}  # name -> b2s_ts_profile_device counts of a device frame

    @classmethod
    def of_frame(cls, frame):
        if frame.index.names[0]:
            frame = frame.reset_index()
        # dtypes by position: a name that appears twice is refused by the planner, not by a lookup here
        return cls(frame.columns, dict(zip(frame.columns, frame.dtypes)), len(frame), frame=frame)

    @classmethod
    def of_device(cls, source, timestamp_names):
        """CUDA columns (a mapping, or a DeviceColumnBatch whose index columns come first, as reset_index() puts them);
        an int64 column named in `timestamp_names` is datetime64[ns].  Described, not acquired: nothing is read yet."""
        cols = columnar.device_columns(source)
        if len({c.n for c in cols.values()}) > 1:
            raise ValueError("All arrays must be of the same length")
        for name, c in cols.items():
            if str(c.dtype) == "int64" and name in timestamp_names:
                c.dtype = np.dtype("datetime64[ns]")
        n = next(iter(cols.values())).n if cols else 0
        return cls(cols, {k: c.dtype for k, c in cols.items()}, n, device=cols)

    @staticmethod
    def of(source, timestamp_names):
        if columnar.is_columnar(source) and columnar.is_device_source(source):
            return _Columns.of_device(source, timestamp_names)
        return _Columns.of_frame(source)

    def select(self, names, renamed):
        """columns `names`, renamed `renamed`, in that order (the entity-less spine); a device frame keeps its encoded keys
        under the new names (the set's own, made at registration).  Timestamps are profiled again by each query, as the
        host path checks its frame's each time."""
        if self.device is None:
            frame = self.frame[names].copy(deep=False)
            frame.columns = renamed
            return _Columns.of_frame(frame.reset_index(drop=True))
        new = dict(zip(names, renamed))
        out = _Columns(renamed, {new[c]: self.dtypes[c] for c in names}, self.n, device={new[c]: self.device[c] for c in names})
        out.keys = {(tuple(new[k] for k in ks), kind): v for (ks, kind), v in self.keys.items() if all(k in new for k in ks)}
        return out

    def to_host(self):
        """the same columns on the host (one copy each): what `get_offline_features` assembles its frame from"""
        if self.device is None:
            return self
        import pandas as pd

        return _Columns.of_frame(pd.DataFrame({c: self.device[c].numpy().view(self.dtypes[c]) for c in self.columns}, copy=False))

    def acquire(self, names):
        """-> {name: device address} of the named device columns, the library stream ordered behind their producers"""
        return {c: self.device[c].acquire().ptr for c in names}

    def release(self):
        if self.device is not None:
            for c in self.device.values():
                c.release()

    def key_kind(self, names, what):
        if self.device is not None:
            for k in names:
                if k in self.dtypes and self.dtypes[k].kind in "OSU":
                    raise LoweringError(f"{what}: key {k!r} of dtype {self.dtypes[k]} is a string key: there are no string "
                                        "columns on the device (hash them on the host)")
            return _key_kind({k: np.empty(0, self.dtypes[k]) for k in names}, names, what)
        return _key_kind(self.frame, names, what)

    def encode_keys(self, names, kind, what):
        """numpy int64 keys of a host frame; a DeviceArray of a device frame (b2s_keys_encode_device, once per key)"""
        if self.device is None:
            return _encode_keys(self.frame, names, kind, what)
        at = (tuple(names), kind)
        if at not in self.keys:
            lib = nat.init()
            keys = nat.DeviceArray(nat.darray_alloc(8 * self.n), (self.n,), np.int64)
            if self.n:
                ptrs = self.acquire(names)
                kc = (nat.KeyCol * len(names))(*[nat.KeyCol(ptrs[k], self.dtypes[k].itemsize, int(self.dtypes[k].kind == "i"))
                                                 for k in names])
                nat.check(lib.b2s_keys_encode_device(kc, len(names), self.n, keys.ptr, None))
            self.keys[at] = keys
        return self.keys[at]

    def timestamps(self, name, what, profile=True):
        """-> (int64 nanoseconds: a host array, or a device address), unit, [NaT, not whole us, ms, s] counts (a host
        frame without `profile`: [NaT] alone)"""
        if self.device is None:
            ts_ns, unit = _ns(self.frame[name], what)
            if not profile:
                return ts_ns, unit, [int((ts_ns == _NAT).sum())]
            real = ts_ns[ts_ns != _NAT]
            return ts_ns, unit, [len(ts_ns) - len(real)] + [int((real % f).any()) for f in (10**3, 10**6, 10**9)]
        self.timestamp_dtype(name, what)
        ptr = self.acquire([name])[name]
        if name not in self.profiles:
            counts = np.zeros(4, dtype=np.int64)
            nat.check(nat.init().b2s_ts_profile_device(ptr, self.n, nat._p(counts, C.c_int64), None))
            self.profiles[name] = [int(v) for v in counts]
        return ptr, "ns", self.profiles[name]

    def timestamp_dtype(self, name, what):
        """CUDA timestamps are int64 nanoseconds (datetime64[ns]); any other dtype is refused as `keys._ns` refuses it"""
        dt = self.dtypes[name]
        if dt != np.dtype("datetime64[ns]"):
            raise LoweringError(f"{what} has dtype {dt}: the as-of join takes tz-naive datetime64 timestamps")

    def array(self, name):
        """a column's data for the join: a numpy array, or a device address"""
        return self.frame[name].to_numpy() if self.device is None else self.acquire([name])[name]


def _ts_factor(counts):
    """the coarsest unit every timestamp is a whole number of (10^9 when there are none): a query whose timestamps are
    coarser would round them"""
    return next((f for f, c in zip((10**9, 10**6, 10**3), counts[:0:-1]) if not c), 1)


class OfflineSource:
    """one feature set's offline rows, registered with its device index (built once): a pandas frame, or CUDA columns
    that stay in HBM"""

    def __init__(self, featureset, frame):
        self.featureset = featureset
        self.name = featureset.name
        self.entities = [e.name for e in featureset.entities]
        self.timestamp_key = featureset.timestamp_key
        self.keys = None
        rows = _Columns.of(frame, {self.timestamp_key} if self.timestamp_key else set())
        missing = [k for k in self.entities + ([self.timestamp_key] if self.timestamp_key else []) if k not in rows.columns]
        if missing:
            raise MLRunInvalidArgumentError(f"feature set {self.name}: the offline frame has no column {missing[0]!r}")
        if not self.entities:
            raise LoweringError(f"feature set {self.name} has no entities: only keyed feature sets are joined on the device")
        self.rows = rows
        self.frame = rows.frame
        what = f"feature set {self.name}"
        self.key_kind = rows.key_kind(self.entities, what)
        if rows.device is not None:
            self._register_device(rows, what)
            return
        frame = rows.frame
        keys = rows.encode_keys(self.entities, self.key_kind, what)
        if self.key_kind == "str":
            strings = frame[self.entities[0]].to_numpy()
            if len(np.unique(keys)) != len(set(strings.tolist())):
                raise MLRunInvalidArgumentError(f"feature set {self.name}: two entity keys share a 64-bit hash")
        if self.timestamp_key:
            ts_ns, _unit, counts = rows.timestamps(self.timestamp_key, f"{what} timestamp {self.timestamp_key!r}")
            self.has_nat, self.ts_factor = counts[0] > 0, _ts_factor(counts)
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

    def _register_device(self, rows, what):
        """the index of CUDA columns, built where they are: keys encoded (kept as a library array, so that later writes to
        the caller's entity columns do not change the set), the timestamps profiled, narrow ints and bool widened to int32
        in temporaries; only counters come back"""
        self.features, plan, word, widen = {}, [], 0, []
        for name in rows.columns:
            if name in self.entities or name == self.timestamp_key:
                continue
            dt = rows.dtypes[name]
            s = str(dt)
            if s == "float32":
                width, miss = 4, _NAN32
            elif s == "float64":
                width, miss = 8, _NAN64
            elif s in _INT_DTYPES:
                width, miss = 4, 0
                if s != "int32":
                    widen.append(name)
            elif dt.kind == "M":
                width, miss = 8, _NAT
            else:
                self.features[name] = (None, s, None)  # refused when a vector selects it
                continue
            self.features[name] = (word, s, miss)
            plan.append((name, width))
            word += width // 4
        if self.timestamp_key:
            rows.timestamp_dtype(self.timestamp_key, f"{what} timestamp {self.timestamp_key!r}")  # refused before any call
        lib = nat.init()
        n = rows.n
        try:
            if self.timestamp_key:
                d_ts, _unit, counts = rows.timestamps(self.timestamp_key, f"{what} timestamp {self.timestamp_key!r}")
                self.has_nat, self.ts_factor = counts[0] > 0, _ts_factor(counts)
                zeros = None
            self.keys = rows.encode_keys(self.entities, self.key_kind, what)
            if not self.timestamp_key:
                zeros = nat.DeviceArray(nat.darray_alloc(8 * n, zero=True), (n,), np.int64)
                d_ts, self.has_nat, self.ts_factor = zeros.ptr, False, 10**9
            ptrs = rows.acquire([name for name, _w in plan])
            # 1- and 2-byte ints and bool as int32, in one convert launch into one temporary block
            pitch = (4 * n + 255) // 256 * 256
            temp = nat.DeviceArray(nat.darray_alloc(max(pitch * len(widen), 8)), (max(pitch * len(widen), 8),), np.uint8) \
                if widen else None
            kinds = {"int8": nat.CONV_I8_I32, "uint8": nat.CONV_U8_I32, "bool": nat.CONV_U8_I32, "int16": nat.CONV_I16_I32,
                     "uint16": nat.CONV_U16_I32}
            ops = []
            for j, name in enumerate(widen):
                ops.append(nat.Convert(ptrs[name], temp.ptr + j * pitch, kinds[str(rows.dtypes[name])], 0))
                ptrs[name] = temp.ptr + j * pitch
            if ops and n:
                nat.check(lib.b2s_cols_convert_device((nat.Convert * len(ops))(*ops), len(ops), n, None, 0, None))
            self.index = PitIndex.device(self.keys.ptr if n else None, d_ts if n else None, n,
                                         [(ptrs[name], width) for name, width in plan])
            del temp, zeros  # the build has synchronised: the temporaries go back now
        except BaseException:
            if self.keys is not None:
                self.keys.release()
            raise
        finally:
            rows.release()

    @property
    def ts_dtype(self):
        return self.rows.dtypes[self.timestamp_key]

    def close(self):
        index = getattr(self, "index", None)
        if index is not None:
            index.close()
        if self.keys is not None:
            self.keys.release()
        self.rows.keys, self.rows.profiles = {}, {}


def register_offline_frame(featureset, frame):
    """hand over a feature set's offline rows (the frame its targets would hold); the device index is built here.  `frame`
    is a pandas frame, or CUDA columns: a `columnar.DeviceColumnBatch` (`FeatureSet.ingest`'s result; its `index` holds the
    entity columns) or a mapping of CUDA columns, whose int64 `timestamp_key` column is nanoseconds.  The source registered
    from CUDA columns behaves as the one registered from the equal pandas frame, and its columns stay in HBM: only counters
    cross to the host."""
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
                order_by=None, spark_service=None, timestamp_for_filtering=None, additional_filters=None, on_host=False):
    """the one planner of `get_offline_features` and `get_offline_tensors`: refusals, the parsed fields and label, the
    entity-less spine, the join of each set, the entity timestamps and the device descriptors.  The entity frame is read
    through `_Columns`, from a pandas frame or from CUDA columns (`q.device`: then the timestamps, keys and columns of
    the device call are device addresses); `on_host` copies a spine registered from CUDA columns to the host first."""
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
        spine_features = [f"{f}_{spine_name}" for f, _a in fields[spine_name]]
        entity_rows = spine.rows.select(head + [f for f, _a in fields[spine_name]], head + spine_features)
        entity_timestamp_column = spine.timestamp_key
        spine_alias = dict(([(c, c) for c in head] if not drop_indexes else []) +
                           [(f"{f}_{spine_name}", a or f) for f, a in fields.pop(spine_name)])
        index_columns = list(spine.entities)
    else:
        index_columns = []
        entity_rows = _Columns.of(entity_rows, {entity_timestamp_column} if entity_timestamp_column else set())
    names = [str(c) for c in entity_rows.columns]
    if len(set(names)) != len(names):
        raise LoweringError("duplicate column names in the entity frame")
    if entity_less and on_host:
        entity_rows = entity_rows.to_host()
    n = entity_rows.n

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

    def set_refusals(unit):
        for name, src, asof in plan:
            if asof and src.has_nat:
                raise ValueError("Merge keys contain null values on right side")
            if asof and src.ts_factor < _UNIT_NS[unit]:
                raise LoweringError(f"feature set {name}: timestamps finer than the entity column's unit {unit!r} would be "
                                    "rounded by the reference's cast: not lowered")

    # CUDA columns: every refusal is raised before the first launch (the timestamp profile, a key encode), in the host's
    # order.  The one refusal that reads data, NaT on the left side, cannot come first: a key-kind refusal wins over it.
    key_error = None
    if entity_rows.device is not None:
        try:
            for name, src, _asof in plan:
                _entity_key_kind(entity_rows, name, src)
        except LoweringError as err:
            key_error = err
    if any_asof:
        if entity_ts not in entity_rows.columns:
            raise KeyError(entity_ts)
        if key_error is not None:
            entity_rows.timestamp_dtype(entity_ts, f"entity timestamp {entity_ts!r}")
            set_refusals("ns")
            raise key_error
        ts_ns, unit, counts = entity_rows.timestamps(entity_ts, f"entity timestamp {entity_ts!r}", profile=False)
        if counts[0]:
            raise ValueError("Merge keys contain null values on left side")
        set_refusals(unit)
    if key_error is not None:
        raise key_error

    # device call: every set's selected words, its timestamps and found flags; numeric entity columns permuted alongside
    sets = []
    for name, src, asof in plan:
        kind = _entity_key_kind(entity_rows, name, src)
        keys = entity_rows.encode_keys(src.entities, kind, f"entity keys of {name}")
        outs = []
        for f, _a in fields[name]:
            word, s, miss = src.features[f]
            outs.append((word, np.int64 if s.startswith("datetime64") else np.float64 if s == "float64" else np.float32 if s == "float32"
                         else np.int32, miss))
        sets.append((src.index, keys.ptr if entity_rows.device is not None else keys, asof, outs))
    dtypes = entity_rows.dtypes
    dev_cols = [c for c in entity_rows.columns if dtypes[c].kind in "iufMb" and getattr(dtypes[c], "tz", None) is None
                and isinstance(dtypes[c], np.dtype)]
    arrays = [entity_rows.array(c) for c in dev_cols]
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
    q.device = entity_rows.device is not None
    return q


def _entity_key_kind(entity_rows, name, src):
    kind = entity_rows.key_kind(src.entities, f"entity keys of {name}")
    if kind != src.key_kind:
        raise LoweringError(f"feature set {name}: entity keys are {kind}, the set's are {src.key_kind}")
    return kind


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
    correct per feature set.  What the device does not run is refused with LoweringError (there is no pandas fallback).
    Feature sets registered from CUDA columns are joined where their indexes are; without entity rows, a spine registered
    from CUDA columns has the columns the frame uses copied to the host once per call, since the result is a host frame.
    CUDA `entity_rows` are refused: `get_offline_tensors` builds the training set from them without leaving the device."""
    if entity_rows is not None and columnar.is_columnar(entity_rows) and columnar.is_device_source(entity_rows):
        raise LoweringError("entity_rows are CUDA columns: get_offline_features returns a host frame; use get_offline_tensors, "
                            "which builds the training set from them in device memory")
    q = _plan_query(feature_vector, entity_rows, entity_timestamp_column, target=target, run_config=run_config,
                    drop_columns=drop_columns, start_time=start_time, end_time=end_time, with_indexes=with_indexes,
                    update_stats=update_stats, engine=engine, engine_args=engine_args, query=query, order_by=order_by,
                    spark_service=spark_service, timestamp_for_filtering=timestamp_for_filtering,
                    additional_filters=additional_filters, on_host=True)
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
                v = v.view(q.entity_rows.dtypes[c]) if v.dtype != q.entity_rows.dtypes[c] else v
            else:  # strings, categories, objects: permuted on the host in the device's order
                v = q.entity_rows.frame[c].take(order).reset_index(drop=True).array
        elif source[0] == "ts":
            name, src, asof = q.plan[source[1]]
            ts_out = joined[source[1]][1]
            # as-of: cast to the entity column's unit (base.py:389-410); exact: the set's own unit
            tdt = np.dtype(f"datetime64[{q.unit}]") if asof else src.ts_dtype
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
    with the same messages, and datetime features, which a matrix of numbers cannot hold.

    Entity rows may be CUDA columns (a mapping or a `columnar.DeviceColumnBatch`; `entity_timestamp_column` then names an
    int64 / datetime64[ns] column of nanoseconds), and without entity rows the spine may be a set registered from CUDA
    columns: the timestamps, keys and spine columns are then read where they are in HBM, and nothing is uploaded."""
    if np.dtype(dtype) not in (np.float32, np.float64):
        raise ValueError(f"dtype {dtype!r}: the feature matrix is float32 or float64")
    dtype = np.dtype(dtype)
    q = _plan_query(feature_vector, entity_rows, entity_timestamp_column, **options)
    try:
        return _tensors(q, dtype)
    finally:
        q.entity_rows.release()


def _tensors(q, dtype):
    """get_offline_tensors' pack of a planned query"""
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
        col_dtype = q.entity_rows.dtypes[source[1]]
        if col_dtype.kind == "M":
            raise LoweringError(f"{what} {name!r} is a {col_dtype} column: a matrix of numbers has no place for it (drop it from "
                                "the vector)")
        return (-1, used.index(source[1])) + _feat_kind(col_dtype)

    feats = [device_source(name, source, "feature") for name, source in picked]
    label_vec = None
    if label_source is not None:
        label_vec = device_source(f"{q.label[0]}.{q.label[1]}", label_source, "label")
    dev_label = q.dev_label
    if dev_label is not None and dev_label[0] < 0:
        dev_label = (-1, used.index(label_source[1]), dev_label[2])
    if q.device:
        widths = [q.entity_rows.dtypes[c].itemsize for c in used]
        features, label, order, stats = pit_train_pack_device(q.ts_ns, q.n, q.sets, list(zip(arrays, widths)), dev_label, feats,
                                                              label_vec, dtype)
    else:
        features, label, order, stats = pit_train_pack(q.ts_ns, q.sets, arrays, dev_label, feats, label_vec, dtype)
    return TrainingTensors(features, label, order, [name for name, _s in picked], stats["kept"], stats)
