"""Real-time feature enrichment backed by a device-resident online table.

Plugin-API mirror of the parts of mlrun.feature_store the enrichment routers touch: `get_feature_vector(uri)
.get_online_feature_service(impute_policy=...)` -> `OnlineVectorService.get(entity_rows, as_list)`
(mlrun/feature_store/feature_vector.py:903-1067).  The reference reads the online (NoSQL) store once per entity row
through a storey graph; here the vector's online rows live in HBM (`b2s_table_*`, include/b200serve.h) and a batch of
keys is resolved by one kernel launch.  The feature-store control plane (vector definition, targets, stats
calculation jobs) is out of scope: a `FeatureVector` is built from an in-memory frame, or from CUDA columns (a
`columnar.DeviceColumnBatch` or a mapping), and registered by uri.  A vector of CUDA columns builds its table, its
statistics and its label set on the device (b2s_table_create_device and friends): only counters, the 5 x F statistics
and the keys of rows with a truthy label cross to the host, and the service equals the one built from the equal frame.

Values are float32 on the device; impute values (constants or "$mean"-style statistics) are rounded to float32 when the
service is initialised, and the stats table computed here is float32-valued, so `get()` returns the same numbers on
both sides of the C-ABI.  String entity keys are hashed to 64 bits (FNV-1a, collisions among the table's keys are
rejected when the table is built; an unknown key matching a stored hash has probability ~ n_keys / 2^64).
"""

import ctypes as C

import numpy as np

from .. import _native as nat
from ..lowering import LoweringError
from ..serving.resolve import MLRunInvalidArgumentError
from . import columnar

_REGISTRY = {}


def register_feature_vector(uri, vector):
    _REGISTRY[uri] = vector


def get_feature_vector(uri, project=None):
    """mlrun.feature_store.get_feature_vector (feature_store/api.py:73-97) over the process-local registry"""
    try:
        return _REGISTRY[uri]
    except KeyError:
        raise MLRunInvalidArgumentError(f"feature vector {uri!r} is not registered (register_feature_vector)")


def _hash_strings(values):
    data = [str(v).encode() for v in values]
    offsets = np.zeros(len(data) + 1, dtype=np.int64)
    np.cumsum([len(d) for d in data], out=offsets[1:])
    keys = np.empty(len(data), dtype=np.int64)
    nat.check(nat.load().b2s_hash_strings(b"".join(data), offsets.ctypes.data_as(C.POINTER(C.c_int64)), len(data),
                                          keys.ctypes.data_as(C.POINTER(C.c_int64))))
    return keys


class DeviceTable:
    """thin wrapper over b2s_table_* (64-bit keys -> rows of float32 features, optional impute vector)"""

    def __init__(self, keys, values, impute=None):
        nat.init()
        self._lib = nat.load()
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        values = np.ascontiguousarray(values, dtype=np.float32)
        self.n_keys, self.n_feat = values.shape
        imp = None if impute is None else np.ascontiguousarray(impute, dtype=np.float32)
        self._h = C.c_void_p()
        nat.check(self._lib.b2s_table_create(keys.ctypes.data_as(C.POINTER(C.c_int64)), len(keys), nat._p(values, C.c_float),
                                             self.n_feat, nat._p(imp, C.c_float), C.byref(self._h)))

    @classmethod
    def device(cls, d_keys, n_keys, cols, impute=None):
        """the table of n_keys rows whose keys (an int64 address) and feature columns ([nat.TableCol]) are in device memory
        (b2s_table_create_device): the same table b2s_table_create builds from the same values as float32"""
        self = cls.__new__(cls)
        self._lib = nat.init()
        self.n_keys, self.n_feat = int(n_keys), len(cols)
        imp = None if impute is None else np.ascontiguousarray(impute, dtype=np.float32)
        self._h = C.c_void_p()
        nat.check(self._lib.b2s_table_create_device(d_keys, self.n_keys, (nat.TableCol * len(cols))(*cols), self.n_feat,
                                                    nat._p(imp, C.c_float), C.byref(self._h)))
        return self

    def lookup_arrays(self, d_keys):
        """device keys (a DeviceArray of int64) -> ((n, F) float32 imputed rows, (n,) int32 found flags) as DeviceArrays,
        ready when returned"""
        n = d_keys.shape[0]
        rows = nat.DeviceArray(nat.darray_alloc(max(n * self.n_feat * 4, 4)), (n, self.n_feat), np.float32)
        found = nat.DeviceArray(nat.darray_alloc(max(n * 4, 4)), (n,), np.int32)
        if n:
            self.lookup_device(d_keys.ptr, n, rows.ptr, self.n_feat * 4, found.ptr)
            nat.check(self._lib.b2s_device_sync())
        return rows, found

    def enrich_arrays(self, plan, d_keys):
        """device keys -> (outputs, status) of `plan` as DeviceArrays, ready when returned: one fused launch
        (b2s_table_enrich_device), or for plans the gather loader does not cover the gather, the plan's launches and the
        unknown-key bits, as b2s_table_enrich_host runs them"""
        n = d_keys.shape[0]
        out = nat.DeviceArray(nat.darray_alloc(max(n * plan.out_cols * 4, 4)), (n, plan.out_cols), plan.out_dtype)
        status = nat.DeviceArray(nat.darray_alloc(max(n * 4, 4)), (n,), np.int32)
        if n:
            if not self.enrich_device(plan, d_keys.ptr, n, out.ptr, status.ptr):
                if b"merge targets" in (self._lib.b2s_last_error() or b""):
                    nat.check(-6)  # the plan stores its votes elsewhere: refused, as b2s_table_enrich_host refuses it
                rows, found = self.lookup_arrays(d_keys)
                plan.run_device(rows.ptr, n, self.n_feat * 4, out.ptr, status.ptr)
                nat.check(self._lib.b2s_table_mark_unknown_device(found.ptr, status.ptr, n, None))
            nat.check(self._lib.b2s_device_sync())
        return out, status

    def lookup(self, keys, with_stats=False):
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        rows = np.empty((len(keys), self.n_feat), dtype=np.float32)
        found = np.empty(len(keys), dtype=np.int32)
        stats = nat.Stats()
        nat.check(self._lib.b2s_table_lookup_host(self._h, keys.ctypes.data_as(C.POINTER(C.c_int64)), len(keys),
                                                  nat._p(rows, C.c_float), nat._p(found, C.c_int32), C.byref(stats)))
        return (rows, found.astype(bool), stats.as_dict()) if with_stats else (rows, found.astype(bool))

    def enrich(self, plan, keys, with_stats=False):
        """keys -> gather -> `plan` (a finalized DevicePlan over this table's features) -> (outputs, status) on the host, in
        one C call (b2s_table_enrich_host); status carries ROW_UNKNOWN_KEY for keys that are not in the table.  The two
        arrays share one pinned block of the pool (PCIe-speed D2H, no second copy); it is reused once they are collected."""
        keys = np.ascontiguousarray(keys, dtype=np.int64)
        n = len(keys)
        out_b = (n * plan.out_cols * 4 + 63) // 64 * 64
        block = nat.PINNED.take(out_b + n * 4) if n else None
        if block is not None:
            out = np.frombuffer(block, dtype=plan.out_dtype, count=n * plan.out_cols).reshape(n, plan.out_cols)
            status = np.frombuffer(block, dtype=np.int32, count=n, offset=out_b)
        else:
            out = np.empty((n, plan.out_cols), dtype=plan.out_dtype)
            status = np.empty(n, dtype=np.int32)
        stats = nat.Stats() if with_stats else None
        nat.check(self._lib.b2s_table_enrich_host(self._h, plan._h, keys.ctypes.data_as(C.POINTER(C.c_int64)), n, out.ctypes.data,
                                                  out.nbytes, nat._p(status, C.c_int32), C.byref(stats) if with_stats else None))
        return (out, status, stats.as_dict()) if with_stats else (out, status)

    def enrich_device(self, plan, d_keys, n, d_out, d_status=None, stream=None):
        """device keys -> outputs (+ status) in ONE launch: the scoring kernel gathers its rows from the table
        (b2s_table_enrich_device).  Returns False when the plan is not covered by the gather loader (nothing was launched:
        use lookup_device + plan.run_device)."""
        rc = self._lib.b2s_table_enrich_device(self._h, plan._h, d_keys, int(n), d_out, d_status, stream)
        if rc == -6:  # B2S_ERR_UNSUPPORTED
            return False
        nat.check(rc)
        return True

    def lookup_device(self, d_keys, n, d_rows, row_stride, d_found=None, stream=None):
        nat.check(self._lib.b2s_table_lookup_device(self._h, d_keys, int(n), d_rows, int(row_stride), d_found, stream))

    def time_device(self, d_key_ptrs, n, d_rows, row_stride, iters):
        arr = (C.c_void_p * len(d_key_ptrs))(*d_key_ptrs)
        ms = C.c_float()
        nat.check(self._lib.b2s_table_time_device(self._h, arr, len(d_key_ptrs), int(n), d_rows, int(row_stride), None,
                                                  int(iters), C.byref(ms)))
        return ms.value

    def close(self):
        if self._h:
            self._lib.b2s_table_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FeatureVector:
    """name, requested features, index (entity) keys, label column, and the online rows: a frame whose index (or
    `index_keys` columns) holds the entity keys, or CUDA columns -- a `columnar.DeviceColumnBatch` (its `index` holds the
    entity columns, unless `index_keys` name result columns) or a mapping that holds the `index_keys` columns.  CUDA
    columns are described here and read when the service is built; the service equals the one built from the equal frame
    (`batch.to_host().to_pandas()`, or the mapping's columns indexed by `index_keys`)."""

    def __init__(self, name, features, index_keys, frame, stats=None, label_column=None, with_indexes=False):
        self.name = name
        self.features = list(features)
        self.index_keys = list(index_keys)
        self.label_column = label_column
        self.with_indexes = with_indexes
        self.device = None
        if columnar.is_columnar(frame) and columnar.is_device_source(frame):
            self.device = _DeviceRows(frame, self.index_keys)
            frame = None
        elif all(k in frame.columns for k in self.index_keys):
            frame = frame.set_index(self.index_keys)
        self.frame = frame
        self._stats = stats

    def get_stats_table(self):
        """feature statistics (mean / min / max / std / count per feature), float32-valued.  Of CUDA columns: one
        reduction on the device (b2s_table_stats_device); count, min and max equal the frame's, mean and std are within one
        float32 ulp of them (bit-equal where every float64 partial sum is exact: the frame sums sequentially)"""
        if self._stats is None:
            import pandas as pd

            cols = [f for f in self.features if f != self.label_column]
            if self.device is not None:
                stats = dict(zip(("mean", "min", "max", "std", "count"), self.device.stats(cols)))
            else:
                vals = self.frame[cols].to_numpy(dtype=np.float32).copy()
                vals[~np.isfinite(vals)] = np.nan  # statistics of the finite observations
                with np.errstate(all="ignore"):
                    stats = {
                        "mean": np.nanmean(vals.astype(np.float64), axis=0).astype(np.float32),
                        "min": np.nanmin(vals, axis=0), "max": np.nanmax(vals, axis=0),
                        "std": np.nanstd(vals.astype(np.float64), axis=0, ddof=1).astype(np.float32),
                        "count": np.sum(~np.isnan(vals), axis=0).astype(np.float32),
                    }
            self._stats = pd.DataFrame({k: [float(x) for x in v] for k, v in stats.items()}, index=cols)
        return self._stats

    def get_online_feature_service(self, impute_policy=None, **kwargs):
        svc = OnlineVectorService(self, impute_policy)
        svc.initialize()
        return svc


class OnlineVectorService:
    """feature_vector.py:903-1067 with the store read replaced by the device table"""

    def __init__(self, vector, impute_policy=None):
        self.vector = vector
        self.impute_policy = impute_policy or {}
        self._index_columns = vector.index_keys
        self._requested_columns = vector.features
        self._columns = [c for c in vector.features if c != vector.label_column]
        self._impute_values = {}
        self.table = None
        self._string_keys = False
        self._label_alive = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def status(self):
        return "ready"

    def initialize(self):
        """impute values (feature_vector.py:935-968), then the online rows go to the device"""
        self._impute_values = self._resolve_policy(dict(self.impute_policy)) if self.impute_policy else {}
        if self.vector.device is not None:
            return self._initialize_device(self.vector.device)
        frame = self.vector.frame
        values = frame[self._columns].to_numpy(dtype=np.float32)
        keys = self._encode_keys(frame.index, build=True)
        # the label is not an online feature, but in the reference a truthy label keeps an all-zero row from being reported as
        # missing (the `any(data.values())` quirk): remember which entities have one
        label = self.vector.label_column
        self._label_alive = None
        if label and label in frame.columns:
            col = frame[label]
            self._label_alive = np.sort(keys[(col.notna() & col.map(bool)).to_numpy(dtype=bool)])  # a missing label is no label
        impute = np.array([self._impute_values.get(c, np.nan) for c in self._columns], dtype=np.float32)
        self.table = DeviceTable(keys, values, impute if self._impute_values else None)

    def _initialize_device(self, rows):
        """the table, its keys and the truthy-label keys built where the CUDA columns are"""
        feats = rows.table_cols(self._columns, "feature")
        label = self.vector.label_column
        label_col = rows.table_cols([label], "label")[0] if label and label in rows.columns else None
        impute = np.array([self._impute_values.get(c, np.nan) for c in self._columns], dtype=np.float32)
        self._string_keys = len(rows.keys) > 1
        self._label_alive = None
        try:
            keys = _encode_device_keys(rows.keys, self._string_keys)
            cols = [nat.TableCol(c.acquire().ptr, dt.itemsize, kind) for c, dt, kind in feats]
            try:
                self.table = DeviceTable.device(keys.ptr, rows.n, cols, impute if self._impute_values else None)
            except nat.NativeError as err:  # the frame path hashes composite keys first and refuses a repeat there
                if self._string_keys and "duplicate entity key" in str(err):
                    raise MLRunInvalidArgumentError("two entity keys share a 64-bit hash (or a key is duplicated)") from None
                raise
            if label_col is not None:
                c, dt, kind = label_col
                alive, count = np.empty(rows.n, dtype=np.int64), C.c_int64()
                nat.check(nat.load().b2s_table_label_keys_device(keys.ptr, rows.n, C.byref(nat.TableCol(c.acquire().ptr, dt.itemsize, kind)),
                                                                 nat._p(alive, C.c_int64), C.byref(count), None))
                self._label_alive = np.sort(alive[:count.value])
            keys.release()
        finally:
            rows.release()

    def _device_keys(self, keys):
        """CUDA entity keys -> a library int64 array encoded as `_encode_keys` encodes the equal host keys; None for host
        keys.  One CUDA int column for a single entity, or a mapping holding the `index_keys` columns."""
        if isinstance(keys, dict) and keys and columnar.is_device_source(keys):
            cols = columnar.device_columns(keys)
            missing = [k for k in self._index_columns if k not in cols]
            if missing:
                raise LoweringError(f"the CUDA keys have no entity column {missing[0]!r}")
            cols = [cols[k] for k in self._index_columns]
        elif columnar.is_device_column(keys):
            cols = [columnar.DeviceColumn(keys, self._index_columns[0] if self._index_columns else "key")]
        else:
            return None
        _check_key_columns(cols)
        if len(cols) > 1 and not self._string_keys:
            raise MLRunInvalidArgumentError("the online table has integer entity keys")
        try:
            return _encode_device_keys(cols, self._string_keys)
        finally:
            for c in cols:
                c.release()

    def _resolve_policy(self, policy):
        """{feature | "*": constant | "$stat"} -> {feature: float32 value held on the device} (feature_vector.py:935-968)"""
        if self.vector.device is None:
            self.vector.get_stats_table()
        else:  # the refusals of the features come first, as there; the statistics are reduced when a "$" value needs them
            self.vector.device.table_cols(self._columns, "feature")

        def value_of(feature, spec):
            v = self.vector.get_stats_table().loc[feature, spec[1:]] if isinstance(spec, str) and spec.startswith("$") else spec
            v = float(np.float32(v))
            if not np.isfinite(v):
                raise MLRunInvalidArgumentError(f"impute value of feature {feature} is not finite ({v}): not held on the device")
            return v

        default = policy.pop("*", None)
        unknown = [f for f in policy if f not in self._columns]
        if unknown:
            raise MLRunInvalidArgumentError(f"feature {unknown[0]} in impute_policy but not in feature vector")
        values = {} if default is None else {f: value_of(f, default) for f in self._columns if f not in policy}
        values.update({f: value_of(f, spec) for f, spec in policy.items()})
        return values

    def _encode_keys(self, raw, build=False):
        """entity keys -> int64: integers as they are, everything else through the 64-bit string hash"""
        import pandas as pd

        if isinstance(raw, pd.MultiIndex) or (len(raw) and isinstance(raw[0], (tuple, list))):
            raw = [".".join(str(x) for x in k) for k in raw]
            strings = True
        else:
            arr = np.asarray(raw)
            strings = arr.dtype.kind not in "iu"
            raw = arr
        if build:
            self._string_keys = strings
        elif strings != self._string_keys:
            raw, strings = ([str(x) for x in raw], True) if self._string_keys else (raw, strings)
            if not self._string_keys:
                raise MLRunInvalidArgumentError("the online table has integer entity keys")
        if not strings:
            return np.asarray(raw, dtype=np.int64)
        keys = _hash_strings(raw)
        if build and len(np.unique(keys)) != len(keys):
            raise MLRunInvalidArgumentError("two entity keys share a 64-bit hash (or a key is duplicated)")
        return keys

    def _has_truthy_label(self, key):
        alive = self._label_alive
        if alive is None or not len(alive):
            return False
        j = int(np.searchsorted(alive, key))
        return j < len(alive) and alive[j] == key

    # ---- batched engine surface --------------------------------------------------------------------
    def get_matrix(self, keys):
        """entity keys (one per row; tuples for composite keys) -> ((B, F) float32 imputed rows, found mask).  CUDA keys
        (one int column, or a mapping of the `index_keys` int columns) give `_native.DeviceArray`s instead: the rows and
        int32 found flags, ready when returned."""
        d_keys = self._device_keys(keys)
        if d_keys is None:
            return self.table.lookup(self._encode_keys(keys))
        try:
            return self.table.lookup_arrays(d_keys)
        finally:
            d_keys.release()

    # ---- the reference's call ---------------------------------------------------------------------------
    def get(self, entity_rows, as_list=False):
        """feature_vector.py:975-1067"""
        if isinstance(entity_rows, dict):
            entity_rows = [entity_rows]
        if not entity_rows or not isinstance(entity_rows, list) or not isinstance(entity_rows[0], (list, dict)):
            raise MLRunInvalidArgumentError(
                f"input data is of type {type(entity_rows)}. must be a list of lists or list of dicts")
        idx = self._index_columns
        if isinstance(entity_rows[0], list):
            if not idx or len(entity_rows[0]) != len(idx):
                raise MLRunInvalidArgumentError("input list must be in the same size of the index_keys list")
            entity_rows = [{idx[i]: item[i] for i in range(len(idx))} for item in entity_rows]
        keys = [row[idx[0]] if len(idx) == 1 else tuple(row[k] for k in idx) for row in entity_rows]
        encoded = self._encode_keys(keys)
        rows, found = self.table.lookup(encoded)
        results = []
        for i, row in enumerate(entity_rows):
            if not found[i]:
                # the graph returned only the entity columns (:1030-1034) -- unless the row carried more than the keys
                if all(col in idx for col in row):
                    results.append(None)
                    continue
                vals = [None] * len(self._columns)
            else:
                vals = rows[i].tolist()  # a stored NaN without an impute value stays NaN (:1046-1052)
            data = dict(row)
            if not found[i] and self._impute_values:
                vals = [self._impute_values.get(c, v) for c, v in zip(self._columns, vals)]
            data.update(zip(self._columns, vals))
            if not self.vector.with_indexes:
                for name in self.vector.index_keys:
                    data.pop(name, None)
            if not any(data.values()) and not (found[i] and self._has_truthy_label(encoded[i])):
                data = None
            if as_list and data is not None:
                data = [data.get(key, None) for key in self._requested_columns if key != self.vector.label_column]
            results.append(data)
        return results

    def close(self):
        if self.table is not None:
            self.table.close()
            self.table = None


# ------------------------------------------------------------------------------------------------ online rows in HBM
_TCOL_KINDS = {"f": nat.TCOL_FLOAT, "i": nat.TCOL_INT, "u": nat.TCOL_UINT, "b": nat.TCOL_BOOL}


def _check_key_columns(cols):
    """entity columns of CUDA keys: signed ints of one length (the frame path hashes str() of other values, and a device
    has no strings)"""
    for c in cols:
        if c.dtype.kind != "i":
            raise LoweringError(f"entity key {c.name!r} has dtype {c.dtype}: CUDA entity keys are signed int columns (the "
                                "frame path hashes str() of other values)")
    if len({c.n for c in cols}) > 1:
        raise ValueError("All arrays must be of the same length")


def _encode_device_keys(cols, strings):
    """-> a DeviceArray of int64 keys: one column widened (b2s_keys_encode_device), or the FNV-1a hash of the row's
    decimal text joined by "." (b2s_keys_hash_decimal_device), as `_encode_keys` encodes ints and tuples"""
    lib = nat.init()
    n = cols[0].n
    keys = nat.DeviceArray(nat.darray_alloc(max(8 * n, 8)), (n,), np.int64)
    if n:
        kc = (nat.KeyCol * len(cols))(*[nat.KeyCol(c.acquire().ptr, c.dtype.itemsize, 1) for c in cols])
        fn = lib.b2s_keys_hash_decimal_device if strings else lib.b2s_keys_encode_device
        nat.check(fn(kc, len(cols), n, keys.ptr, None))
    return keys


def table_cols(columns, names, what):
    """-> [(DeviceColumn, dtype, nat.TCOL_*)] of the named columns of {name: DeviceColumn}; a missing name is pandas'
    KeyError"""
    missing = [f for f in names if f not in columns]
    if missing:
        import pandas as pd

        pd.DataFrame(columns=list(columns))[names]  # raises the frame path's KeyError
    out = []
    for f in names:
        c = columns[f]
        kind = _TCOL_KINDS.get(c.dtype.kind)
        if kind is None or (c.dtype.kind == "f" and c.dtype.itemsize not in (4, 8)):
            raise LoweringError(f"{what} {f!r} has dtype {c.dtype}: the online table takes float32, float64, (u)int8/16/32/64 "
                                "and bool columns")
        out.append((c, c.dtype, kind))
    return out


class _DeviceRows:
    """a vector's online rows as CUDA columns: `keys` (the entity columns in order) and `columns` {name: DeviceColumn},
    described when the vector is made, acquired by each call that reads them"""

    def __init__(self, source, index_keys):
        cols = columnar.device_columns(source)
        if len({c.n for c in cols.values()}) > 1:
            raise ValueError("All arrays must be of the same length")
        data = list(source.columns) if isinstance(source, columnar.DeviceColumnBatch) else list(cols)
        if isinstance(source, columnar.DeviceColumnBatch) and not all(k in source.columns for k in index_keys):
            names = list(source.index)  # the frame keeps the batch's index
            if not names:
                raise LoweringError("the DeviceColumnBatch has no entity columns (index) and no index_keys columns")
        else:
            names = list(index_keys)
            missing = [k for k in names if k not in cols]
            if not names or missing:
                raise LoweringError(f"the online rows have no entity column {(missing or [None])[0]!r}: CUDA columns hold their "
                                    "keys in the index_keys columns")
        self.keys = [cols[k] for k in names]
        _check_key_columns(self.keys)
        self.columns = {k: cols[k] for k in data if k not in names}
        self.n = self.keys[0].n

    def table_cols(self, names, what):
        return table_cols(self.columns, names, what)

    def stats(self, names):
        """the frame path's statistics of the named features as a (5, F) float32 array: mean, min, max, std, count"""
        feats = self.table_cols(names, "feature")
        out = np.empty((5, len(names)), dtype=np.float32)
        if not names:
            return out
        try:
            lib = nat.init()
            cols = [nat.TableCol(c.acquire().ptr, dt.itemsize, kind) for c, dt, kind in feats]
            nat.check(lib.b2s_table_stats_device((nat.TableCol * len(cols))(*cols), len(cols), self.n, nat._p(out, C.c_float), None))
        finally:
            self.release()
        return out

    def release(self):
        for c in self.keys + list(self.columns.values()):
            c.release()
