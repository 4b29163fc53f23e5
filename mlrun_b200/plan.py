"""DevicePlan: the lowered form of a run of recognised graph steps (thin wrapper over the C-ABI).

A plan consumes rows of `n_in` 4-byte words (float32 features) and produces `out_cols` words per row:
the transformed row (no models), every model's prediction, or the ensemble vote.  See
include/b200serve.h for the reference functions each call replaces.
"""

import ctypes as C

import numpy as np

from . import _native as nat


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def check_rows(X, n_in):
    """X (a numpy array, or anything with its dtype / ndim / shape / byte strides) as rows a plan of n_in columns reads"""
    if X.dtype != np.float32 or X.ndim != 2 or X.shape[1] != n_in or (X.shape[0] and X.strides[1] != 4):
        raise ValueError(f"rows must be a float32 (B, {n_in}) array with unit inner stride")
    return X


# b2s_run_columns_device packs and scores at most this many rows at a time, in one scratch buffer of that many rows
RANGE_ROWS = 1 << 20


def column_ranges(n, out_row_bytes):
    """[(first row, rows, byte offset of the range's outputs)] of b2s_run_columns_device over n rows"""
    return [(r0, min(RANGE_ROWS, n - r0), r0 * out_row_bytes) for r0 in range(0, n, RANGE_ROWS)]


class PackedTrees:
    """SoA tree ensemble in the layout b2s_plan_add_tree_model takes (children are tree-relative)"""

    def __init__(self, tree_offset, feature, threshold, left, right, leaf_value, tree_slot, tree_scale, init,
                 link=nat.LINK_IDENTITY, classes=None, cmp_mode=nat.CMP_LE, default_left=None, nan_ok=False,
                 node_cat=None, cat_offsets=None, cat_words=None, cat_mode=nat.CAT_NONNEG):
        self.tree_offset = _i32(tree_offset)
        self.feature = _i32(feature)
        self.threshold = _f32(threshold)
        self.left = _i32(left)
        self.right = _i32(right)
        self.leaf_value = _f64(leaf_value)
        self.tree_slot = _i32(tree_slot)
        self.tree_scale = _f64(tree_scale)
        self.init = _f64(init)
        self.link = int(link)
        self.classes = None if classes is None else _i32(classes)
        # tree semantics of the library the model comes from (include/b200serve.h, b2s_plan_add_tree_model_ex)
        self.cmp_mode = int(cmp_mode)  # nat.CMP_LE (scikit-learn, LightGBM) | nat.CMP_LT (xgboost)
        self.default_left = None if default_left is None else np.ascontiguousarray(default_left, dtype=np.uint8)
        self.nan_ok = bool(nan_ok)     # predict() routes NaN to the default child instead of refusing it
        # categorical splits (b2s_plan_add_tree_model_cat): node i with node_cat[i] = s >= 0 goes right iff x is a valid
        # code (cat_mode) whose bit is set in cat_words[cat_offsets[s]:cat_offsets[s + 1]]; None: every node is numeric
        self.node_cat = None if node_cat is None else _i32(node_cat)
        self.cat_offsets = None if cat_offsets is None else _i32(cat_offsets)
        self.cat_words = None if cat_words is None else np.ascontiguousarray(cat_words, dtype=np.uint32)
        self.cat_mode = int(cat_mode)  # nat.CAT_NONNEG (xgboost: x >= 0) | nat.CAT_TRUNC (LightGBM: x > -1)

    @property
    def n_trees(self):
        return len(self.tree_slot)

    @property
    def n_scores(self):
        return len(self.init)

    @property
    def n_nodes(self):
        return len(self.feature)


class DevicePlan:
    def __init__(self, n_in):
        self._lib = nat.load()
        self.n_in = int(n_in)
        self._h = C.c_void_p()
        nat.check(self._lib.b2s_plan_create(self.n_in, C.byref(self._h)))
        self.n_out = self.n_in
        self.out_cols = None
        self.out_is_int = None
        self.finalized = False
        self.n_models = 0

    # ---- construction ------------------------------------------------------------------------
    def set_impute(self, fills):
        """fills: {col_index: value}  (Imputer._impute, feature_store/steps.py:397-406)"""
        if not fills:
            return self
        cols = _i32(list(fills.keys()))
        vals = _f32(list(fills.values()))
        nat.check(self._lib.b2s_plan_set_impute(self._h, nat._p(cols, C.c_int32), nat._p(vals, C.c_float), len(cols)))
        return self

    def add_value_map(self, col, mapping):
        keys = _f32(list(mapping.keys()))
        vals = _f32(list(mapping.values()))
        nat.check(self._lib.b2s_plan_add_value_map(self._h, int(col), nat._p(keys, C.c_float), nat._p(vals, C.c_float), len(keys)))
        return self

    def add_range_map(self, col, ranges):
        """ranges: [(lo, hi, value), ...] in match order (MapValues ranges, steps.py:193-198)"""
        lo = _f32([r[0] for r in ranges])
        hi = _f32([r[1] for r in ranges])
        val = _f32([r[2] for r in ranges])
        nat.check(self._lib.b2s_plan_add_range_map(self._h, int(col), nat._p(lo, C.c_float), nat._p(hi, C.c_float),
                                                   nat._p(val, C.c_float), len(lo)))
        return self

    def set_output_schema(self, schema):
        """schema: [(src_col, kind, arg), ...]"""
        src = _i32([s[0] for s in schema])
        kind = _i32([s[1] for s in schema])
        arg = _f32([s[2] for s in schema])
        nat.check(self._lib.b2s_plan_set_output_schema(self._h, nat._p(src, C.c_int32), nat._p(kind, C.c_int32),
                                                       nat._p(arg, C.c_float), len(src)))
        self.n_out = len(src)
        return self

    def add_linear(self, W, b, link=nat.LINK_IDENTITY, classes=None):
        W = _f64(np.atleast_2d(W))
        b = _f64(np.atleast_1d(b))
        if W.shape[1] != self.n_out or W.shape[0] != b.shape[0]:
            raise ValueError(f"linear model shape {W.shape} does not match n_out={self.n_out}")
        cls = None if classes is None else _i32(classes)
        nat.check(self._lib.b2s_plan_add_linear_model(self._h, nat._p(W, C.c_double), nat._p(b, C.c_double), W.shape[0],
                                                      int(link), nat._p(cls, C.c_int32), 0 if cls is None else len(cls)))
        self.n_models += 1
        return self

    def add_trees(self, t: PackedTrees):
        cls = t.classes
        args = (self._h, t.n_trees, nat._p(t.tree_offset, C.c_int32), nat._p(t.feature, C.c_int32),
                nat._p(t.threshold, C.c_float), nat._p(t.left, C.c_int32), nat._p(t.right, C.c_int32),
                nat._p(t.leaf_value, C.c_double), nat._p(t.tree_slot, C.c_int32), nat._p(t.tree_scale, C.c_double),
                nat._p(t.init, C.c_double), t.n_scores, t.link, nat._p(cls, C.c_int32), 0 if cls is None else len(cls),
                getattr(t, "cmp_mode", nat.CMP_LE), nat._p(getattr(t, "default_left", None), C.c_uint8),
                nat.NAN_DEFAULT_CHILD if getattr(t, "nan_ok", False) else nat.NAN_ERROR)
        node_cat = getattr(t, "node_cat", None)
        if node_cat is None:
            nat.check(self._lib.b2s_plan_add_tree_model_ex(*args))
        else:
            offs, words = getattr(t, "cat_offsets", None), getattr(t, "cat_words", None)
            nat.check(self._lib.b2s_plan_add_tree_model_cat(
                *args, nat._p(node_cat, C.c_int32), nat._p(offs, C.c_int32), 0 if offs is None else len(offs) - 1,
                nat._p(words, C.c_uint32), 0 if words is None else len(words), getattr(t, "cat_mode", nat.CAT_NONNEG)))
        self.n_models += 1
        return self

    def set_vote(self, kind, weights):
        w = _f64(weights)
        nat.check(self._lib.b2s_plan_set_vote(self._h, int(kind), nat._p(w, C.c_double), len(w)))
        return self

    def finalize(self):
        nat.init()
        nat.check(self._lib.b2s_plan_finalize(self._h))
        oc, oi = C.c_int32(), C.c_int32()
        nat.check(self._lib.b2s_plan_out_info(self._h, C.byref(oc), C.byref(oi)))
        self.out_cols, self.out_is_int = oc.value, bool(oi.value)
        self.finalized = True
        return self

    @property
    def kernel(self):
        """which CUDA kernel family this plan launches"""
        return self._lib.b2s_plan_kernel(self._h).decode()

    @property
    def last_kernel(self):
        """which kernel family served the most recent launch (nat.KERNELS: "dense", "rows", "rowthread/tma", ...; None
        before the first): unlike `kernel`, it shows the run-time fallbacks of small host batches and unaligned rows"""
        return nat.KERNELS[self._lib.b2s_plan_last_kernel(self._h)]

    @property
    def out_dtype(self):
        return np.int32 if self.out_is_int else np.float32

    # ---- execution ---------------------------------------------------------------------------
    def _check_rows(self, X):
        return check_rows(X, self.n_in)

    def _stride(self, X):
        return X.strides[0] if X.shape[0] else self.n_in * 4  # an empty array reports no usable strides

    def run(self, X, with_status=False, with_stats=False):
        """synchronous host call: pinned staging -> H2D -> kernels -> D2H (b2s_run_host)"""
        X = self._check_rows(X)
        n = X.shape[0]
        out, status = self._result_arrays(n)
        stats = nat.Stats()
        nat.check(self._lib.b2s_run_host(self._h, nat.ptr(X), n, self._stride(X), nat.ptr(out), out.nbytes, nat.ptr(status), C.byref(stats)))
        res = (out,)
        if with_status:
            res += (status,)
        if with_stats:
            res += (stats.as_dict(),)
        return res if len(res) > 1 else out

    def _result_arrays(self, n):
        """(outputs, status) for n rows.  Large results live in one block of the pinned pool: it is resident (a fresh
        np.empty of 8 MB costs ~2 000 first-touch page faults per call) and goes back to the pool when both arrays are
        collected; small ones are plain arrays (the pool's bookkeeping would cost more than it saves)."""
        out_bytes = (n * self.out_cols * 4 + 63) // 64 * 64
        block = nat.PINNED.take(out_bytes + n * 4) if out_bytes + n * 4 >= (1 << 20) else None
        if block is None:
            return np.empty((n, self.out_cols), dtype=self.out_dtype), np.empty(n, dtype=np.int32)
        out = np.frombuffer(block, dtype=self.out_dtype, count=n * self.out_cols).reshape(n, self.out_cols)
        return out, np.frombuffer(block, dtype=np.int32, count=n, offset=out_bytes)

    def submit(self, X):
        X = self._check_rows(X)
        t = C.c_uint64()
        nat.check(self._lib.b2s_submit(self._h, nat.ptr(X), X.shape[0], self._stride(X), C.byref(t)))
        return (t.value, X.shape[0])

    def wait(self, ticket, with_status=False, with_stats=False):
        t, n = ticket
        out = np.empty((n, self.out_cols), dtype=self.out_dtype)
        status = np.empty(n, dtype=np.int32)
        stats = nat.Stats()
        nat.check(self._lib.b2s_wait(self._h, t, nat.ptr(out), out.nbytes, nat.ptr(status), C.byref(stats)))
        res = (out,)
        if with_status:
            res += (status,)
        if with_stats:
            res += (stats.as_dict(),)
        return res if len(res) > 1 else out

    def flush(self):
        nat.check(self._lib.b2s_flush(self._h))

    def set_ring(self, ring_slots=0, max_batch=0, max_wait_us=-1):
        """ring configuration of this plan (before its first submit); zeros / -1 keep the library defaults"""
        nat.check(self._lib.b2s_plan_set_ring(self._h, int(ring_slots), int(max_batch), int(max_wait_us)))
        return self

    def ring_bench(self, X, n_threads, rows_per_submit, seconds):
        """events/s and round-trip latency of submit -> wait from native producer threads (b2s_ring_bench)"""
        X = self._check_rows(X)
        ev, p50, p99 = C.c_int64(), C.c_double(), C.c_double()
        nat.check(self._lib.b2s_ring_bench(self._h, X.ctypes.data, X.shape[0], self._stride(X), int(n_threads),
                                           int(rows_per_submit), float(seconds), C.byref(ev), C.byref(p50), C.byref(p99)))
        return {"events_per_s": ev.value / float(seconds), "p50_us": p50.value, "p99_us": p99.value,
                "producers": int(n_threads), "rows_per_submit": int(rows_per_submit)}

    def run_device(self, d_rows, n_rows, row_stride, d_out, d_status=None, stream=None):
        nat.check(self._lib.b2s_run_device(self._h, d_rows, n_rows, row_stride, d_out, d_status, stream))

    def run_columns_device(self, cols, n, d_out, d_status=None, stream=None):
        """n rows of `n_in` device columns ([nat.TableCol], one per input column) -> outputs (+ status) in HBM
        (b2s_run_columns_device): packed into float32 rows range by range (`column_ranges`), each range then scored by
        the plan's own launches.  Returns the call's stats (its `kernels`: per range, the pack and the plan's launches)."""
        arr = (nat.TableCol * max(len(cols), 1))(*cols)
        stats = nat.Stats()
        nat.check(self._lib.b2s_run_columns_device(self._h, arr, len(cols), int(n), d_out, d_status, C.byref(stats), stream))
        return stats.as_dict()

    def set_merge_targets(self, peer_ptrs, row_offset):
        """fused ensemble-merge: every output row is stored into each peer buffer at row_offset + row"""
        arr = (C.c_void_p * max(len(peer_ptrs), 1))(*peer_ptrs)
        nat.check(self._lib.b2s_plan_set_merge_targets(self._h, arr, len(peer_ptrs), int(row_offset)))

    def time_device(self, d_row_ptrs, n_rows, row_stride, d_out, iters):
        """CUDA-event time (ms) of `iters` back-to-back launches over rotating input buffers"""
        arr = (C.c_void_p * len(d_row_ptrs))(*d_row_ptrs)
        ms = C.c_float()
        nat.check(self._lib.b2s_time_device(self._h, arr, len(d_row_ptrs), n_rows, row_stride, d_out, iters, C.byref(ms)))
        return ms.value

    def close(self):
        if self._h:
            self._lib.b2s_plan_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
