"""numpy emulation of a DevicePlan's arithmetic (tests only).

Lets the CPU suite validate `mlrun_b200.lowering` (fills / maps / schema) and `mlrun_b200.packing`
(sklearn -> device formats) against the oracle without a GPU.  It mirrors the kernel's semantics:
float32 inputs, float32 comparisons, float64 accumulation in column / tree order."""

import numpy as np

from mlrun_b200 import _native as nat


def transform(prog, X):
    """stage 1 + schema of a ColumnProgram -> expanded float32 matrix (B, n_out)"""
    X = np.array(X, dtype=np.float32, copy=True)
    for src, fill in prog.fills.items():
        col = X[:, src]
        col[np.isnan(col)] = np.float32(fill)
    for src, maps in prog.maps.items():
        x = X[:, src]
        for kind, m in maps:
            out = x.copy()
            done = np.zeros(len(x), dtype=bool)
            if kind == "value":
                for k, v in m.items():
                    hit = (~done) & (x == np.float32(k))
                    out[hit] = np.float32(v)
                    done |= hit
            else:
                for lo, hi, v in m:
                    hit = (~done) & (x >= np.float32(lo)) & (x < np.float32(hi))
                    out[hit] = np.float32(v)
                    done |= hit
            x = out
        X[:, src] = x
    cols = []
    for _name, src, kind, arg in prog.cols:
        if kind == nat.OUT_ONEHOT:
            cols.append((X[:, src] == np.float32(arg)).astype(np.float32))
        else:
            cols.append(X[:, src])
    return np.stack(cols, axis=1)


def link(scores, link_kind, classes):
    if link_kind == nat.LINK_IDENTITY:
        return scores[:, 0]
    if link_kind == nat.LINK_BINARY_GT:
        idx = (scores[:, 0] > 0).astype(int)
    elif link_kind == nat.LINK_BINARY_GE:
        idx = (scores[:, 0] >= 0).astype(int)
    else:
        idx = np.argmax(scores, axis=1)
    return idx if classes is None else np.asarray(classes)[idx]


def linear_predict(packed, E):
    scores = E.astype(np.float64) @ packed["W"].T + packed["b"]
    return link(scores, packed["link"], packed["classes"])


def device_thresholds(t):
    """what b2s_plan_add_tree_model_ex stores: `x < t` (xgboost, CMP_LT) becomes `x <= prev_float32(t)`"""
    thr = np.asarray(t.threshold, dtype=np.float32).copy()
    if getattr(t, "cmp_mode", nat.CMP_LE) == nat.CMP_LT:
        split = t.feature >= 0
        low = thr == -np.inf
        thr[split] = np.nextafter(thr[split], np.float32(-np.inf))
        thr[split & low] = np.nan  # nothing is below -inf: every value goes right
    return thr


def trees_predict(t, E):
    B = E.shape[0]
    scores = np.tile(t.init, (B, 1)).astype(np.float64)
    thr_all = device_thresholds(t)
    dleft = getattr(t, "default_left", None)
    for ti in range(t.n_trees):
        base = t.tree_offset[ti]
        node = np.zeros(B, dtype=np.int64)
        active = t.feature[base + node] >= 0
        while active.any():
            f = t.feature[base + node]
            thr = thr_all[base + node]
            x = E[np.arange(B), np.where(f >= 0, f, 0)]
            with np.errstate(invalid="ignore"):
                go_left = x <= thr
            if dleft is not None:  # a missing value follows the node's default child (kernel: the NaN-routing tile copies)
                go_left = np.where(np.isnan(x), dleft[base + node] != 0, go_left)
            nxt = np.where(go_left, t.left[base + node], t.right[base + node])
            node = np.where(active, nxt, node)
            active = t.feature[base + node] >= 0
        scores[:, t.tree_slot[ti]] += t.tree_scale[ti] * t.leaf_value[base + node]
    return link(scores, t.link, t.classes)


def predict(models, E):
    out = []
    for kind, packed in models:
        out.append(linear_predict(packed, E) if kind == "linear" else trees_predict(packed, E))
    return np.stack(out, axis=1)


# ------------------------------------------------------------------------------------------ columnar ingest plan
def run_column_ops(iplan, df):
    """numpy emulation of columns_kernel over the ops an IngestPlan handed to the C-ABI (mlrun_b200/csrc/b2s_columns.cuh):
    float32 / int32 words, fp64 compares against fp64 tables, maps to float32 (int32 when an int32 column maps to int32
    integers), outputs in slot order.  -> (outputs, violations, misses)"""
    from mlrun_b200 import _native as nat

    src = {}
    for name, kind in iplan.schema:
        a = df[name].to_numpy()
        if kind == nat.COL_I64:
            a = a.astype("datetime64[ns]").view(np.int64)
        elif kind == nat.COL_I32:
            a = a.astype(np.int32)
        src[iplan.prog.in_slot[name]] = a
    return run_column_ops_on_slots(iplan, src)


def run_column_ops_on_slots(iplan, src):
    """the same over input slot arrays {slot: array} (what IngestPlan._inputs hands to b2s_cols_run_host)"""
    import pandas as pd

    from mlrun_b200 import _native as nat

    outs, bad, miss = [], [], []
    for kind, slot, skind, fill, arg, check in iplan.ops:
        a = src[slot]
        if skind == nat.COL_F32:
            w = a.astype(np.float32).copy()
            if fill is not None:
                w[np.isnan(w)] = np.float32(fill)
        else:
            w = a
        x = w.astype(np.float64) if skind != nat.COL_I64 else None
        n_miss = None
        if kind == "copy":
            outs.append(w)
        elif kind == "check":
            pass
        elif kind in ("range", "value"):
            val, hit = x.copy(), np.zeros(len(x), dtype=bool)
            if kind == "range":
                for lo, hi, v in arg:
                    inr = (~hit) & (x >= lo) & (x < hi)
                    val[inr] = v
                    hit |= inr
            else:
                for k, v in arg.items():
                    inr = (~hit) & (x == k)
                    val[inr] = v
                    hit |= inr
            n_miss = int((~hit).sum())
            x = val
            labels = [r[2] for r in arg] if kind == "range" else list(arg.values())
            int_words = skind == nat.COL_I32 and all(float(v).is_integer() and -2**31 <= v <= 2**31 - 1 for v in labels)
            outs.append(val.astype(np.int32 if int_words else np.float32))  # int32 words keep int32 values exact
        elif kind == "onehot":
            anyhit = np.zeros(len(x), dtype=bool)
            for c in arg:
                col = x == c
                anyhit |= col
                outs.append(col.astype(np.int32))
            n_miss = int((~anyhit).sum())
        elif kind == "date":
            ts = pd.Series(a.view("datetime64[ns]"))
            part = {v: k for k, v in nat.DATE_PARTS.items()}[arg]
            v = ts.dt.isocalendar().week if part in ("week", "weekofyear") else getattr(ts.dt, part)
            nat_rows = ts.isna().to_numpy()
            outs.append(np.where(nat_rows, -1, np.nan_to_num(v.to_numpy(dtype=np.float64), nan=-1)).astype(np.int32))
            n_miss = int(nat_rows.sum())
        if n_miss is not None:
            miss.append(n_miss)
        if check and (check[0] is not None or check[1] is not None):
            v = np.zeros(len(x), dtype=bool)
            if check[0] is not None:
                v |= x < check[0]
            if check[1] is not None:
                v |= x > check[1]
            bad.append(int(v.sum()))
    return outs, bad, miss


class EmulatedColumns:
    """stand-in for a finalized ColumnsPlan (tests only): `run_host` fills the output slot arrays from the numpy emulation
    above, so IngestPlan.run / FeatureSet.ingest -- column extraction, result block, dtypes, violation and miss counters,
    the DataFrame assembly -- run end to end on CPU"""

    def __init__(self, iplan, real):
        self._iplan, self._real = iplan, real
        real._read_info()

    def __getattr__(self, name):
        return getattr(self._real, name)

    def run_host(self, in_slots, n_rows, out_slots, with_stats=False):
        from mlrun_b200 import _native as nat

        ip = self._iplan
        outs, bad, miss = run_column_ops_on_slots(ip, in_slots)
        slot, k = 0, 0
        for kind, _s, skind, _f, arg, _c in ip.ops:  # output slots are numbered in op order
            if kind == "check":
                continue
            width = len(arg) if kind == "onehot" else 1
            for j in range(width):
                dst = out_slots[slot + j]
                dst[...] = outs[k].view(dst.dtype) if dst.dtype.itemsize == 8 and outs[k].dtype.itemsize == 8 else outs[k]
                k += 1
            slot += width + (1 if (kind == "copy" and skind == nat.COL_I64) else 0)
        counters = np.zeros(max(self._real.n_counters, 1), dtype=np.uint64)
        for (cnt, _name, _v), n in zip(ip.checks, bad):
            counters[cnt] = n
        for (cnt, _name, _what), n in zip(ip.miss, miss):
            counters[cnt] = n
        counters = counters[: self._real.n_counters]
        return (counters, {"rows": int(n_rows), "kernels": 0}) if with_stats else counters


def install_columns(monkeypatch):
    """IngestPlans built from here on run on the emulation (and take their result blocks from ordinary memory)"""
    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bi

    real_init = bi.IngestPlan.__init__

    def init(self, prog, finalize=True):
        real_init(self, prog, finalize=False)
        if finalize:
            self.plan = EmulatedColumns(self, self.plan)

    monkeypatch.setattr(bi.IngestPlan, "__init__", init)
    import ctypes

    class PageablePool:  # result blocks like the pinned pool's, from ordinary memory
        @staticmethod
        def take(nbytes):
            return (ctypes.c_char * max(int(nbytes), 1))()

    monkeypatch.setattr(nat, "PINNED", PageablePool())
