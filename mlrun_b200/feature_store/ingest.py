"""Feature-set ingestion on the device: DataFrame in -> transformed DataFrame out.

Plugin-API mirror of the reference's ingest caller for in-memory frames: `FeatureSet(...).graph.to(...)`,
`FeatureSet.ingest(df)` (mlrun/feature_store/feature_set.py:1004-1090) -> `init_featureset_graph`
(mlrun/feature_store/ingestion.py:38-127), which pushes the frame ROW BY ROW through the step DAG
(storey.DataframeSource, datastore/sources.py:886-895) and re-assembles a frame (ReduceToDataFrame,
datastore/targets.py:1856-1868).  Here the steps are walked symbolically over the frame's schema
(`FrameProgram`, same per-row semantics) and lowered to ONE columnar device plan (`mlrun_b200.columns`); the frame's
columns go to the GPU as they are (contiguous typed arrays) and the result columns come back the same way.

`FeatureSet.add_aggregation` (storey.AggregateByKey, emitting every event) runs after the columns plan as one more device
call over the keyed, timestamped result columns (`AggregationPlan`, b2s_agg_run_host): float64 columns land in the same
result block.

Out of scope (control plane / storage): targets, feature-set metadata / stats inference, sources other than a
DataFrame.  Steps or dtypes the device cannot hold raise `LoweringError`: there is no per-row Python fallback.
"""

import ctypes as C
import math
import re

import numpy as np

from .. import _native as nat
from ..columns import F32, I32, I64, ColumnsPlan
from ..lowering import LoweringError
from ..serving.resolve import MLRunInvalidArgumentError

_INT_DTYPES = ("int8", "int16", "int32", "uint8", "uint16", "bool")


def _short(value):
    """reports carry at most 40 characters of a violating value (mlrun/features.py:24-35)"""
    text = str(value)
    return text if len(text) <= 40 else text[:40] + "..."


class MinMaxValidator:
    """mlrun/features.py:265-321 -- range check whose only effect is a report (check_type is metadata here)"""

    kind = "minmax"

    def __init__(self, check_type=None, severity=None, min=None, max=None):
        self.check_type = check_type
        self.severity = severity
        self.min = min
        self.max = max

    def check(self, value):
        try:
            if self.min is not None and value < self.min:
                return False, {"message": "value is smaller than min", "min": self.min, "value": _short(value)}
            if self.max is not None and value > self.max:
                return False, {"message": "value is greater than max", "max": self.max, "value": _short(value)}
        except Exception as err:  # noqa: BLE001 -- the reference reports comparison errors as violations
            return False, {"message": str(err), "type": self.kind}
        return True, {}


def _num(v, what):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
        raise LoweringError(f"{what}: {v!r} is not numeric -- string / object values are not held on the device")
    return float(v)


def _f32_exact(v, what):
    v = _num(v, what)
    if math.isfinite(v) and float(np.float32(v)) != v:
        raise LoweringError(f"{what}: {v!r} is not exactly representable in the float32 output column")
    return v


class _Col:
    """one column of the event as the steps see it"""

    __slots__ = ("name", "slot", "kind", "fill", "op", "arg", "check", "group")

    def __init__(self, name, slot, kind):
        self.name, self.slot, self.kind = name, slot, kind
        self.fill = None    # Imputer value (float sources)
        self.op = None      # None | "range" | "value" | "onehot" | "date"
        self.arg = None     # ranges / mapping / category index / date part
        self.check = None   # (min, max, validator)
        self.group = None   # one-hot group: the _Group shared by the expanded columns


class _Group:
    def __init__(self, src, cats):
        self.src, self.cats = src, cats
        self.first_out = None
        self.miss = None


def frame_schema(df):
    """[(column name, kind)] of a DataFrame, or LoweringError for dtypes the device does not take as they are"""
    schema = []
    for name in df.columns:
        dt = df[name].dtype
        s = str(dt)
        if s == "float32":
            kind = F32
        elif s in _INT_DTYPES:
            kind = I32
        elif s.startswith("datetime64"):
            kind = I64
        else:
            raise LoweringError(
                f"column {name!r} has dtype {s}: the device takes float32, (u)int8/16/32, bool and datetime64 columns; "
                "cast float64/int64 columns explicitly (a silent down-cast would change values)")
        schema.append((str(name), kind))
    return schema


class FrameProgram:
    """symbolic execution of feature-store steps over the frame's columns, with the storey engine's per-row
    semantics (feature_store/steps.py `_do_storey` methods)"""

    def __init__(self, schema):
        self.schema = list(schema)
        names = [n for n, _ in self.schema]
        if len(set(names)) != len(names):
            raise LoweringError("duplicate column names")
        self.cols, slot = [], 0
        for name, kind in self.schema:
            self.cols.append(_Col(name, slot, kind))
            slot += 2 if kind == I64 else 1
        self.n_in_slots = slot
        self.in_slot = {c.name: c.slot for c in self.cols}
        self.checked_dropped = []
        self.validators = []
        self.steps = []

    # ---- step handlers ------------------------------------------------------------------------
    def imputer(self, step):
        """Imputer._impute (steps.py:397-406): every missing value -> mapping.get(feature, default_value)"""
        mapping, default = step.mapping or {}, step.default_value
        for c in self.cols:
            fill = mapping.get(c.name, default)
            if fill is None:
                continue  # NaN -> None: still missing when the frame is re-assembled
            if c.kind == I32 or c.op in ("onehot", "date"):
                continue  # integers are never missing
            if c.kind == I64:
                raise LoweringError(f"Imputer would replace NaT in the timestamp column {c.name!r}: not held on the device")
            if c.op is not None:
                raise LoweringError(f"Imputer after MapValues on column {c.name!r} is not lowered")
            if c.fill is None:
                c.fill = _f32_exact(fill, f"Imputer fill for {c.name!r}")

    def map_values(self, step):
        """MapValues._do_storey (steps.py:203-216)"""
        mapped = []
        for c in self.cols:
            if c.name not in step.mapping:
                continue
            if c.op is not None or c.kind == I64:
                raise LoweringError(f"MapValues on the derived / timestamp column {c.name!r} is not lowered")
            fmap = step.mapping[c.name]
            m = _Col(f"{c.name}_{step.suffix}" if step.with_original_features else c.name, c.slot, c.kind)
            m.fill = c.fill
            if "ranges" in fmap:
                if len(fmap) > 1:
                    raise LoweringError("MapValues mixing ranges and value replacements is rejected by the reference")
                m.op, m.arg = "range", []
                for val, (lo, hi) in fmap["ranges"].items():
                    lo = -math.inf if lo == "-inf" else _num(lo, f"MapValues range of {c.name!r}")
                    hi = math.inf if hi == "inf" else _num(hi, f"MapValues range of {c.name!r}")
                    m.arg.append((lo, hi, _f32_exact(val, f"MapValues range label of {c.name!r}"), val))
            else:
                m.op = "value"
                m.arg = [(_num(k, f"MapValues key of {c.name!r}"), _f32_exact(v, f"MapValues value of {c.name!r}"), v)
                         for k, v in fmap.items()]
            mapped.append(m)
        # storey mode emits the mapped features first, then (optionally) the untouched event
        self.cols = mapped + (self.cols if step.with_original_features else [])

    def one_hot(self, step):
        """OneHotEncoder._do_storey (steps.py:473-478): the feature is replaced in place by one field per category"""
        new = []
        for c in self.cols:
            cats = step.mapping.get(c.name)
            if not cats:
                new.append(c)
                continue
            if c.op is not None or c.kind == I64:
                raise LoweringError(f"OneHotEncoder on the derived / timestamp column {c.name!r} is not lowered")
            if c.kind != I32:
                # a float value equal to an integer category makes the reference add a stray "<col>_<value>" field next
                # to the encoded ones (steps.py:462-470 writes encoding[f"{feature}_{value}"] for the float spelling)
                raise LoweringError(f"OneHotEncoder source {c.name!r} must be an integer column (cast the codes to int32)")
            cats = list(dict.fromkeys(cats))
            for v in cats:
                if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                    raise LoweringError(f"OneHotEncoder categories of {c.name!r} must be integers on the device (got {v!r})")
            g = _Group(c, [float(v) for v in cats])
            for i, v in enumerate(cats):
                e = _Col(f"{c.name}_{step._sanitized_category(v)}", c.slot, c.kind)
                e.op, e.arg, e.group = "onehot", i, g
                new.append(e)
        self.cols = new

    def date_extractor(self, step):
        """DateExtractor._do_storey (steps.py:593-602)"""
        ts = next((c for c in self.cols if c.name == step.timestamp_col), None)
        if ts is None:
            raise MLRunInvalidArgumentError(f"{step.timestamp_col} does not exist in the event")
        if ts.kind != I64 or ts.op is not None:
            raise LoweringError(f"DateExtractor needs {step.timestamp_col!r} to be a datetime64 column")
        for part in step.parts:
            if part not in nat.DATE_PARTS:
                raise LoweringError(f"DateExtractor part {part!r} is not computed on the device (have {sorted(nat.DATE_PARTS)})")
            name = f"{step.timestamp_col}_{part}"
            e = _Col(name, ts.slot, I64)
            e.op, e.arg = "date", nat.DATE_PARTS[part]
            at = next((i for i, c in enumerate(self.cols) if c.name == name), None)
            if at is None:
                self.cols.append(e)
            else:
                self.cols[at] = e  # the event already had that key: overwritten in place

    def drop_features(self, step):
        """DropFeatures._do_storey (steps.py:721-729)"""
        drop = set(step.features)
        have = {c.name for c in self.cols}
        for f in step.features:
            if f not in have:
                raise MLRunInvalidArgumentError(f"The ingesting data doesn't contain a feature named '{f}'")
        for c in self.cols:
            if c.name in drop and c.check is not None:
                if c.op in ("onehot", "date"):
                    raise LoweringError(f"validated derived column {c.name!r} cannot be dropped on the device")
                self.checked_dropped.append(c)
        self.cols = [c for c in self.cols if c.name not in drop]

    def validator(self, step):
        """FeaturesetValidator._do_storey (steps.py:117-128): report only; here violations are counted"""
        for name, v in step._validators.items():
            c = next((c for c in self.cols if c.name == name), None)
            if c is None:
                continue  # `if name in body`
            if getattr(v, "kind", "minmax") != "minmax" and not hasattr(v, "min"):
                raise LoweringError(f"validator of {name!r}: only MinMaxValidator is lowered")
            if c.op in ("onehot", "date") or c.kind == I64:
                raise LoweringError(f"validator on the derived / timestamp column {name!r} is not lowered")
            if c.check is not None:
                raise LoweringError(f"column {name!r} is validated twice")
            lo = None if v.min is None else _num(v.min, f"validator min of {name!r}")
            hi = None if v.max is None else _num(v.max, f"validator max of {name!r}")
            c.check = (lo, hi, v)
        self.validators.append(step)

    def apply(self, step):
        handler = {"Imputer": self.imputer, "MapValues": self.map_values, "OneHotEncoder": self.one_hot,
                   "DateExtractor": self.date_extractor, "DropFeatures": self.drop_features,
                   "FeaturesetValidator": self.validator}.get(type(step).__name__)
        if handler is None:
            raise LoweringError(f"step {type(step).__name__} is not lowered to the columnar device plan")
        handler(step)
        self.steps.append(type(step).__name__)
        if len({c.name for c in self.cols}) != len(self.cols):
            raise LoweringError("two output columns share a name")  # a dict would keep one: not reproduced
        return self

    # ---- plan ----------------------------------------------------------------------------------
    def build(self):
        return IngestPlan(self)


class IngestPlan:
    """the device plan of a FrameProgram + the frame boundary (DataFrame columns <-> slots)"""

    def __init__(self, prog, finalize=True):
        self.prog = prog
        self.schema = prog.schema
        plan = ColumnsPlan(prog.n_in_slots)
        self.ops = []  # what was handed to the C-ABI, in order: (kind, source slot, source kind, fill, argument, check)
        self.out = []  # per output column: (name, slot, how, col)
        self.checks = []  # (counter, column name, validator)
        self.miss = []    # (counter, column name, what)
        self.rounding_maps = []  # (source slot, column name): maps of an int32 column whose float32 output rounds beyond 2^24
        for c in prog.cols:
            chk = None if c.check is None else c.check[:2]
            if c.op is None:
                slot, cnt = plan.add_copy(c.slot, c.kind, fill=c.fill, keep=True, check=chk)
                self.ops.append(("copy", c.slot, c.kind, c.fill, None, chk))
                how = {F32: "f32", I32: "i32", I64: "dt"}[c.kind]
            elif c.op == "range":
                slot, miss, cnt = plan.add_range_map(c.slot, c.kind, [r[:3] for r in c.arg], fill=c.fill, check=chk)
                self.ops.append(("range", c.slot, c.kind, c.fill, [r[:3] for r in c.arg], chk))
                self.miss.append((miss, c.name, "matched no range"))
                how = ("map", miss, _int_labels(r[3] for r in c.arg), _int32_words(c.kind, [r[2] for r in c.arg]))
            elif c.op == "value":
                slot, miss, cnt = plan.add_value_map(c.slot, c.kind, {k: v for k, v, _ in c.arg}, fill=c.fill, check=chk)
                self.ops.append(("value", c.slot, c.kind, c.fill, {k: v for k, v, _ in c.arg}, chk))
                self.miss.append((miss, c.name, "matched no key"))
                how = ("map", miss, _int_labels(r[2] for r in c.arg), _int32_words(c.kind, [r[1] for r in c.arg]))
            elif c.op == "onehot":
                g = c.group
                if g.first_out is None:
                    g.first_out, g.miss = plan.add_onehot(g.src.slot, g.src.kind, g.cats, fill=g.src.fill)
                    self.ops.append(("onehot", g.src.slot, g.src.kind, g.src.fill, list(g.cats), None))
                    self.miss.append((g.miss, g.src.name, "matched no category"))
                slot, cnt, how = g.first_out + c.arg, -1, "i32"
            else:  # date
                slot, miss = plan.add_date_part(c.slot, c.arg)
                self.ops.append(("date", c.slot, I64, None, c.arg, None))
                self.miss.append((miss, c.name, "NaT"))
                cnt, how = -1, ("date", miss, c.arg in nat.DATE_BOOL_PARTS)
            if cnt >= 0:
                self.checks.append((cnt, c.name, c.check[2]))
            if isinstance(how, tuple) and how[0] == "map" and c.kind == I32 and not how[3]:
                self.rounding_maps.append((c.slot, c.name))
            self.out.append((c.name, slot, how))
        for c in prog.checked_dropped:
            chk = c.check[:2]
            if c.op is None:
                _, cnt = plan.add_copy(c.slot, c.kind, fill=c.fill, keep=False, check=chk)
                self.ops.append(("check", c.slot, c.kind, c.fill, None, chk))
            else:
                raise LoweringError(f"validated then dropped mapped column {c.name!r} is not lowered")
            self.checks.append((cnt, c.name, c.check[2]))
        self.plan = plan.finalize() if finalize else plan
        self.counters = None
        self.violations = {}
        self.unmatched = {}
        self.stats = None
        self.agg = None  # AggregationPlan of the graph's aggregation step, if it has one

    @property
    def out_names(self):
        return [o[0] for o in self.out]

    def _inputs(self, df):
        """the frame's columns as contiguous arrays, without copies where pandas allows it"""
        raw = self._block_columns(df)
        ins, keep = {}, []
        for name, kind in self.schema:
            a = raw[name] if raw is not None else df[name].to_numpy()
            if kind == I64:
                a = a.astype("datetime64[ns]", copy=False).view(np.int64)
            elif kind == I32 and a.dtype != np.int32:
                a = a.astype(np.int32)
            a = np.ascontiguousarray(a)
            keep.append(a)
            ins[self.prog.in_slot[name]] = a
        return ins, keep

    @staticmethod
    def _block_columns(df):
        """{column: array} taken one dtype at a time: for a consolidated frame (one block per dtype) `to_numpy()` of the
        same-dtype sub-frame is a view whose columns are contiguous, 4x cheaper than 255 `df[name]` look-ups.  Frames that
        are not consolidated (or a pandas without the block counter) use the per-column path: None."""
        nblocks = getattr(getattr(df, "_mgr", None), "nblocks", None)
        dtypes = df.dtypes
        kinds = set(dtypes)
        if nblocks is None or nblocks > len(kinds) or not df.columns.is_unique:
            return None
        out = {}
        for dt in kinds:
            sub = df.select_dtypes(include=[dt]) if len(kinds) > 1 else df  # the dtype's block(s), not a copy
            names = sub.columns
            block = sub.to_numpy()
            if block.ndim != 2 or not (block.flags["F_CONTIGUOUS"] or block.shape[1] == 1):
                return None  # pandas had to assemble it: the columns would be strided copies
            for j, name in enumerate(names):
                out[name] = block[:, j]
        return out

    def run(self, df, reference_dtypes=False, keys=None):
        """transform the frame; returns a new DataFrame with the same index.  `reference_dtypes=True` widens integer
        results to int64 (what a frame re-assembled from Python ints has) at the price of a host-side copy.  `keys`: the
        rows' encoded entity keys (int64), which a plan with an aggregation needs."""
        import pandas as pd

        if not _same_labels_and_dtypes(df, getattr(self, "_seen", None)):  # a frame like one already checked skips the walk
            if frame_schema(df) != self.schema:
                raise ValueError("the frame does not carry the schema this plan was lowered for")
            self._seen = (df.columns, list(df.dtypes))
        n = len(df)
        ins, _keep = self._inputs(df)
        data, bufs, block, layout = self._run_arrays(ins, n, reference_dtypes, keys)
        return self._assemble(data, bufs, block, layout, n, df.index)

    def _run_arrays(self, ins, n, reference_dtypes=False, keys=None):
        """{input slot: contiguous column array} -> ({result column: array}, landing views, their pinned block, offsets):
        the device run and the dtype rules of the result, with no DataFrame on either side"""
        if self.agg is not None and (keys is None or len(keys) != n):
            raise ValueError("a plan with an aggregation needs the encoded entity key of every row")
        # result columns live in one pinned block (fast D2H, no second copy); the frame built over them keeps the block
        # alive and it returns to the pool when the frame is collected
        for slot, name in self.rounding_maps:
            a = ins[slot]
            if (a.astype(np.float32).astype(np.int64) != a).any():
                raise LoweringError(
                    f"MapValues {name!r}: its values are not all int32 integers, so it writes float32, and the int32 source "
                    "holds values float32 cannot represent (beyond 2^24): they would be rounded where they pass through. "
                    "Map to integers, or cast the column to float32 explicitly")
        specs, extra = self._landing()
        agg_names = self.agg.out_names if self.agg is not None else []
        layout, off = [], 0
        for dt in [sp[2] for sp in specs] + [np.dtype(np.int32)] * len(extra) + [np.dtype(np.float64)] * len(agg_names):
            layout.append(off)
            off += (n * dt.itemsize + 63) // 64 * 64
        block = nat.PINNED.take(off) if n else None

        def column(i, dt):
            return np.frombuffer(block, dtype=dt, count=n, offset=layout[i]) if block is not None else np.empty(n, dtype=dt)

        bufs, outs = {}, {}
        for i, (name, slot, dt) in enumerate(specs):
            bufs[name] = outs[slot] = column(i, dt)
        # slots written by the device but not part of the result (dropped one-hot members) still need a landing buffer
        for j, s_ in enumerate(extra):
            outs[s_] = column(len(specs) + j, np.dtype(np.int32))
        self.counters, self.stats = self.plan.run_host(ins, n, outs, with_stats=True)
        if self.agg is not None:  # cross-row: the whole frame in one call, over the result columns just landed
            for j, name in enumerate(agg_names):
                bufs[name] = column(len(specs) + len(extra) + j, np.dtype(np.float64))
            self.agg.run(keys, ins[self.agg.ts_slot], {c: bufs[c] for c in self.agg.sources}, n, bufs)
        data = {}
        for name, _slot, how in self.out:
            a = bufs[name]
            if how == "dt":
                a = a.view("datetime64[ns]")
            elif isinstance(how, tuple) and how[0] == "map":
                if how[3]:  # int32 words: integer labels keep them, integral float labels make the column float
                    a = a.astype(np.float64) if not how[2] else (a.astype(np.int64) if reference_dtypes else a)
                elif how[2] and self.counters[how[1]] == 0:
                    a = a.astype(np.int64 if reference_dtypes else np.int32)  # every row got an integer label
            elif isinstance(how, tuple) and how[0] == "date":
                if self.counters[how[1]]:
                    a = np.where(a < 0, np.nan, a.astype(np.float64))  # NaT rows
                elif how[2]:
                    a = a.astype(np.bool_)  # the is_* parts are booleans
                elif reference_dtypes:
                    a = a.astype(np.int64)
            elif how == "i32" and reference_dtypes:
                a = a.astype(np.int64)
            data[name] = a
        for name in agg_names:
            data[name] = bufs[name]
        self.violations = {name: int(self.counters[cnt]) for cnt, name, _v in self.checks}
        self.unmatched = {name: int(self.counters[cnt]) for cnt, name, _w in self.miss if self.counters[cnt]}
        for cnt, name, v in self.checks:
            if self.counters[cnt]:
                print(f"{v.severity}! {name} has {int(self.counters[cnt])} values outside [{v.min}, {v.max}]")
        for step in self.prog.validators:
            step.violations = getattr(step, "violations", 0) + sum(
                int(self.counters[cnt]) for cnt, name, v in self.checks if v in step._validators.values())
        return data, bufs, block, layout

    def run_columns(self, columns, reference_dtypes=False, keys=None):
        """columnar twin of `run` (SURVEY 8(f) #1: "Arrow/DLPack in, Arrow/Parquet-ready columns out"): `columns` maps every
        schema column to a contiguous 1-D array of its dtype (numpy, or anything `columnar.as_columns` understands: Arrow
        tables / record batches, DLPack producers); returns a `columnar.ColumnBatch` whose arrays live in one pinned block.
        No pandas object is built or taken apart; pinned inputs (`columnar.pinned_columns`) cross PCIe at full speed and
        frames of 128 Ki rows and more are pipelined in row ranges."""
        from . import columnar

        cols = columnar.as_columns(columns)
        n = None
        ins = {}
        for name, kind in self.schema:
            if name not in cols:
                raise ValueError(f"column {name!r} of the plan's schema is missing")
            a = cols[name]
            want = {F32: ("float32",), I32: _INT_DTYPES, I64: ("datetime64[ns]", "int64")}[kind]
            if a.ndim != 1 or str(a.dtype) not in want:
                raise ValueError(f"column {name!r}: expected a 1-D {' / '.join(want)} array, got {a.dtype} {a.shape}")
            if kind == I64:
                a = a.view(np.int64)
            elif kind == I32 and a.dtype != np.int32:
                a = a.astype(np.int32)
            a = np.ascontiguousarray(a)
            if n is None:
                n = len(a)
            elif len(a) != n:
                raise ValueError("columns of different lengths")
            ins[self.prog.in_slot[name]] = a
        data, _bufs, block, _layout = self._run_arrays(ins, n or 0, reference_dtypes, keys)
        return columnar.ColumnBatch(data, n or 0, block)

    def run_device(self, cols, key_cols=None):
        """device twin of `run_columns`: `cols` maps every schema column to an acquired `columnar.DeviceColumn` (timestamps
        as 8-byte columns); `key_cols` are the entity key columns a plan with an aggregation needs.  Returns a
        `columnar.DeviceColumnBatch` whose columns are the host path's, dtype for dtype and bit for bit, and never leave
        HBM: the columns are staged into one slot block (one convert launch, which also counts int32 map sources float32
        would round), keys are encoded on the device, the columns plan and the aggregation run there, and the counters come
        back in one small copy before one more convert launch gives the result columns their dtypes."""
        from . import columnar

        n = None
        for name, kind in self.schema:
            if name not in cols:
                raise ValueError(f"column {name!r} of the plan's schema is missing")
            c = cols[name]
            want = {F32: ("float32",), I32: _INT_DTYPES, I64: ("datetime64[ns]", "int64")}[kind]
            if str(c.dtype) not in want:
                raise ValueError(f"column {name!r}: expected a 1-D {' / '.join(want)} array, got {c.dtype} ({c.n},)")
            if n is None:
                n = c.n
            elif c.n != n:
                raise ValueError("columns of different lengths")
        n = n or 0
        if self.agg is not None and (key_cols is None or any(k.n != n for k in key_cols)):
            raise ValueError("a plan with an aggregation needs the encoded entity key of every row")
        lib = nat.init()
        before = nat.launch_count()
        stride = max(256, (n * 4 + 255) // 256 * 256)
        n_cnt = self.plan.n_counters
        counters = nat.DeviceArray(nat.darray_alloc(8 * (n_cnt + 3 + len(self.rounding_maps)), zero=True),
                                   (n_cnt + 3 + len(self.rounding_maps),), np.uint64)
        stage = nat.DeviceArray(nat.darray_alloc(stride * self.plan.n_in), (stride * self.plan.n_in,), np.uint8)
        widen = {"float32": nat.CONV_COPY4, "int32": nat.CONV_COPY4, "int8": nat.CONV_I8_I32, "uint8": nat.CONV_U8_I32,
                 "bool": nat.CONV_U8_I32, "int16": nat.CONV_I16_I32, "uint16": nat.CONV_U16_I32, "int64": nat.CONV_COPY8,
                 "datetime64[ns]": nat.CONV_COPY8}
        ops = [nat.Convert(cols[name].ptr, stage.ptr + self.prog.in_slot[name] * stride, widen[str(cols[name].dtype)], 0)
               for name, _kind in self.schema]
        source_of = {self.prog.in_slot[name]: cols[name] for name, _kind in self.schema}
        for j, (slot, _name) in enumerate(self.rounding_maps):
            if str(source_of[slot].dtype) == "int32":  # narrower ints all fit float32
                ops.append(nat.Convert(source_of[slot].ptr, None, nat.CONV_CHECK_F32, n_cnt + 3 + j))
        staged = sum(c.n * c.dtype.itemsize for c in cols.values())
        _convert(lib, ops, n, counters)
        keys = None
        if self.agg is not None:
            keys = nat.DeviceArray(nat.darray_alloc(8 * n), (n,), np.int64)
            kc = (nat.KeyCol * len(key_cols))(*[nat.KeyCol(k.ptr, k.dtype.itemsize, int(k.dtype.kind == "i")) for k in key_cols])
            nat.check(lib.b2s_keys_encode_device(kc, len(key_cols), n, keys.ptr, None))
        specs, _extra = self._landing()
        agg_names = self.agg.out_names if self.agg is not None else []
        col_bytes = (n * 8 + 255) // 256 * 256
        block = nat.darray_alloc(stride * self.plan.n_out + col_bytes * len(agg_names))
        try:
            base = C.c_void_p()
            nat.check(lib.b2s_darray_info(block, C.byref(base), None))
            base = base.value
            self.plan.run_device(stage.ptr, stride, n, base, stride, counters.ptr)
            agg_at = {name: stride * self.plan.n_out + j * col_bytes for j, name in enumerate(agg_names)}
            if self.agg is not None:
                slot_of = {name: slot for name, slot, _dt in specs}
                self.agg.run_device(keys.ptr, stage.ptr + self.agg.ts_slot * stride, n,
                                    {c: base + slot_of[c] * stride for c in self.agg.sources},
                                    {name: base + at for name, at in agg_at.items()}, counters.ptr + 8 * n_cnt)
            got = counters.numpy()  # the one copy back: waits for every launch above
            self.counters = got[:n_cnt]
            for j, (_slot, name) in enumerate(self.rounding_maps):
                if got[n_cnt + 3 + j]:
                    raise LoweringError(
                        f"MapValues {name!r}: its values are not all int32 integers, so it writes float32, and the int32 source "
                        "holds values float32 cannot represent (beyond 2^24): they would be rounded where they pass through. "
                        "Map to integers, or cast the column to float32 explicitly")
            if self.agg is not None:
                self.agg.counters = got[n_cnt: n_cnt + 3]
                self.agg.check_counters()
            data, convs, conv_at, conv_bytes = {}, [], {}, 0
            dt_of = {name: dt for name, _slot, dt in specs}
            slot_of = {name: slot for name, slot, _dt in specs}
            for name, _slot, how in self.out:
                kind, to = None, None
                if isinstance(how, tuple) and how[0] == "map":
                    if how[3] and not how[2]:
                        kind, to = nat.CONV_I32_F64, np.float64
                    elif not how[3] and how[2] and self.counters[how[1]] == 0:
                        kind, to = nat.CONV_F32_I32, np.int32
                elif isinstance(how, tuple) and how[0] == "date":
                    if self.counters[how[1]]:
                        kind, to = nat.CONV_DATE_F64, np.float64
                    elif how[2]:
                        kind, to = nat.CONV_I32_BOOL, np.bool_
                if kind is not None:
                    conv_at[name] = (conv_bytes, kind, np.dtype(to))
                    conv_bytes += (n * np.dtype(to).itemsize + 255) // 256 * 256
            conv_block = nat.darray_alloc(conv_bytes) if conv_at else None
            try:
                for name, _slot, how in self.out:
                    if name in conv_at:
                        at, kind, to = conv_at[name]
                        data[name] = nat.darray_view(conv_block, at, (n,), to)
                        convs.append(nat.Convert(base + slot_of[name] * stride, data[name].ptr, kind, 0))
                    else:
                        data[name] = nat.darray_view(block, slot_of[name] * stride, (n,),
                                                     "datetime64[ns]" if how == "dt" else dt_of[name])
                for name in agg_names:
                    data[name] = nat.darray_view(block, agg_at[name], (n,), np.float64)
                if convs:
                    _convert(lib, convs, n, counters)
                    nat.check(lib.b2s_device_sync())
            finally:
                if conv_block:
                    lib.b2s_darray_release(conv_block)
        finally:
            lib.b2s_darray_release(block)  # the views hold the block from here on
        self.violations = {name: int(self.counters[cnt]) for cnt, name, _v in self.checks}
        self.unmatched = {name: int(self.counters[cnt]) for cnt, name, _w in self.miss if self.counters[cnt]}
        for cnt, name, v in self.checks:
            if self.counters[cnt]:
                print(f"{v.severity}! {name} has {int(self.counters[cnt])} values outside [{v.min}, {v.max}]")
        for step in self.prog.validators:
            step.violations = getattr(step, "violations", 0) + sum(
                int(self.counters[cnt]) for cnt, name, v in self.checks if v in step._validators.values())
        converted = sum(n * to.itemsize for _at, _k, to in conv_at.values())
        self.stats = {"rows": n, "kernels": nat.launch_count() - before, "staged_bytes": staged, "converted_bytes": converted}
        return columnar.DeviceColumnBatch(data, n)

    def _assemble(self, data, bufs, block, layout, n, index):
        """the result frame.  Columns that stayed in their landing buffers and sit next to each other in the result block
        with one dtype become ONE 2-D pandas block (a strided view of the block, no copy): the frame has a handful of blocks
        instead of one per column -- cheaper to build and consolidated for whatever the caller does next."""
        import pandas as pd

        names = list(data)
        if block is None or len(names) < 2:
            return pd.DataFrame(data, index=index, copy=False)
        pieces, loose, i = [], {}, 0

        def flush_loose():
            if loose:
                pieces.append(pd.DataFrame(dict(loose), index=index, copy=False))
                loose.clear()

        while i < len(names):
            a = data[names[i]]
            stride = (n * a.dtype.itemsize + 63) // 64 * 64
            j = i
            if a is bufs[names[i]]:  # untouched landing view: extend the run while dtype and spacing hold
                while (j + 1 < len(names) and data[names[j + 1]] is bufs[names[j + 1]] and data[names[j + 1]].dtype == a.dtype
                       and layout[j + 1] - layout[j] == stride):
                    j += 1
            if j > i:
                flush_loose()
                k, words = j - i + 1, stride // a.dtype.itemsize
                rows = np.frombuffer(block, dtype=a.dtype, count=(k - 1) * words + n, offset=layout[i])
                run = np.lib.stride_tricks.as_strided(rows, shape=(n, k), strides=(a.dtype.itemsize, stride), writeable=True)
                pieces.append(pd.DataFrame(run, columns=names[i:j + 1], index=index, copy=False))
            else:
                loose[names[i]] = a
            i = j + 1
        flush_loose()
        if len(pieces) == 1:
            return pieces[0]
        concat_kw = {} if int(pd.__version__.split(".")[0]) >= 3 else {"copy": False}  # pandas 3: lazy copies by default
        return pd.concat(pieces, axis=1, **concat_kw)

    def _landing(self):
        """(name, slot, dtype) of every result column + the slots the device writes that are not part of the result (dropped
        one-hot members): they still need a landing buffer.  Depends on the plan only: computed once."""
        cached = getattr(self, "_landing_cache", None)
        if cached is None:
            specs = []
            for name, slot, how in self.out:
                is_f32 = how == "f32" or (isinstance(how, tuple) and how[0] == "map" and not how[3])
                dt = np.int64 if how == "dt" else (np.float32 if is_f32 else np.int32)
                specs.append((name, slot, np.dtype(dt)))
            taken = {sp[1] for sp in specs} | {slot + 1 for _n, slot, how in self.out if how == "dt"}  # + second halves
            extra = [s for s in range(self.plan.n_out) if s not in taken]
            cached = self._landing_cache = (specs, extra)
        return cached


def _int_labels(labels):
    return all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in labels)


def _int32_words(kind, values):
    """a map writes int32 words when its source is int32 and every value it maps to is an int32 integer (the rule of
    b2s_cols_add_range_map / _value_map): a value that passes through then stays exact; otherwise it writes float32"""
    return kind == I32 and all(float(v).is_integer() and -2**31 <= v <= 2**31 - 1 for v in values)


def _same_labels_and_dtypes(df, seen):
    """seen = (columns Index, [dtypes]) of an earlier frame; Index.equals is vectorised (50 us for 255 columns where
    building a tuple key of labels and dtypes costs 1 ms)"""
    return seen is not None and df.columns.equals(seen[0]) and list(df.dtypes) == seen[1]


# ------------------------------------------------------------------------------------------ windowed aggregations
AGGREGATES_STEP = "Aggregates"  # feature_set.py:55 aggregates_step, the default step name
_DURATION_NS = {"s": 10**9, "m": 60 * 10**9, "h": 3600 * 10**9, "d": 86400 * 10**9}
_MAX_WINDOWS, _MAX_SPECS, _MAX_SOURCES = 16, 64, 16  # b2s_agg_run_host's limits


def _duration_ns(text, what):
    """'10m' -> nanoseconds; units s / m / h / d"""
    m = re.fullmatch(r"\s*(\d+)\s*([A-Za-z]+)\s*", str(text))
    if not m or m.group(2) not in _DURATION_NS:
        raise LoweringError(f"{what} {text!r}: windows and periods are <count><unit> with unit s, m, h or d")
    ns = int(m.group(1)) * _DURATION_NS[m.group(2)]
    if not 0 < ns < 2**63:
        raise LoweringError(f"{what} {text!r} is empty or beyond the int64 nanosecond range")
    return ns


class AggregateByKey:
    """storey.AggregateByKey as FeatureSet.add_aggregation places it in the graph: its class arguments only.  It is never
    run per event; `AggregationPlan` lowers it to one device call over the whole frame."""

    def __init__(self, aggregates=None, table=None, time_field=None, emit_policy=None, key_field=None, **kwargs):
        self.aggregates = [dict(a) for a in aggregates or []]
        self.table, self.time_field, self.emit_policy, self.key_field = table, time_field, emit_policy, key_field
        self.name = kwargs.get("name")

    def do(self, event):
        raise LoweringError("AggregateByKey runs on the device over a whole frame (FeatureSet.ingest), not per event")


class _AggSpec:
    __slots__ = ("column", "kind", "ops", "period_ns", "windows_ns", "outs")

    def __init__(self, column, kind, ops, period_ns, windows_ns, outs):
        self.column, self.kind, self.ops, self.period_ns, self.windows_ns = column, kind, ops, period_ns, windows_ns
        self.outs = outs  # output column names in the C-ABI's order: op bits ascending, windows inner


class AggregationPlan:
    """an AggregateByKey step over the result columns of an IngestPlan (emit every event).  Everything the device does not
    compute is refused here, before any copy: no timestamp key or entities, sources that are not float32 / int32 result
    columns, unknown operations or units, a period that does not divide a window, another emit policy."""

    def __init__(self, step, plan, timestamp_key, entities):
        if not timestamp_key:
            raise LoweringError("an aggregation needs the feature set's timestamp_key: windows are event-time windows")
        if not entities:
            raise LoweringError("an aggregation needs the feature set's entities: it aggregates per key")
        ep = step.emit_policy
        if ep is not None and type(ep).__name__ != "EmitEveryEvent" and not (isinstance(ep, dict) and ep.get("mode") == "every_event"):
            raise LoweringError(f"emit policy {ep!r}: only EmitEveryEvent (the storey default) is lowered")
        if step.time_field not in (None, timestamp_key):
            raise LoweringError(f"aggregation time field {step.time_field!r} is not the feature set's timestamp_key")
        if dict(plan.schema).get(timestamp_key) != I64:
            raise LoweringError(f"timestamp_key {timestamp_key!r} must be a datetime64 column of the ingested frame")
        self.ts_slot = plan.prog.in_slot[timestamp_key]
        landing = {name: dt for name, _slot, dt in plan._landing()[0]}
        how = {name: h for name, _slot, h in plan.out}
        self.specs, self.out_names, self.sources = [], [], []
        for agg in step.aggregates:
            col = agg.get("column")
            if col in entities or col == timestamp_key:
                raise LoweringError(f"aggregation of {col!r}: entities and the timestamp are not aggregated")
            dt = landing.get(col)
            if dt is None or isinstance(how[col], tuple) and how[col][0] == "date" or dt not in (np.float32, np.int32):
                raise LoweringError(f"aggregation of {col!r}: the source must be a float32 or int32 result column of the graph")
            ops = list(dict.fromkeys(agg.get("operations") or []))
            bad = [o for o in ops if o not in nat.AGG_OPS]
            if not ops or bad:
                raise LoweringError(f"aggregation {agg.get('name')!r}: operations {bad or ops} (have {list(nat.AGG_OPS)})")
            windows = list(dict.fromkeys(agg.get("windows") or []))
            if not windows or len(windows) > _MAX_WINDOWS:
                raise LoweringError(f"aggregation {agg.get('name')!r}: 1 .. {_MAX_WINDOWS} windows")
            windows_ns = [_duration_ns(w, "window") for w in windows]
            period_ns = _duration_ns(agg["period"], "period") if agg.get("period") else 0
            if period_ns and any(w % period_ns for w in windows_ns):
                raise LoweringError(f"aggregation {agg.get('name')!r}: period {agg['period']} must divide every window {windows}")
            names = {(o, w): f"{agg['name']}_{o}_{w}" for o in ops for w in windows}
            self.out_names += [names[o, w] for o in ops for w in windows]  # feature_set.py:847-849
            by_bit = sorted(ops, key=nat.AGG_OPS.get)
            self.specs.append(_AggSpec(col, nat.COL_F32 if dt == np.float32 else nat.COL_I32, sum(nat.AGG_OPS[o] for o in ops),
                                       period_ns, windows_ns, [names[o, w] for o in by_bit for w in windows]))
            if col not in self.sources:
                self.sources.append(col)
        if len(self.specs) > _MAX_SPECS or len(self.sources) > _MAX_SOURCES:
            raise LoweringError(f"at most {_MAX_SPECS} aggregations over {_MAX_SOURCES} columns per feature set")
        taken = set(how)
        for name in self.out_names:
            if name in taken:
                raise LoweringError(f"aggregate column {name!r} collides with another column of the result")
            taken.add(name)
        self.counters = None
        self.stats = None

    def run(self, keys, ts, sources, n, outs):
        """keys / ts: int64 [n]; sources: {column: float32 / int32 [n]}; outs: {aggregate column: float64 [n]} (filled).
        Raises LoweringError after the run for late events, NaT timestamps or NaN values."""
        specs = [(sources[sp.column], sp.kind, sp.ops, sp.period_ns, sp.windows_ns, [outs[o] for o in sp.outs]) for sp in self.specs]
        self.counters, self.stats = aggregate_host(keys, ts, specs, n)
        self.check_counters()

    def run_device(self, d_keys, d_ts, n, d_sources, d_outs, d_counters):
        """one b2s_agg_run_device call over device addresses: sources {column: address}, outs {aggregate column: address of
        float64 [n]}; the three counters accumulate at d_counters (zeroed) for the caller to read and `check_counters`"""
        c_specs = (nat.AggSpec * len(self.specs))()
        keep = []
        for i, sp in enumerate(self.specs):
            win = np.ascontiguousarray(sp.windows_ns, dtype=np.int64)
            ptrs = (C.c_void_p * len(sp.outs))(*[d_outs[o] for o in sp.outs])
            keep += [win, ptrs]
            c_specs[i] = nat.AggSpec(d_sources[sp.column], sp.kind, sp.ops, sp.period_ns, len(win),
                                     win.ctypes.data_as(C.POINTER(C.c_int64)), ptrs)
        before = nat.launch_count()
        nat.check(nat.load().b2s_agg_run_device(d_keys, d_ts, n, c_specs, len(self.specs), d_counters, None))
        self.stats = {"rows": n, "kernels": nat.launch_count() - before}

    def check_counters(self):
        late, nat_rows, nans = (int(c) for c in self.counters)
        if late:
            raise LoweringError(f"{late} rows have a timestamp below the previous row of their key: late and out-of-order events "
                                "are not aggregated on the device (sort each key's rows by time)")
        if nat_rows:
            raise LoweringError(f"{nat_rows} rows have a NaT timestamp: they belong to no window")
        if nans:
            raise LoweringError(f"{nans} aggregated values are NaN: impute them before the aggregation")


def _convert(lib, ops, n, counters):
    """one b2s_cols_convert_device launch on the library stream"""
    arr = (nat.Convert * len(ops))(*ops)
    nat.check(lib.b2s_cols_convert_device(arr, len(ops), n, counters.ptr, counters.shape[0], None))


def aggregate_host(keys, ts, specs, n):
    """one b2s_agg_run_host call.  specs: [(source [n] float32 / int32, COL_* kind, op bits, period ns, [window ns],
    [float64 [n] output per (op bit ascending, window)])] -> (counters uint64 [3], stats dict)"""
    lib = nat.init() if n else nat.load()
    keys = np.ascontiguousarray(keys, dtype=np.int64)
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    c_specs = (nat.AggSpec * len(specs))()
    keep = []
    for i, (src, kind, ops, period_ns, windows_ns, arrays) in enumerate(specs):
        src = np.ascontiguousarray(src)
        win = np.ascontiguousarray(windows_ns, dtype=np.int64)
        ptrs = (C.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])
        keep += [src, win, ptrs]
        c_specs[i] = nat.AggSpec(src.ctypes.data, kind, ops, period_ns, len(win), win.ctypes.data_as(C.POINTER(C.c_int64)), ptrs)
    counters = np.zeros(3, dtype=np.uint64)
    stats = nat.Stats()
    nat.check(lib.b2s_agg_run_host(keys.ctypes.data, ts.ctypes.data, n, c_specs, len(specs), counters.ctypes.data, C.byref(stats)))
    return counters, stats.as_dict()


def _aggregation_key(graph):
    """what of the graph's aggregation steps a cached plan depends on"""
    return repr([(name, step.class_args) for name, step in graph.steps.items()
                 if str(getattr(step, "class_name", "") or "") == "storey.AggregateByKey"])


def lower_steps(steps, df_or_schema):
    schema = df_or_schema if isinstance(df_or_schema, list) else frame_schema(df_or_schema)
    prog = FrameProgram(schema)
    for s in steps:
        prog.apply(s)
    return prog.build()


# ------------------------------------------------------------------------------------------ FeatureSet mirror
class Entity:
    def __init__(self, name=None, value_type=None, description=None, labels=None):
        self.name, self.value_type, self.description, self.labels = name, value_type, description, labels or {}


class Feature:
    """mlrun/features.py:92-150: only what validation reads"""

    def __init__(self, value_type=None, dims=None, description=None, aggregate=None, name=None, validator=None,
                 default=None, labels=None):
        self.name, self.value_type, self.description, self.validator = name or "", value_type, description, validator
        self.default, self.labels = default, labels or {}
        self.aggregate = aggregate


class FeatureSet:
    """the part of mlrun.feature_store.FeatureSet the ingest path touches (feature_set.py:319-520, 1004-1090):
    a named transformation graph (`.graph`, `.add_step`/`graph.to`), entities that become the frame's index
    (ingestion.py:84-87 `entities_to_index`) and `ingest(df)`"""

    def __init__(self, name=None, description=None, entities=None, timestamp_key=None, engine=None, label_column=None,
                 relations=None, passthrough=None):
        from ..serving.graph import RootFlowStep

        self.name = name
        self.description = description
        self.entities = [Entity(e) if isinstance(e, str) else e for e in (entities or [])]
        self.timestamp_key = timestamp_key
        self.engine = engine or "storey"
        self.label_column = label_column
        self.passthrough = passthrough
        self.features = {}
        self._aggregations = {}
        self._graph = RootFlowStep()
        self._graph.engine = "sync"  # steps are only resolved here; the device plan replaces the executor
        self._plan = None
        self._plan_key = None

    @property
    def graph(self):
        return self._graph

    def __getitem__(self, name):
        return self.features[name]

    def __setitem__(self, key, item):
        self.add_feature(item, key)

    def add_feature(self, feature, name=None):
        """feature_set.py:646-656 -- `fset["bid"] = Feature(validator=MinMaxValidator(min=52, severity="info"))`"""
        name = name or feature.name
        if not name:
            raise MLRunInvalidArgumentError("feature name must be specified")
        feature.name = name
        self.features[name] = feature

    def add_step(self, *args, **kwargs):
        last = self._graph
        names = list(self._graph.steps.keys()) if hasattr(self._graph, "steps") else []
        if names:
            last = self._graph[names[-1]]
        return last.to(*args, **kwargs)

    @property
    def spec(self):
        """what the steps' `validate_args` read of a feature set (feature_set.py FeatureSetSpec)"""
        import types

        return types.SimpleNamespace(entities={e.name: e for e in self.entities}, label_column=self.label_column,
                                     timestamp_key=self.timestamp_key, graph=self._graph)

    def validate_steps(self, namespace=None):
        """ingest-time argument checks of the graph's steps (feature_set.py:508-534): every step class that has a
        `validate_args` classmethod sees the feature set and its own constructor arguments"""
        from . import transforms

        known = {k: getattr(transforms, k) for k in dir(transforms) if not k.startswith("_")}
        known.update(namespace or {})
        for step in self._graph.steps.values():
            obj = getattr(step, "_object", None)
            cls = type(obj) if obj is not None else known.get(str(step.class_name or "").rsplit(".", 1)[-1])
            check = getattr(cls, "validate_args", None)
            if check is None:
                continue
            args = dict(step.class_args or {})
            if obj is not None:  # a step added as an object: its arguments are its attributes
                args = {k: getattr(obj, k) for k in ("mapping", "features") if hasattr(obj, k)}
            check(self, **args)

    def _add_aggregation_to_existing(self, new_aggregation):
        """feature_set.py:689-713"""
        name = new_aggregation["name"]
        if name in self._aggregations:
            current_aggr = self._aggregations[name]
            if current_aggr["windows"] != new_aggregation["windows"]:
                raise MLRunInvalidArgumentError(
                    f"Aggregation with name {name} already exists but with window {current_aggr['windows']}. "
                    f"Please provide name for the aggregation")
            if current_aggr["period"] != new_aggregation["period"]:
                raise MLRunInvalidArgumentError(
                    f"Aggregation with name {name} already exists but with period {current_aggr['period']}. "
                    f"Please provide name for the aggregation")
            if current_aggr["column"] != new_aggregation["column"]:
                raise MLRunInvalidArgumentError(
                    f"Aggregation with name {name} already exists but for different column {current_aggr['column']}. "
                    f"Please provide name for the aggregation")
            # the reference takes list(set(...)), whose order varies between processes: the same operations, first-seen order
            current_aggr["operations"] = list(dict.fromkeys(current_aggr["operations"] + new_aggregation["operations"]))
            return
        self._aggregations[name] = new_aggregation

    def add_aggregation(self, column, operations, windows, period=None, name=None, step_name=None, after=None, before=None,
                        emit_policy=None):
        """feature_set.py:715-851 -- `fset.add_aggregation("ask", ["sum", "max"], "1h", "10m", name="asks")`: a
        storey.AggregateByKey step whose columns `{name}_{operation}_{window}` are computed on the device at ingest"""
        if isinstance(operations, str):
            raise MLRunInvalidArgumentError("Invalid parameters provided - operations must be a list.")
        name = name or column
        if isinstance(windows, str):
            windows = [windows]
        # FeatureAggregation(...).to_dict(): fields that are None are left out
        aggregation = {k: v for k, v in (("name", name), ("column", column), ("operations", list(operations)),
                                         ("windows", windows), ("period", period)) if v is not None}

        def upsert_feature(feature_name):
            if feature_name in self.features:
                self.features[feature_name].aggregate = True
            else:
                self.add_feature(Feature(name=column, aggregate=True, value_type="float"), feature_name)  # named by its key

        step_name = step_name or AGGREGATES_STEP
        graph = self._graph
        if step_name in graph.steps:
            step = graph.steps[step_name]
            self._add_aggregation_to_existing(aggregation)
            step.class_args["aggregates"] = list(self._aggregations.values())
            if emit_policy is not None:
                step.class_args["emit_policy"] = emit_policy
        else:
            self._aggregations[aggregation["name"]] = aggregation
            if before is None and after is None:
                after = "$prev"
            if self.engine and self.engine != "storey":
                raise LoweringError(f"aggregations of the {self.engine} engine are not lowered: use the storey engine")
            # the reference's storey step takes no emit policy (EmitEveryEvent is storey's default); one given here is kept
            # so that the lowering can refuse any other
            extra = {"emit_policy": emit_policy} if emit_policy is not None else {}
            step = graph.add_step(name=step_name, after=after, before=before, class_name="storey.AggregateByKey",
                                  time_field=self.timestamp_key, aggregates=[aggregation], table=".", **extra)
        for operation in operations:
            for window in windows:
                upsert_feature(f"{name}_{operation}_{window}")
        return step

    def _split_aggregation(self, objs):
        """the graph's objects -> (the steps of the columns plan, the AggregateByKey step or None)"""
        at = [i for i, o in enumerate(objs) if isinstance(o, AggregateByKey)]
        if not at:
            return objs, None
        if len(at) > 1:
            raise LoweringError("a second aggregation step is not lowered: add every aggregation to one step")
        if at[0] != len(objs) - 1:
            raise LoweringError(f"step {type(objs[at[0] + 1]).__name__} after the aggregation step is not lowered: the "
                                "aggregation must be the graph's last step")
        return objs[:-1], objs[-1]

    def _lower(self, namespace, df_or_schema):
        objs, agg = self._split_aggregation(self._step_objects(namespace))
        plan = lower_steps(objs, df_or_schema)
        if agg is not None:
            plan.agg = AggregationPlan(agg, plan, self.timestamp_key, [e.name for e in self.entities])
        return plan

    def _encoded_keys(self, frame):
        """the rows' 64-bit entity keys, as the point-in-time join encodes them (keys.py)"""
        from .keys import _encode_keys, _key_kind

        names = [e.name for e in self.entities]
        if frame is None or not all(k in frame.columns for k in names):
            raise LoweringError(f"the aggregation's entity columns {names} must all be in the ingested data")
        what = f"feature set {self.name}"
        kind = _key_kind(frame, names, what)
        keys = _encode_keys(frame, names, kind, what)
        if kind == "str" and len(np.unique(keys)) != len(set(frame[names[0]].to_numpy().tolist())):
            raise MLRunInvalidArgumentError(f"feature set {self.name}: two entity keys share a 64-bit hash")
        return keys

    def _step_objects(self, namespace):
        from ..serving.compiler import _chain, _transform_object
        from ..serving.host import create_graph_server
        from . import transforms

        ns = {k: getattr(transforms, k) for k in dir(transforms) if not k.startswith("_")}
        ns["storey.AggregateByKey"] = AggregateByKey
        ns.update(namespace or {})
        server = create_graph_server(graph=self._graph, parameters={})
        server.init_states(context=None, namespace=ns)
        server.init_object(ns)
        objs = [_transform_object(s) for s in _chain(self._graph)]
        for o in objs:
            # FeaturesetValidator.__init__ (steps.py:94-116) takes its validators from the feature set's features
            if type(o).__name__ == "FeaturesetValidator" and not o._validators and o.featureset in (".", self.name):
                o._validators = {k: f.validator for k, f in self.features.items()
                                 if f.validator is not None and (not o.columns or k in o.columns)}
        return objs

    def ingest(self, source=None, targets=None, namespace=None, return_df=True, reference_dtypes=False, **kwargs):
        """DataFrame -> transformed DataFrame through one device plan (targets are out of scope: pass none)"""
        if targets:
            raise LoweringError("targets are storage (out of scope): ingest returns the frame")
        from . import columnar

        if columnar.is_columnar(source) and columnar.is_device_source(source):
            batch = self._ingest_device(source, namespace, reference_dtypes)
            return batch if return_df else None
        if columnar.is_columnar(source):
            # columnar sources (dict of arrays, Arrow table / record batch, DLPack producers): no DataFrame on either side;
            # entity columns are carried through untouched (they would be the frame's index)
            cols = columnar.as_columns(source)
            keys = [e.name for e in self.entities if e.name in cols]
            carried = {k: cols.pop(k) for k in keys}
            schema = columnar.schema_of(cols)
            key = ("columns", schema, _aggregation_key(self._graph))
            if self._plan is None or not isinstance(self._plan_key[0], str) or self._plan_key != key:
                self.validate_steps(namespace)
                self._plan = self._lower(namespace, schema)
                self._plan_key = key
            enc = None
            if self._plan.agg is not None:
                import pandas as pd

                enc = self._encoded_keys(pd.DataFrame(carried, copy=False) if carried else None)
            batch = self._plan.run_columns(cols, reference_dtypes=reference_dtypes, keys=enc)
            batch.index = carried
            return batch if return_df else None
        if not (hasattr(source, "columns") and hasattr(source, "index")):
            raise MLRunInvalidArgumentError("illegal source")  # ingestion.py:77-78; only frames are taken here
        df = source
        keys = [e.name for e in self.entities]
        key_frame = None
        if keys and all(k in df.columns for k in keys):
            key_frame = df
            df = df.set_index(keys)
        agg_key = _aggregation_key(self._graph)
        if (self._plan is None or isinstance(self._plan_key[0], str) or not _same_labels_and_dtypes(df, self._plan_key)
                or self._plan_key[2] != agg_key):
            self.validate_steps(namespace)
            self._plan = self._lower(namespace, df)
            self._plan_key = (df.columns, list(df.dtypes), agg_key)
        enc = self._encoded_keys(key_frame) if self._plan.agg is not None else None
        out = self._plan.run(df, reference_dtypes=reference_dtypes, keys=enc)
        return out if return_df else None

    def _ingest_device(self, source, namespace, reference_dtypes):
        """CUDA columns -> DeviceColumnBatch: the columnar path with the data kept in HBM.  Everything refused is refused
        before any copy or launch."""
        from . import columnar

        if reference_dtypes:
            raise LoweringError("reference_dtypes=True widens integer results to int64, which no offline step takes: CUDA "
                                "columns are ingested with the device dtypes")
        cols = columnar.device_columns(source)
        keys = [e.name for e in self.entities if e.name in cols]
        carried = {k: cols.pop(k) for k in keys}
        ts_names = {self.timestamp_key} if self.timestamp_key else set()
        if any(str(c.dtype) == "int64" and k not in ts_names for k, c in cols.items()):
            for step in self._graph.steps.values():  # DateExtractor's timestamp_col, read off the graph as validate_steps does
                obj = getattr(step, "_object", None)
                cls = type(obj).__name__ if obj is not None else str(step.class_name or "").rsplit(".", 1)[-1]
                if cls == "DateExtractor":
                    col = getattr(obj, "timestamp_col", None) if obj is not None else (step.class_args or {}).get("timestamp_col")
                    ts_names.add(col or "timestamp")
        schema, dtypes = columnar.device_schema(cols, ts_names)
        for k, c in cols.items():
            c.dtype = dtypes[k]
        agg_key = _aggregation_key(self._graph)
        key_cols = None
        if agg_key != "[]" and self.entities:  # an aggregation step by name: its keys are refused before the plan is lowered
            key_cols = self._device_key_columns(carried)
        key = ("columns", schema, agg_key)
        if self._plan is None or not isinstance(self._plan_key[0], str) or self._plan_key != key:
            self.validate_steps(namespace)
            self._plan = self._lower(namespace, schema)
            self._plan_key = key
        if self._plan.agg is None:
            key_cols = None
        elif key_cols is None:  # the plan aggregates (whatever the step is called): the host path's check, at its place
            key_cols = self._device_key_columns(carried)
        held = list(cols.values()) + (key_cols or [])
        try:
            for c in held:
                c.acquire()
            batch = self._plan.run_device(cols, key_cols)
        finally:
            for c in held:
                c.release()
        batch.index = {k: c.obj for k, c in carried.items()}
        return batch

    def _device_key_columns(self, carried):
        """the entity key columns of CUDA columns, refused as `_encoded_keys` refuses them, and string keys (no string column
        lives on the device)"""
        from .keys import _key_kind

        names = [e.name for e in self.entities]
        if not names or not all(k in carried for k in names):
            raise LoweringError(f"the aggregation's entity columns {names} must all be in the ingested data")
        what = f"feature set {self.name}"
        for k in names:
            if carried[k].dtype.kind in "OSU":
                raise LoweringError(f"{what}: key {k!r} of dtype {carried[k].dtype} is a string key: there are no string "
                                    "columns on the device (hash them on the host)")
        _key_kind({k: np.empty(0, carried[k].dtype) for k in names}, names, what)
        return [carried[k] for k in names]

    @property
    def plan(self):
        return self._plan


def ingest(featureset=None, source=None, targets=None, namespace=None, return_df=True, **kwargs):
    """module-level spelling, mlrun.feature_store.api.ingest (feature_store/api.py:404-520)"""
    return featureset.ingest(source, targets=targets, namespace=namespace, return_df=return_df, **kwargs)
