"""Columnar sources and results of feature-set ingest: the DataFrame-free boundary (SURVEY.md 8(f) #1).

The reference's ingest walks a DataFrame one dict per row (`storey.DataframeSource`, mlrun/datastore/sources.py:886-895)
and re-assembles a DataFrame (`ReduceToDataFrame`, mlrun/datastore/targets.py:1856-1868).  The device plan is columnar on
both sides, so the cheapest boundary is columnar too: a mapping column -> contiguous array in, a `ColumnBatch` out, both
convertible to / from Arrow without copies.  At ~2.3 KB per row the path is PCIe bound; what decides its speed is whether the
buffers are pinned (`pinned_columns` / `ColumnBatch` are) and whether the frame is long enough to be pipelined.
"""

import ctypes as C

import numpy as np

from .. import _native as nat
from .ingest import F32, I32, I64, _INT_DTYPES, LoweringError


def is_columnar(source):
    """dict of arrays, pyarrow Table / RecordBatch, or a (Device)ColumnBatch (a DataFrame is not: it takes the frame path)"""
    if isinstance(source, (dict, ColumnBatch, DeviceColumnBatch)):
        return True
    mod = type(source).__module__.split(".")[0]
    return mod == "pyarrow" and hasattr(source, "column_names")


def _as_array(value, name):
    if isinstance(value, np.ndarray):
        return value
    if type(value).__module__.split(".")[0] == "pyarrow":  # ChunkedArray / Array: zero-copy when it has no nulls
        if hasattr(value, "combine_chunks") and getattr(value, "num_chunks", 1) != 1:
            value = value.combine_chunks()
        elif hasattr(value, "chunk"):
            value = value.chunk(0)
        if value.null_count:
            raise ValueError(f"column {name!r} has Arrow nulls: give float columns NaN (the Imputer's input) and fill the others")
        return value.to_numpy(zero_copy_only=True)
    if hasattr(value, "__dlpack__"):
        return np.from_dlpack(value)
    return np.asarray(value)


def as_columns(source):
    """-> {name: 1-D numpy array}, without copying where the producer allows it"""
    if isinstance(source, ColumnBatch):
        return dict(source.columns)
    if isinstance(source, dict):
        return {str(k): _as_array(v, k) for k, v in source.items()}
    if hasattr(source, "column_names"):  # pyarrow.Table / RecordBatch
        return {str(n): _as_array(source.column(n), n) for n in source.column_names}
    raise TypeError(f"{type(source).__name__} is not a columnar source")


def schema_of(columns):
    """[(name, kind)] like ingest.frame_schema, from arrays"""
    schema = []
    for name, a in columns.items():
        s = str(a.dtype)
        if s == "float32":
            kind = F32
        elif s in _INT_DTYPES:
            kind = I32
        elif s.startswith("datetime64") or s == "int64":
            if s == "int64":
                raise LoweringError(f"column {name!r} is int64: only timestamps (datetime64[ns]) are 8-byte columns; cast counters "
                                    "to int32 explicitly (a silent down-cast would change values)")
            kind = I64
        else:
            raise LoweringError(f"column {name!r} has dtype {s}: the device takes float32, (u)int8/16/32, bool and datetime64 columns")
        schema.append((str(name), kind))
    return schema


def pinned_columns(schema, n_rows):
    """{name: pinned (cudaMallocHost) array}: fill these instead of pageable arrays and the H2D copies run at PCIe speed
    (and can overlap the kernels).  `schema`: [(name, dtype)] or a mapping name -> dtype / array."""
    items = list(schema.items() if isinstance(schema, dict) else schema)
    dts = [(str(name), dt.dtype if hasattr(dt, "dtype") else np.dtype(dt)) for name, dt in items]
    # ONE pinned block, columns 64-byte aligned one after the other: neighbours of the same width sit at a constant pitch, which
    # lets b2s_cols_run_host move a row range of all of them with a single 2-D copy (the arrays keep the block alive)
    n_rows = int(n_rows)
    offs, off = [], 0
    for _name, dt in dts:
        offs.append(off)
        off += (n_rows * dt.itemsize + 63) // 64 * 64
    block = nat.pinned_empty((max(off, 64),), np.uint8)
    return {name: block[o: o + n_rows * dt.itemsize].view(dt) for (name, dt), o in zip(dts, offs)}


class ColumnBatch:
    """result of a columnar ingest: ordered {name: array}; the arrays are views of one pinned block that lives as long as
    any of them does.  `index` carries the entity columns of the source, untouched."""

    def __init__(self, columns, n_rows, block=None):
        self.columns = dict(columns)
        self.n_rows = int(n_rows)
        self.index = {}
        self._block = block

    def __getitem__(self, name):
        return self.columns[name]

    def __len__(self):
        return self.n_rows

    @property
    def names(self):
        return list(self.columns)

    def to_arrow(self):
        """pyarrow.Table over the same memory (numeric columns without nulls convert without a copy)"""
        import pyarrow as pa

        cols = {**self.index, **self.columns}
        return pa.table({k: pa.array(v) for k, v in cols.items()})

    def to_pandas(self):
        import pandas as pd

        frame = pd.DataFrame(self.columns, copy=False)
        if self.index:
            frame.index = pd.MultiIndex.from_arrays(list(self.index.values()), names=list(self.index)) if len(self.index) > 1 \
                else pd.Index(next(iter(self.index.values())), name=next(iter(self.index)))
        return frame


# ------------------------------------------------------------------------------------------ device-resident columns
_KDLCUDA = 2
# DLPack (code, bits) -> numpy dtype
_DL_DTYPES = {(0, 8): "int8", (0, 16): "int16", (0, 32): "int32", (0, 64): "int64", (1, 8): "uint8", (1, 16): "uint16",
              (1, 32): "uint32", (1, 64): "uint64", (2, 16): "float16", (2, 32): "float32", (2, 64): "float64", (6, 8): "bool"}


class _DLDataType(C.Structure):
    _fields_ = [("code", C.c_uint8), ("bits", C.c_uint8), ("lanes", C.c_uint16)]


class _DLTensor(C.Structure):
    _fields_ = [("data", C.c_void_p), ("device_type", C.c_int32), ("device_id", C.c_int32), ("ndim", C.c_int32),
                ("dtype", _DLDataType), ("shape", C.POINTER(C.c_int64)), ("strides", C.POINTER(C.c_int64)),
                ("byte_offset", C.c_uint64)]


_capsule_get = C.PyDLL(None)["PyCapsule_GetPointer"]  # its own function object (see _native)
_capsule_get.restype, _capsule_get.argtypes = C.c_void_p, [C.py_object, C.c_char_p]


def is_device_column(value):
    """a CUDA column: exposes __cuda_array_interface__, or DLPack on a kDLCUDA device"""
    if isinstance(value, (np.ndarray, DeviceColumn)):
        return isinstance(value, DeviceColumn)
    if hasattr(value, "__dlpack_device__"):
        return int(value.__dlpack_device__()[0]) == _KDLCUDA
    try:
        return hasattr(value, "__cuda_array_interface__")
    except Exception:  # noqa: BLE001 -- a producer whose interface raises is not a CUDA column
        return False


def is_device_source(source):
    """True when every column of a columnar source is a CUDA column, False when none is; ValueError for a mix"""
    if isinstance(source, DeviceColumnBatch):
        return True
    if not isinstance(source, dict) or not source:
        return False
    on = [str(k) for k, v in source.items() if is_device_column(v)]
    if on and len(on) != len(source):
        off = [str(k) for k in source if str(k) not in on]
        raise ValueError(f"columns {on} are CUDA columns and {off} are host columns: give all columns on one side")
    return bool(on)


def _capsule_tensor(capsule, name):
    """the DLTensor of an unconsumed DLPack capsule -> (tensor, numpy dtype, shape, element strides or None)"""
    t = _DLTensor.from_address(_capsule_get(capsule, b"dltensor"))
    dt = _DL_DTYPES.get((t.dtype.code, t.dtype.bits)) if t.dtype.lanes == 1 else None
    if dt is None:
        raise ValueError(f"column {name!r}: DLPack dtype code {t.dtype.code} bits {t.dtype.bits} lanes {t.dtype.lanes} is not "
                         "a numeric column dtype")
    shape = tuple(t.shape[i] for i in range(t.ndim))
    strides = tuple(t.strides[i] for i in range(t.ndim)) if t.strides else None
    return t, np.dtype(dt), shape, strides


class DeviceColumn:
    """one 1-D C-contiguous column in device memory as its producer exported it.  Construction reads what the producer
    states (shape, strides, dtype, device) without touching the library: from the CUDA array interface, or else from a
    DLPack capsule taken with stream=-1 (no synchronisation) and dropped at once.  `acquire` orders the library stream
    behind the producer (DLPack: the producer makes the stream it is given wait; CUDA array interface v3: the library stream
    waits for `stream`) and holds a DLPack capsule until `release`.

    With matrix=True the object is any array instead: `shape`, `ndim` and byte `strides` are recorded as the producer states
    them and the caller judges them (a row matrix: `plan.check_rows`)."""

    def __init__(self, obj, name, matrix=False):
        self.obj, self.name, self.matrix = obj, name, matrix
        self.ptr = None
        self._capsule = None
        self._cai = None
        self.device = None
        if hasattr(obj, "__dlpack_device__"):
            kind, self.device = (int(x) for x in obj.__dlpack_device__())
            if kind != _KDLCUDA:
                raise ValueError(f"column {name!r} is not in CUDA device memory (DLPack device type {kind})")
        cai = getattr(obj, "__cuda_array_interface__", None)
        if cai is not None:
            self._cai = cai
            self._shape(tuple(cai["shape"]), cai.get("strides"), np.dtype(cai["typestr"]), byte_strides=True)
            if cai.get("mask") is not None:
                raise ValueError(f"column {name!r} has a mask: give float columns NaN (the Imputer's input) and fill the others")
        elif not hasattr(obj, "__dlpack__"):
            raise TypeError(f"column {name!r} exposes neither __cuda_array_interface__ nor DLPack")
        if self.device is not None and self.device != nat.library_device():
            raise ValueError(f"column {name!r} is on CUDA device {self.device}; the library runs on device {nat.library_device()}")
        if cai is None:
            _t, dt, shape, strides = _capsule_tensor(self._take(-1), name)  # dropped here: its deleter runs when collected
            self._shape(shape, strides, dt, byte_strides=False)

    def _take(self, stream):
        try:
            return self.obj.__dlpack__(stream=stream)
        except TypeError:  # producers that take no stream argument hand over data that is ready
            return self.obj.__dlpack__()

    def _shape(self, shape, strides, dtype, byte_strides):
        if self.matrix:
            self.dtype, self.shape = dtype, tuple(int(d) for d in shape)
            if strides is None:  # C order
                strides = [dtype.itemsize * int(np.prod(self.shape[i + 1:])) for i in range(len(self.shape))]
            elif not byte_strides:
                strides = [s * dtype.itemsize for s in strides]
            self.strides, self.ndim = tuple(int(s) for s in strides), len(self.shape)
            self.n = self.shape[0] if self.shape else 1
            return
        if len(shape) != 1:
            raise ValueError(f"column {self.name!r}: expected a 1-D column, got shape {shape}")
        step = dtype.itemsize if byte_strides else 1
        if strides is not None and shape[0] > 1 and tuple(strides) != (step,):
            raise ValueError(f"column {self.name!r} is not C-contiguous (strides {tuple(strides)}): make it contiguous first")
        self.dtype, self.n = dtype, int(shape[0])

    def acquire(self):
        if self.ptr is not None:
            return self
        if hasattr(self.obj, "__dlpack__"):
            capsule = self._take(nat.init().b2s_stream())
            t, dt, shape, strides = _capsule_tensor(capsule, self.name)
            if t.device_type != _KDLCUDA or t.device_id != nat.library_device():
                raise ValueError(f"column {self.name!r} is on DLPack device ({t.device_type}, {t.device_id}); the library runs "
                                 f"on CUDA device {nat.library_device()}")
            described = self.dtype
            self._shape(shape, strides, dt, byte_strides=False)
            if described.kind == "M" and self.dtype == np.int64:
                self.dtype = described  # DLPack has no timestamps: the interface or the set named it datetime64[ns]
            self._capsule = capsule
            self.ptr = (t.data or 0) + t.byte_offset
            return self
        lib = nat.init()
        ptr = int(self._cai["data"][0] or 0)
        if ptr and self.n:
            dev = C.c_int32()
            nat.check(lib.b2s_pointer_device(ptr, C.byref(dev)))
            if dev.value != nat.library_device():
                where = "host memory" if dev.value < 0 else f"CUDA device {dev.value}"
                raise ValueError(f"column {self.name!r} is in {where}; the library runs on device {nat.library_device()}")
        stream = self._cai.get("stream") if int(self._cai.get("version", 2)) >= 3 else None
        if stream is not None:
            nat.check(lib.b2s_stream_wait(int(stream)))
        self.ptr = ptr
        return self

    def release(self):
        self._capsule = None  # an unconsumed capsule calls its producer's deleter when collected
        self.ptr = None

    def numpy(self):
        """a host copy (the producer's writes are awaited as for a run)"""
        self.acquire()
        try:
            out = np.empty(self.n, dtype=self.dtype)
            if out.nbytes:
                nat.check(nat.load().b2s_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes))
            return out
        finally:
            self.release()


def device_columns(source):
    """-> {name: DeviceColumn} of a source whose columns are all CUDA columns (described, not yet acquired)"""
    if isinstance(source, DeviceColumnBatch):
        return {**{k: DeviceColumn(v, k) for k, v in source.index.items()}, **{k: DeviceColumn(v, k) for k, v in source.columns.items()}}
    return {str(k): DeviceColumn(v, str(k)) for k, v in source.items()}


def device_schema(cols, timestamp_names):
    """schema_of for CUDA columns: torch has no datetime dtype, so an int64 column is a datetime64[ns] column when it is
    named in `timestamp_names` (the set's timestamp_key, DateExtractor timestamp columns); every other int64 is refused as
    on the host"""
    class _Dt:
        def __init__(self, dtype):
            self.dtype = dtype

    known = {}
    for name, c in cols.items():
        dt = c.dtype
        if str(dt) == "int64" and name in timestamp_names:
            dt = np.dtype("datetime64[ns]")
        known[name] = _Dt(dt)
    schema = schema_of(known)
    return schema, {name: d.dtype for name, d in known.items()}


class DeviceColumnBatch:
    """result of an ingest of CUDA columns: ordered {name: DeviceArray} in HBM, views of library allocations that live as
    long as any view does.  `index` carries the source's entity columns, untouched (the caller's objects)."""

    def __init__(self, columns, n_rows, index=None):
        self.columns = dict(columns)
        self.n_rows = int(n_rows)
        self.index = dict(index or {})

    def __getitem__(self, name):
        return self.columns[name]

    def __len__(self):
        return self.n_rows

    @property
    def names(self):
        return list(self.columns)

    def to_host(self):
        """the equal ColumnBatch (one D2H copy per column)"""
        out = ColumnBatch({k: v.numpy() for k, v in self.columns.items()}, self.n_rows)
        out.index = {k: DeviceColumn(v, k).numpy() for k, v in self.index.items()}
        return out
