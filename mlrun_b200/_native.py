"""ctypes binding of libb200serve.so (include/b200serve.h).

There is no CPU fallback: if the library is missing, or no GPU is present when a device call is made,
a `NativeError` is raised.  Loading the library itself does not need a GPU (the CPU test-suite checks
that every symbol of the header is exported).
"""

import ctypes as C
import collections
import os
import threading
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200serve.so")

# mirrors of the header's constants
OUT_COPY, OUT_ONEHOT = 0, 1
LINK_IDENTITY, LINK_BINARY_GT, LINK_BINARY_GE, LINK_ARGMAX = 0, 1, 2, 3
VOTE_NONE, VOTE_MEAN, VOTE_MAJORITY = 0, 1, 2
ROW_NONFINITE_INPUT, ROW_BAD_LABEL, ROW_UNKNOWN_KEY = 1, 2, 4
CMP_LE, CMP_LT = 0, 1          # left when x <= threshold (scikit-learn, LightGBM) | x < threshold (xgboost)
NAN_ERROR, NAN_DEFAULT_CHILD = 0, 1
CAT_NONNEG, CAT_TRUNC = 0, 1   # a valid category code is x >= 0 (xgboost) | x > -1, trunc(x) >= 0 (LightGBM)
COL_F32, COL_I32, COL_I64 = 0, 1, 2
# B2S_KERNEL_* (b2s_plan_last_kernel) -> name
KERNELS = {0: None, 1: "dense", 2: "trees3/tma", 3: "trees3", 6: "rowthread/tma", 7: "rowthread/ldgsts",
           8: "rowthread/host", 10: "rows", 11: "store", 12: "trees3_cat/tma", 13: "trees3_cat", 14: "rows_cat",
           15: "rowthread/bulk"}
DATE_PARTS = {"year": 0, "month": 1, "day": 2, "hour": 3, "minute": 4, "second": 5, "day_of_week": 6, "dayofweek": 6,
              "weekday": 6, "day_of_year": 7, "dayofyear": 7, "quarter": 8, "is_leap_year": 9, "days_in_month": 10,
              "daysinmonth": 10, "is_month_start": 11, "is_month_end": 12, "is_quarter_start": 13, "is_quarter_end": 14,
              "is_year_start": 15, "is_year_end": 16, "week": 17, "weekofyear": 17}
DATE_BOOL_PARTS = {9, 11, 12, 13, 14, 15, 16}


class NativeError(RuntimeError):
    """the CUDA engine is unavailable or a C-ABI call failed"""


class Stats(C.Structure):
    _fields_ = [("rows", C.c_int64), ("h2d_ms", C.c_float), ("kernel_ms", C.c_float), ("d2h_ms", C.c_float),
                ("queue_us", C.c_float), ("kernels", C.c_int32), ("nonfinite_rows", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class DevInfo(C.Structure):
    _fields_ = [("ordinal", C.c_int32), ("sm_count", C.c_int32), ("cc_major", C.c_int32), ("cc_minor", C.c_int32),
                ("total_mem", C.c_int64), ("l2_bytes", C.c_int64), ("smem_per_block_optin", C.c_int64),
                ("name", C.c_char * 128)]


_vp, _i32, _i64, _u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_pi32, _pf32, _pf64 = C.POINTER(C.c_int32), C.POINTER(C.c_float), C.POINTER(C.c_double)


class PitOut(C.Structure):
    _fields_ = [("src_word", _i32), ("bytes", _i32), ("miss", _u64), ("out", _vp)]


class PitSet(C.Structure):
    _fields_ = [("index", _vp), ("keys", _vp), ("asof", _i32), ("n_out", _i32), ("outs", C.POINTER(PitOut)),
                ("ts_out", _vp), ("found", _vp)]


class PitCol(C.Structure):
    _fields_ = [("src", _vp), ("dst", _vp), ("bytes", _i32)]


PIT_LABEL_FOUND, PIT_LABEL_NAN, PIT_LABEL_NAT = 0, 1, 2


class PitLabel(C.Structure):
    _fields_ = [("set", _i32), ("out", _i32), ("kind", _i32)]


PIT_FEAT_FLOAT, PIT_FEAT_INT, PIT_FEAT_UINT, PIT_FEAT_BOOL = 0, 1, 2, 3


class PitFeat(C.Structure):
    _fields_ = [("set", _i32), ("out", _i32), ("bytes", _i32), ("kind", _i32)]


class PitTensors(C.Structure):
    _fields_ = [("features", _vp), ("label", _vp), ("order", _vp), ("kept", _i64)]


# B2S_AGG_* operation bits, in the order of the outputs of one aggregation
AGG_OPS = {"count": 1, "sum": 2, "sqr": 4, "max": 8, "min": 16, "first": 32, "last": 64, "avg": 128, "stdvar": 256, "stddev": 512}


class AggSpec(C.Structure):
    _fields_ = [("src", _vp), ("kind", _i32), ("ops", C.c_uint32), ("period_ns", _i64), ("n_windows", _i32),
                ("windows_ns", C.POINTER(_i64)), ("outs", C.POINTER(_vp))]

# B2S_CONV_* kinds of b2s_cols_convert_device
CONV_COPY4, CONV_COPY8, CONV_I8_I32, CONV_U8_I32, CONV_I16_I32, CONV_U16_I32 = 0, 1, 2, 3, 4, 5
CONV_I32_F64, CONV_F32_I32, CONV_DATE_F64, CONV_I32_BOOL, CONV_CHECK_F32 = 6, 7, 8, 9, 10


class Convert(C.Structure):
    _fields_ = [("src", _vp), ("dst", _vp), ("kind", _i32), ("counter", _i32)]


class KeyCol(C.Structure):
    _fields_ = [("src", _vp), ("bytes", _i32), ("is_signed", _i32)]


# B2S_TCOL_* kinds of b2s_table_col
TCOL_FLOAT, TCOL_INT, TCOL_UINT, TCOL_BOOL = 0, 1, 2, 3


class TableCol(C.Structure):
    _fields_ = [("src", _vp), ("bytes", _i32), ("kind", _i32)]


# name -> (restype, argtypes); the single source of truth for the exported surface
SIGNATURES = {
    "b2s_version": (C.c_int, []),
    "b2s_last_error": (C.c_char_p, []),
    "b2s_init": (C.c_int, [C.c_int, C.c_char_p]),
    "b2s_shutdown": (C.c_int, []),
    "b2s_device_info": (C.c_int, [C.POINTER(DevInfo)]),
    "b2s_launch_count": (_i64, []),
    "b2s_plan_create": (C.c_int, [_i32, C.POINTER(_vp)]),
    "b2s_plan_destroy": (C.c_int, [_vp]),
    "b2s_plan_set_impute": (C.c_int, [_vp, _pi32, _pf32, _i32]),
    "b2s_plan_add_value_map": (C.c_int, [_vp, _i32, _pf32, _pf32, _i32]),
    "b2s_plan_add_range_map": (C.c_int, [_vp, _i32, _pf32, _pf32, _pf32, _i32]),
    "b2s_plan_set_output_schema": (C.c_int, [_vp, _pi32, _pi32, _pf32, _i32]),
    "b2s_plan_add_linear_model": (C.c_int, [_vp, _pf64, _pf64, _i32, _i32, _pi32, _i32]),
    "b2s_plan_add_tree_model": (C.c_int, [_vp, _i32, _pi32, _pi32, _pf32, _pi32, _pi32, _pf64, _pi32, _pf64, _pf64,
                                          _i32, _i32, _pi32, _i32]),
    "b2s_plan_add_tree_model_ex": (C.c_int, [_vp, _i32, _pi32, _pi32, _pf32, _pi32, _pi32, _pf64, _pi32, _pf64, _pf64,
                                             _i32, _i32, _pi32, _i32, _i32, C.POINTER(C.c_uint8), _i32]),
    "b2s_plan_add_tree_model_cat": (C.c_int, [_vp, _i32, _pi32, _pi32, _pf32, _pi32, _pi32, _pf64, _pi32, _pf64, _pf64,
                                              _i32, _i32, _pi32, _i32, _i32, C.POINTER(C.c_uint8), _i32,
                                              _pi32, _pi32, _i32, C.POINTER(C.c_uint32), _i32, _i32]),
    "b2s_plan_set_vote": (C.c_int, [_vp, _i32, _pf64, _i32]),
    "b2s_plan_finalize": (C.c_int, [_vp]),
    "b2s_plan_out_info": (C.c_int, [_vp, _pi32, _pi32]),
    "b2s_plan_kernel": (C.c_char_p, [_vp]),
    "b2s_plan_last_kernel": (_i32, [_vp]),
    "b2s_run_device": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _vp]),
    "b2s_run_columns_device": (C.c_int, [_vp, C.POINTER(TableCol), _i32, _i64, _vp, _vp, C.POINTER(Stats), _vp]),
    "b2s_run_host": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _i64, _vp, C.POINTER(Stats)]),
    "b2s_submit": (C.c_int, [_vp, _vp, _i64, _i64, C.POINTER(_u64)]),
    "b2s_wait": (C.c_int, [_vp, _u64, _vp, _i64, _vp, C.POINTER(Stats)]),
    "b2s_flush": (C.c_int, [_vp]),
    "b2s_plan_set_ring": (C.c_int, [_vp, _i32, _i64, _i32]),
    "b2s_ring_bench": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _i32, C.c_double, C.POINTER(_i64), C.POINTER(C.c_double),
                                 C.POINTER(C.c_double)]),
    "b2s_plan_set_merge_targets": (C.c_int, [_vp, C.POINTER(_vp), _i32, _i64]),
    "b2s_comm_create": (C.c_int, [_i32, _i32, _i64, _i32, C.POINTER(_vp)]),
    "b2s_comm_handle": (C.c_int, [_vp, _vp]),
    "b2s_comm_connect": (C.c_int, [_vp, _vp]),
    "b2s_plan_attach_comm": (C.c_int, [_vp, _vp]),
    "b2s_comm_wait": (C.c_int, [_vp, _vp, C.POINTER(_vp), C.POINTER(C.c_uint32)]),
    "b2s_comm_wait_lag": (C.c_int, [_vp, _vp, C.c_int32, C.POINTER(_vp), C.POINTER(C.c_uint32)]),
    "b2s_comm_set_fused_wait": (C.c_int, [_vp, C.c_int32]),
    "b2s_comm_check": (C.c_int, [_vp]),
    "b2s_comm_destroy": (C.c_int, [_vp]),
    "b2s_ipc_export": (C.c_int, [_vp, _vp]),
    "b2s_ipc_open": (C.c_int, [_vp, C.POINTER(_vp)]),
    "b2s_ipc_close": (C.c_int, [_vp]),
    "b2s_alloc_pinned": (_vp, [C.c_size_t]),
    "b2s_free_pinned": (C.c_int, [_vp]),
    "b2s_device_alloc": (_vp, [C.c_size_t]),
    "b2s_device_free": (C.c_int, [_vp]),
    "b2s_memcpy_h2d": (C.c_int, [_vp, _vp, C.c_size_t]),
    "b2s_memcpy_d2h": (C.c_int, [_vp, _vp, C.c_size_t]),
    "b2s_device_sync": (C.c_int, []),
    "b2s_time_device": (C.c_int, [_vp, C.POINTER(_vp), _i32, _i64, _i64, _vp, _i32, _pf32]),
    # columnar ingest
    "b2s_cols_create": (C.c_int, [_i32, C.POINTER(_vp)]),
    "b2s_cols_destroy": (C.c_int, [_vp]),
    "b2s_cols_add_copy": (C.c_int, [_vp, _i32, _i32, _i32, C.c_float, _i32, _i32, C.c_double, C.c_double, _pi32, _pi32]),
    "b2s_cols_add_range_map": (C.c_int, [_vp, _i32, _i32, _i32, C.c_float, _pf64, _pf64, _pf64, _i32, _i32, C.c_double,
                                         C.c_double, _pi32, _pi32, _pi32]),
    "b2s_cols_add_value_map": (C.c_int, [_vp, _i32, _i32, _i32, C.c_float, _pf64, _pf64, _i32, _i32, C.c_double, C.c_double,
                                         _pi32, _pi32, _pi32]),
    "b2s_cols_add_onehot": (C.c_int, [_vp, _i32, _i32, _i32, C.c_float, _pf64, _i32, _pi32, _pi32]),
    "b2s_cols_add_date_part": (C.c_int, [_vp, _i32, _i32, _pi32, _pi32]),
    "b2s_cols_finalize": (C.c_int, [_vp]),
    "b2s_cols_info": (C.c_int, [_vp, _pi32, _pi32]),
    "b2s_cols_run_device": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _i64, _vp, _vp]),
    "b2s_cols_run_host": (C.c_int, [_vp, C.POINTER(_vp), _i64, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(Stats)]),
    # online feature table
    "b2s_table_create": (C.c_int, [C.POINTER(_i64), _i64, _pf32, _i32, _pf32, C.POINTER(_vp)]),
    "b2s_table_destroy": (C.c_int, [_vp]),
    "b2s_table_info": (C.c_int, [_vp, C.POINTER(_i64), _pi32, C.POINTER(_i64)]),
    "b2s_table_lookup_device": (C.c_int, [_vp, _vp, _i64, _vp, _i64, _vp, _vp]),
    "b2s_table_lookup_host": (C.c_int, [_vp, C.POINTER(_i64), _i64, _pf32, _pi32, C.POINTER(Stats)]),
    "b2s_table_enrich_device": (C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp]),
    "b2s_table_enrich_host": (C.c_int, [_vp, _vp, C.POINTER(_i64), _i64, _vp, _i64, _pi32, C.POINTER(Stats)]),
    "b2s_table_time_device": (C.c_int, [_vp, C.POINTER(_vp), _i32, _i64, _vp, _i64, _vp, _i32, _pf32]),
    "b2s_hash_strings": (C.c_int, [C.c_char_p, C.POINTER(_i64), _i64, C.POINTER(_i64)]),
    "b2s_table_create_device": (C.c_int, [_vp, _i64, C.POINTER(TableCol), _i32, _pf32, C.POINTER(_vp)]),
    "b2s_table_stats_device": (C.c_int, [C.POINTER(TableCol), _i32, _i64, _pf32, _vp]),
    "b2s_table_label_keys_device": (C.c_int, [_vp, _i64, C.POINTER(TableCol), C.POINTER(_i64), C.POINTER(_i64), _vp]),
    "b2s_table_mark_unknown_device": (C.c_int, [_vp, _vp, _i64, _vp]),
    # point-in-time (as-of) joins
    "b2s_pit_index_create": (C.c_int, [_vp, _vp, _i64, C.POINTER(_vp), _pi32, _i32, C.POINTER(_vp)]),
    "b2s_pit_index_create_device": (C.c_int, [_vp, _vp, _i64, C.POINTER(_vp), _pi32, _i32, C.POINTER(_vp)]),
    "b2s_pit_index_destroy": (C.c_int, [_vp]),
    "b2s_pit_index_info": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), _pi32, C.POINTER(_i64)]),
    "b2s_pit_join_device": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, _vp, _vp, _vp]),
    "b2s_pit_join_host": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, _vp, _vp, C.POINTER(Stats)]),
    "b2s_pit_train_device": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, C.POINTER(PitLabel), _vp, _vp,
                                       _vp, _vp]),
    "b2s_pit_train_host": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, C.POINTER(PitLabel), _vp, _vp, _vp,
                                     _pf32, C.POINTER(Stats)]),
    "b2s_pit_train_pack": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, C.POINTER(PitLabel),
                                     C.POINTER(PitFeat), _i32, C.POINTER(PitFeat), _i32, C.POINTER(PitTensors), _pf32,
                                     C.POINTER(Stats)]),
    "b2s_pit_train_pack_device": (C.c_int, [_vp, _i64, C.POINTER(PitSet), _i32, C.POINTER(PitCol), _i32, C.POINTER(PitLabel),
                                            C.POINTER(PitFeat), _i32, C.POINTER(PitFeat), _i32, C.POINTER(PitTensors), _pf32,
                                            C.POINTER(Stats)]),
    # device arrays handed to the caller
    "b2s_darray_info": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_i64)]),
    "b2s_darray_release": (C.c_int, [_vp]),
    "b2s_darray_dlpack": (_vp, [_vp, _i32, C.POINTER(_i64), _i32, _i32]),
    "b2s_dlpack_delete": (C.c_int, [_vp]),
    "b2s_darray_live": (_i64, []),
    "b2s_darray_alloc": (C.c_int, [_i64, _i32, C.POINTER(_vp)]),
    "b2s_darray_view": (C.c_int, [_vp, _i64, _i64, C.POINTER(_vp)]),
    # feature-set ingest of device-resident columns
    "b2s_stream": (_vp, []),
    "b2s_stream_wait": (C.c_int, [_vp]),
    "b2s_pointer_device": (C.c_int, [_vp, _pi32]),
    "b2s_cols_convert_device": (C.c_int, [C.POINTER(Convert), _i32, _i64, _vp, _i32, _vp]),
    "b2s_keys_encode_device": (C.c_int, [C.POINTER(KeyCol), _i32, _i64, _vp, _vp]),
    "b2s_keys_hash_decimal_device": (C.c_int, [C.POINTER(KeyCol), _i32, _i64, _vp, _vp]),
    "b2s_ts_profile_device": (C.c_int, [_vp, _i64, C.POINTER(_i64), _vp]),
    # windowed aggregations
    "b2s_agg_run_device": (C.c_int, [_vp, _vp, _i64, C.POINTER(AggSpec), _i32, _vp, _vp]),
    "b2s_agg_run_host": (C.c_int, [_vp, _vp, _i64, C.POINTER(AggSpec), _i32, _vp, C.POINTER(Stats)]),
    "b2s_agg_time_device": (C.c_int, [_vp, _vp, _i64, C.POINTER(AggSpec), _i32, _vp, _i32, _pf32, _pf32]),
    # body codec
    "b2s_json_parse_inputs": (C.c_int, [C.c_char_p, _i64, _pf32, _i64, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64),
                                        C.POINTER(_i64)]),
    "b2s_json_format_outputs": (C.c_int, [_vp, _i32, _i64, _i64, _i32, C.c_char_p, _i64, C.POINTER(_i64)]),
    "b2s_cols_time_device": (C.c_int, [_vp, C.POINTER(_vp), _i32, _i64, _i64, _vp, _i64, _vp, _i32, _pf32]),
}

_lib = None
_lock = threading.Lock()
_inited = False


def load():
    """dlopen the library (no GPU needed) and declare every signature"""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(
                    f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                    "(nvcc, sm_90a). mlrun_b200 has no CPU fallback for device steps."
                )
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        msg = load().b2s_last_error()
        raise NativeError(f"b200serve error {rc}: {msg.decode() if msg else ''}")


def init(device=None, cfg=None):
    """bring up the device once per process (device ordinal defaults to LOCAL_RANK or 0)"""
    global _inited
    lib = load()
    if _inited:
        return lib
    with _lock:
        if not _inited:
            if device is None:
                device = int(os.environ.get("LOCAL_RANK", "0"))
            cfg = cfg or os.environ.get("B200SERVE_CFG", "")
            check(lib.b2s_init(int(device), cfg.encode() if cfg else None))
            _inited = True
    return lib


def device_info():
    lib = init()
    info = DevInfo()
    check(lib.b2s_device_info(C.byref(info)))
    return {"name": info.name.decode(), "sm_count": info.sm_count, "cc": (info.cc_major, info.cc_minor),
            "total_mem": info.total_mem, "l2_bytes": info.l2_bytes, "smem_optin": info.smem_per_block_optin}


def launch_count():
    return int(load().b2s_launch_count())


def ptr(arr):
    """address of a numpy array's first element, 3x cheaper than `arr.ctypes.data` (which builds a helper object per call:
    1.2 us, three of them per serving call); read-only, empty and non-contiguous arrays take the ordinary route"""
    try:
        return C.addressof(C.c_char.from_buffer(arr))
    except (TypeError, ValueError):
        return arr.ctypes.data


def _p(arr, ctype):
    return arr.ctypes.data_as(C.POINTER(ctype)) if arr is not None else None


class DeviceBuffer:
    """a cudaMalloc'd buffer owned by the library (ctypes callers need no other CUDA binding)"""

    def __init__(self, nbytes):
        lib = init()
        self.nbytes = int(nbytes)
        self.ptr = lib.b2s_device_alloc(self.nbytes)
        if not self.ptr:
            raise NativeError(f"device alloc of {nbytes} bytes failed: {lib.b2s_last_error().decode()}")

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        check(load().b2s_memcpy_h2d(self.ptr, arr.ctypes.data, arr.nbytes))
        return self

    def download(self, dtype, shape):
        out = np.empty(shape, dtype=dtype)
        check(load().b2s_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes))
        return out

    def free(self):
        if self.ptr:
            load().b2s_device_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def ipc_export(dptr):
    """64-byte CUDA IPC handle of a buffer from DeviceBuffer / b2s_device_alloc"""
    buf = C.create_string_buffer(64)
    check(load().b2s_ipc_export(dptr, buf))
    return bytes(buf.raw)


def ipc_open(handle):
    out = C.c_void_p()
    check(load().b2s_ipc_open(C.create_string_buffer(handle, 64), C.byref(out)))
    return out.value


def pinned_empty(shape, dtype=np.float32):
    """numpy array over cudaMallocHost memory (kept alive by the returned array's base object)"""
    lib = init()
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    ptr = lib.b2s_alloc_pinned(max(nbytes, 1))
    if not ptr:
        raise NativeError("pinned alloc failed")
    buf = (C.c_char * max(nbytes, 1)).from_address(ptr)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    # the block goes back to the driver when the last array over it is collected (arrays keep `buf` alive as their base)
    weakref.finalize(buf, _free_pinned, ptr)
    return arr


def _free_pinned(ptr):
    try:
        if _lib is not None:
            _lib.b2s_free_pinned(ptr)
    except Exception:
        pass


class _Lease:
    """keeps a pinned block out of the pool while any numpy array over it is alive (the arrays' base buffer holds it)"""

    def __init__(self, pool, ptr, size):
        self.pool, self.ptr, self.size = pool, ptr, size

    def __del__(self):
        # may run inside a garbage-collection pass triggered while take() holds the pool lock on this very thread:
        # only append to a deque here (atomic, lock free); take() drains it
        try:
            self.pool._returned.append((self.ptr, self.size))
        except Exception:
            pass


class PinnedPool:
    """cudaMallocHost blocks for results that go straight into numpy / DataFrame columns: D2H copies into pinned memory run
    at PCIe speed, and the block is reused once the arrays built over it are garbage collected.  At most `max_blocks`
    blocks exist; beyond that `take` returns None and the caller uses pageable memory."""

    def __init__(self, max_blocks=6, granule=1 << 20):
        self.max_blocks, self.granule = max_blocks, granule
        self._free = {}
        self._n = 0
        self._mu = threading.RLock()
        self._returned = collections.deque()  # blocks whose arrays died (filled by _Lease.__del__ without the lock)

    def take(self, nbytes):
        size = max(self.granule, (int(nbytes) + self.granule - 1) // self.granule * self.granule)
        with self._mu:
            self._drain()
            ptrs = self._free.get(size)
            ptr = ptrs.pop() if ptrs else None
            if ptr is None:
                if self._n >= self.max_blocks:
                    victim = next((s for s, p in self._free.items() if p), None)  # a free block of another size makes room
                    if victim is None:
                        return None
                    load().b2s_free_pinned(self._free[victim].pop())
                    self._n -= 1
                ptr = init().b2s_alloc_pinned(size)
                if not ptr:
                    return None
                self._n += 1
        buf = (C.c_char * size).from_address(ptr)
        buf._lease = _Lease(self, ptr, size)
        return buf

    def _drain(self):
        while True:
            try:
                ptr, size = self._returned.popleft()
            except IndexError:
                return
            self._free.setdefault(size, []).append(ptr)

    def _give_back(self, ptr, size):
        self._returned.append((ptr, size))


PINNED = PinnedPool()


# DLPack data type codes of the typestrs a DeviceArray can have (datetime64[ns] goes out as int64)
_DLPACK_CODES = {"f": 2, "i": 0, "u": 1, "b": 6, "M": 0}
_DLTENSOR = b"dltensor"
_pyapi = C.PyDLL(None)  # own function objects: other modules retype the ones ctypes.pythonapi shares
_capsule_new = _pyapi.PyCapsule_New
_capsule_new.restype, _capsule_new.argtypes = C.py_object, [C.c_void_p, C.c_char_p, C.c_void_p]
_capsule_valid = _pyapi.PyCapsule_IsValid
_capsule_valid.restype, _capsule_valid.argtypes = C.c_int, [C.c_void_p, C.c_char_p]
_capsule_pointer = _pyapi.PyCapsule_GetPointer
_capsule_pointer.restype, _capsule_pointer.argtypes = C.c_void_p, [C.c_void_p, C.c_char_p]


@C.CFUNCTYPE(None, C.c_void_p)
def _capsule_destructor(capsule):
    """a capsule that no consumer took still holds its tensor: the library's deleter frees it (a consumer renames the
    capsule and calls the deleter itself)"""
    if _capsule_valid(capsule, _DLTENSOR):
        load().b2s_dlpack_delete(_capsule_pointer(capsule, _DLTENSOR))


class DeviceArray:
    """a C-order array in device memory the library allocated (b2s_darray_t), freed when the last owner lets go: this
    object, a consumer of `__cuda_array_interface__` (which keeps this object alive) or of `__dlpack__` (which holds its
    own reference, dropped by the library's deleter).  Ready when it is handed out."""

    def __init__(self, handle, shape, dtype):
        self._h = handle
        self.shape = tuple(int(d) for d in shape)
        self.dtype = np.dtype(dtype)
        ptr, nbytes = C.c_void_p(), C.c_int64()
        check(load().b2s_darray_info(handle, C.byref(ptr), C.byref(nbytes)))
        self.ptr = ptr.value

    @property
    def nbytes(self):
        return int(np.prod(self.shape)) * self.dtype.itemsize

    @property
    def __cuda_array_interface__(self):
        return {"shape": self.shape, "typestr": self.dtype.str, "data": (self.ptr, False), "version": 3, "strides": None,
                "stream": None}

    def __dlpack_device__(self):
        return (2, _device_ordinal())  # kDLCUDA

    def __dlpack__(self, *, stream=None, max_version=None, dl_device=None, copy=None):
        if copy:
            raise BufferError("a DeviceArray is handed over without a copy")
        if dl_device is not None and tuple(dl_device) != self.__dlpack_device__():
            raise BufferError(f"the array is on {self.__dlpack_device__()}, not {tuple(dl_device)}")
        shape = (C.c_int64 * max(len(self.shape), 1))(*self.shape)
        managed = load().b2s_darray_dlpack(self._h, len(self.shape), shape, _DLPACK_CODES[self.dtype.kind], self.dtype.itemsize * 8)
        if not managed:
            raise NativeError(f"DLPack export failed: {load().b2s_last_error().decode()}")
        return _capsule_new(managed, _DLTENSOR, C.cast(_capsule_destructor, C.c_void_p))

    def numpy(self):
        """a host copy"""
        out = np.empty(self.shape, dtype=self.dtype)
        if out.nbytes:
            check(load().b2s_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes))
        return out

    def release(self):
        if self._h:
            load().b2s_darray_release(self._h)
            self._h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def darray_alloc(nbytes, zero=False):
    """a new library-owned device array of `nbytes` bytes (zeroed on the library stream with zero=True) -> its handle"""
    h = C.c_void_p()
    check(init().b2s_darray_alloc(int(nbytes), int(bool(zero)), C.byref(h)))
    return h.value


def darray_view(base, offset, shape, dtype):
    """DeviceArray over bytes [offset, ...) of the array `base` (a handle), which it keeps alive"""
    h = C.c_void_p()
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    check(load().b2s_darray_view(base, int(offset), nbytes, C.byref(h)))
    return DeviceArray(h.value, shape, dtype)


def library_device():
    """the device ordinal the library runs on: the one b2s_init took, or the one init() would take"""
    return _device_ordinal() if _inited else int(os.environ.get("LOCAL_RANK", "0"))


def _device_ordinal():
    info = DevInfo()
    check(load().b2s_device_info(C.byref(info)))
    return int(info.ordinal)


def darray_live():
    """device arrays the library has handed out and not yet freed"""
    return int(load().b2s_darray_live())
