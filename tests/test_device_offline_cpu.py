"""Feature sets registered from CUDA columns and CUDA entity rows, without a GPU: every refusal of the device registration and
of CUDA entity rows is raised before the library is loaded (its entry points are replaced by ones that fail the test), with
the type and message the host path raises for the equal pandas frame.  CUDA columns are stood in for by objects that
expose a CUDA array interface or a DLPack device over an address nothing reads."""

import types

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import columnar
from mlrun_b200.feature_store import ingest as bi
from mlrun_b200.feature_store import offline as boff
from mlrun_b200.lowering import LoweringError
from mlrun_b200.serving.resolve import MLRunInvalidArgumentError


class CudaCol:
    """a column that states a CUDA array interface (v3) over an address nothing reads"""

    def __init__(self, a, strides=None, typestr=None):
        a = np.asarray(a)
        self.__cuda_array_interface__ = {"shape": a.shape, "typestr": typestr or a.dtype.str, "data": (0x7F00_0000_0000, False),
                                         "version": 3, "strides": strides, "stream": None}


class OtherDevice:
    """DLPack on CUDA device 1"""

    def __dlpack_device__(self):
        return (2, 1)

    def __dlpack__(self, stream=None):
        raise AssertionError("the column must be refused before it is taken")


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("the library was called")

    monkeypatch.setattr(nat, "load", fail)
    monkeypatch.setattr(nat, "init", fail)
    monkeypatch.setattr(nat, "_inited", False)
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    monkeypatch.setattr(boff, "_OFFLINE", {})


def cuda(a, **k):
    return CudaCol(a, **k)


def columns(n=8, ids=None, ts=True, **extra):
    cols = {"id": cuda(np.zeros(n, np.int64) if ids is None else ids)}
    if ts:
        cols["ts"] = cuda(np.zeros(n, np.int64))
    cols["x"] = cuda(np.zeros(n, np.float32))
    cols.update(extra)
    return cols


def fset(entities=("id",), ts="ts"):
    return bi.FeatureSet("s", entities=list(entities), timestamp_key=ts)


def host_error(fs, frame):
    """what registering the equal pandas frame raises, with the library stubbed out: (type, message)"""
    with pytest.raises(Exception) as err:
        boff.register_offline_frame(fs, frame)
    return type(err.value), str(err.value)


def device_error(fs, source):
    with pytest.raises(Exception) as err:
        boff.register_offline_frame(fs, source)
    assert not isinstance(err.value, AssertionError), err.value
    return type(err.value), str(err.value)


# ---- registration --------------------------------------------------------------------------------------------------------
def test_a_mixed_source_is_refused():
    with pytest.raises(ValueError, match="CUDA columns and .* host columns"):
        boff.register_offline_frame(fset(), {"id": cuda(np.zeros(8, np.int64)), "x": np.zeros(8, np.float32)})


def test_a_column_on_another_device_is_refused():
    with pytest.raises(ValueError, match="CUDA device 1; the library runs on device 0"):
        boff.register_offline_frame(fset(), {**columns(), "y": OtherDevice()})


@pytest.mark.parametrize("shape,strides,match", [((8,), (8,), "not C-contiguous"), ((2, 4), None, "1-D")])
def test_non_contiguous_and_2d_columns_are_refused(shape, strides, match):
    with pytest.raises(ValueError, match=match):
        boff.register_offline_frame(fset(), {**columns(), "y": cuda(np.zeros(shape, np.float32), strides=strides)})


def test_columns_of_different_lengths_are_refused_as_pandas_refuses_them():
    with pytest.raises(ValueError) as host:
        pd.DataFrame({"id": np.zeros(8, np.int64), "x": np.zeros(7, np.float32)})
    assert device_error(fset(ts=None), {"id": cuda(np.zeros(8, np.int64)), "x": cuda(np.zeros(7, np.float32))}) == \
        (ValueError, str(host.value))


@pytest.mark.parametrize("drop", ["id", "ts"])
def test_a_missing_entity_or_timestamp_column_is_refused_alike(drop):
    cols = columns()
    del cols[drop]
    frame = pd.DataFrame({k: np.zeros(8, np.int64 if k != "x" else np.float32) for k in cols})
    got = device_error(fset(), cols)
    assert got == host_error(fset(), frame) and got[0] is MLRunInvalidArgumentError


def test_a_set_without_entities_is_refused_alike():
    frame = pd.DataFrame({"ts": np.zeros(8, "datetime64[ns]"), "x": np.zeros(8, np.float32)})
    got = device_error(fset(entities=()), columns(ts=True))
    assert got == host_error(fset(entities=()), frame) and got[0] is LoweringError


@pytest.mark.parametrize("dtype", [np.bool_, np.float32, np.float64, np.uint64])
def test_keys_the_device_cannot_encode_are_refused_alike(dtype):
    ids = np.zeros(8, dtype)
    frame = pd.DataFrame({"id": ids, "ts": np.zeros(8, "datetime64[ns]"), "x": np.zeros(8, np.float32)})
    got = device_error(fset(), columns(ids=ids))
    assert got == host_error(fset(), frame) and got[0] is LoweringError and "are not lowered" in got[1]


@pytest.mark.parametrize("typestr", ["|S8", "|O"])
def test_string_keys_are_refused(typestr):
    with pytest.raises(LoweringError, match="is a string key: there are no string columns on the device"):
        boff.register_offline_frame(fset(), columns(ids=np.zeros(8, np.int64)) | {"id": cuda(np.zeros(8, np.int64), typestr=typestr)})


@pytest.mark.parametrize("dtype", [np.int32, np.float64, np.uint64, "datetime64[ms]"])
def test_a_timestamp_that_is_not_int64_nanoseconds_is_refused_alike(dtype):
    ts = np.zeros(8, dtype)
    frame = pd.DataFrame({"id": np.zeros(8, np.int64), "ts": ts, "x": np.zeros(8, np.float32)})
    got = device_error(fset(), {**columns(ts=False), "ts": cuda(ts)})
    want = host_error(fset(), frame)
    if str(np.dtype(dtype)) == "datetime64[ms]":  # a ms frame is registered on the host; the device takes ns alone
        assert got[0] is LoweringError and "has dtype datetime64[ms]" in got[1]
    else:
        assert got == want and got[0] is LoweringError


# ---- CUDA entity rows ----------------------------------------------------------------------------------------------------
def registered(name="s", entities=("id",), ts="ts", key_kind="int", longest_run=1):
    """a registered set as the planner reads it (its index is never called before these refusals)"""
    src = boff.OfflineSource.__new__(boff.OfflineSource)
    src.name, src.entities, src.timestamp_key, src.key_kind = name, list(entities), ts, key_kind
    src.features = {"f": (0, "float32", boff._NAN32)}
    src.has_nat, src.ts_factor = False, 1
    src.index = types.SimpleNamespace(longest_run=longest_run)
    boff._OFFLINE[name] = src
    return src


VEC = boff.FeatureVector("v", ["s.f"])


def test_cuda_entity_rows_are_refused_by_get_offline_features():
    registered()
    with pytest.raises(LoweringError, match="get_offline_tensors"):
        boff.get_offline_features(VEC, columns(), "ts")
    with pytest.raises(LoweringError, match="get_offline_tensors"):
        boff.get_offline_features(VEC, columnar.DeviceColumnBatch({"ts": cuda(np.zeros(8, np.int64))}, 8,
                                                                  index={"id": cuda(np.zeros(8, np.int64))}), "ts")


def test_mixed_and_misshapen_entity_rows_are_refused():
    registered()
    with pytest.raises(ValueError, match="CUDA columns and .* host columns"):
        boff.get_offline_tensors(VEC, {**columns(), "y": np.zeros(8)}, "ts")
    with pytest.raises(ValueError, match="CUDA device 1"):
        boff.get_offline_tensors(VEC, {**columns(), "y": OtherDevice()}, "ts")
    with pytest.raises(ValueError, match="1-D"):
        boff.get_offline_tensors(VEC, {**columns(), "y": cuda(np.zeros((2, 4)))}, "ts")
    with pytest.raises(ValueError, match="not C-contiguous"):
        boff.get_offline_tensors(VEC, {**columns(), "y": cuda(np.zeros(8), strides=(16,))}, "ts")
    with pytest.raises(ValueError, match="All arrays must be of the same length"):
        boff.get_offline_tensors(VEC, {**columns(), "y": cuda(np.zeros(7))}, "ts")


def planner_error(rows, ts="ts"):
    with pytest.raises(Exception) as err:
        boff.get_offline_tensors(VEC, rows, ts)
    assert not isinstance(err.value, AssertionError), err.value
    return type(err.value), str(err.value)


def frame_of(cols):
    return pd.DataFrame({k: np.zeros(8, np.dtype(c.__cuda_array_interface__["typestr"])) for k, c in cols.items()})


@pytest.mark.parametrize("case", ["no key column", "no timestamp column", "float keys", "bool keys", "uint64 keys",
                                  "int32 timestamps", "float timestamps"])
def test_entity_row_refusals_equal_the_pandas_frames(case):
    registered()
    cols = columns()
    if case == "no key column":
        del cols["id"]
    elif case == "no timestamp column":
        del cols["ts"]
    elif case.endswith("keys"):
        cols["id"] = cuda(np.zeros(8, {"float": np.float32, "bool": np.bool_, "uint64": np.uint64}[case.split()[0]]))
    else:
        cols["ts"] = cuda(np.zeros(8, {"int32": np.int32, "float": np.float64}[case.split()[0]]))
    host = frame_of(cols)
    if "ts" in host and host["ts"].dtype == np.int64:
        host["ts"] = host["ts"].astype("datetime64[ns]")
    assert planner_error(cols) == planner_error(host)


def test_string_entity_keys_are_refused():
    registered()
    with pytest.raises(LoweringError, match="is a string key"):
        boff.get_offline_tensors(VEC, {**columns(), "id": cuda(np.zeros(8, np.int64), typestr="|S8")}, "ts")


def test_a_key_kind_mismatch_and_several_rows_per_key_are_refused_alike():
    registered(key_kind="pair")
    cols = columns()
    assert planner_error(cols) == planner_error(frame_of(cols).assign(ts=np.zeros(8, "datetime64[ns]")))
    boff._OFFLINE.clear()
    registered(ts=None, longest_run=3)
    got = planner_error(cols, None)
    assert got == planner_error(frame_of(cols), None) and "several rows per key" in got[1]


def spine(device):
    """a registered set whose rows are a pandas frame or CUDA columns, as the entity-less planner reads them"""
    src = registered()
    src.features = {"f": (0, "float32", boff._NAN32), "g": (1, "float32", boff._NAN32)}
    if device:
        src.rows = boff._Columns.of_device({"id": cuda(np.zeros(8, np.int64)), "ts": cuda(np.zeros(8, np.int64)),
                                            "f": cuda(np.zeros(8, np.float32)), "g": cuda(np.zeros(8, np.float32))}, {"ts"})
    else:
        src.rows = boff._Columns.of_frame(pd.DataFrame({"id": np.zeros(8, np.int64), "ts": np.zeros(8, "datetime64[ns]"),
                                                        "f": np.zeros(8, np.float32), "g": np.zeros(8, np.float32)}))
    return src


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("vector", [boff.FeatureVector("v", ["s.f", "s.g"], label_feature="s.g"),
                                    boff.FeatureVector("v", ["s.f", "s.f as y"])])
def test_a_spine_column_selected_twice_is_refused_alike(device, vector):
    spine(device)
    for fn in (boff.get_offline_features, boff.get_offline_tensors):
        with pytest.raises(LoweringError, match="duplicate column names in the entity frame"):
            fn(vector)


def test_two_defects_are_refused_in_the_host_order():
    """a missing timestamp column comes before float keys, as on the host"""
    registered()
    cols = columns(ids=np.zeros(8, np.float32), ts=False)
    assert planner_error(cols) == planner_error(frame_of(cols)) and planner_error(cols)[0] is KeyError
    boff._OFFLINE["s"].has_nat = True  # the set's NaT comes before the keys
    cols = columns(ids=np.zeros(8, np.float32))
    host = frame_of(cols).assign(ts=np.zeros(8, "datetime64[ns]"))
    assert planner_error(cols) == planner_error(host) and "right side" in planner_error(cols)[1]
