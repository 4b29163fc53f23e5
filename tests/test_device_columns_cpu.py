"""Feature-set ingest of CUDA columns, without a GPU: which sources take the device path, and every refusal of that path,
each raised before the library is loaded or the device brought up (the library entry points are replaced by ones that fail
the test).  CUDA columns are stood in for by objects that expose a CUDA array interface or a DLPack device."""

import numpy as np
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import columnar
from mlrun_b200.feature_store import ingest as bi
from mlrun_b200.feature_store import steps as bs
from mlrun_b200.lowering import LoweringError


class CudaCol:
    """a column that states a CUDA array interface (v3) over an address nothing reads"""

    def __init__(self, a, strides=None):
        a = np.asarray(a)
        self.__cuda_array_interface__ = {"shape": a.shape, "typestr": a.dtype.str, "data": (0x7F00_0000_0000, False),
                                         "version": 3, "strides": strides, "stream": None}


class OtherDevice:
    """DLPack on CUDA device 1"""

    def __dlpack_device__(self):
        return (2, 1)

    def __dlpack__(self, stream=None):
        raise AssertionError("the column must be refused before it is taken")


class DLPackOnly:
    """DLPack on CUDA device 0 and no CUDA array interface (a JAX-like producer); the capsule describes a host array, which
    is all a description reads.  Records the stream each capsule was asked for."""

    def __init__(self, a):
        self.a, self.streams = np.asarray(a), []

    def __dlpack_device__(self):
        return (2, 0)

    def __dlpack__(self, stream=None):
        self.streams.append(stream)
        return self.a.__dlpack__()


class HostDLPack:
    def __dlpack_device__(self):
        return (1, 0)


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("the library was called")

    monkeypatch.setattr(nat, "load", fail)
    monkeypatch.setattr(nat, "init", fail)
    monkeypatch.setattr(nat, "_inited", False)
    monkeypatch.delenv("LOCAL_RANK", raising=False)


def f32(n=8):
    return CudaCol(np.zeros(n, np.float32))


def agg_set():
    fs = bi.FeatureSet("tx", entities=["id"], timestamp_key="ts")
    fs.add_aggregation("x", ["sum"], ["1h"], "10m")
    return fs


def test_sources_are_classified_by_where_their_columns_live():
    assert columnar.is_device_source({"x": f32(), "ts": CudaCol(np.zeros(8, np.int64))})
    assert not columnar.is_device_source({"x": np.zeros(8, np.float32)})
    assert not columnar.is_device_source({"x": HostDLPack()})
    assert columnar.is_device_source(columnar.DeviceColumnBatch({}, 0))
    assert not columnar.is_device_source(columnar.ColumnBatch({}, 0))
    assert not columnar.is_device_source({})


def test_a_mixed_source_is_refused():
    fs = bi.FeatureSet("s", timestamp_key="ts")
    with pytest.raises(ValueError, match="CUDA columns and .* host columns"):
        fs.ingest({"x": f32(), "y": np.zeros(8, np.float32)})


def test_a_column_on_another_device_is_refused():
    fs = bi.FeatureSet("s")
    with pytest.raises(ValueError, match="CUDA device 1; the library runs on device 0"):
        fs.ingest({"x": f32(), "y": OtherDevice()})


@pytest.mark.parametrize("shape,strides,match", [((8,), (8,), "not C-contiguous"), ((2, 4), None, "1-D")])
def test_non_contiguous_and_2d_columns_are_refused(shape, strides, match):
    col = CudaCol(np.zeros(shape, np.float32), strides=strides)
    with pytest.raises(ValueError, match=match):
        bi.FeatureSet("s").ingest({"x": col})


def test_int64_is_a_timestamp_only_where_the_set_names_one():
    fs = bi.FeatureSet("s", timestamp_key="ts")
    with pytest.raises(LoweringError, match="column 'n' is int64: only timestamps"):
        fs.ingest({"ts": CudaCol(np.zeros(8, np.int64)), "n": CudaCol(np.zeros(8, np.int64))})
    cols = {"ts": columnar.DeviceColumn(CudaCol(np.zeros(8, np.int64)), "ts"),
            "when": columnar.DeviceColumn(CudaCol(np.zeros(8, np.int64)), "when"),
            "x": columnar.DeviceColumn(f32(), "x"),
            "dt": columnar.DeviceColumn(CudaCol(np.zeros(8, "datetime64[ns]")), "dt")}
    schema, dtypes = columnar.device_schema(cols, {"ts", "when"})
    assert schema == [("ts", bi.I64), ("when", bi.I64), ("x", bi.F32), ("dt", bi.I64)]
    assert str(dtypes["ts"]) == "datetime64[ns]" and str(dtypes["x"]) == "float32"
    with pytest.raises(LoweringError, match="has dtype float64"):
        columnar.device_schema({"y": columnar.DeviceColumn(CudaCol(np.zeros(8)), "y")}, set())


def test_date_extractor_timestamp_column_is_a_timestamp():
    """the lowering that follows the schema check needs the library: reaching it is the proof the int64 was taken"""
    fs = bi.FeatureSet("s")
    fs.graph.to(bs.DateExtractor(parts=["hour"], timestamp_col="when"))
    with pytest.raises(AssertionError, match="the library was called"):
        fs.ingest({"when": CudaCol(np.zeros(8, np.int64)), "x": f32()})


@pytest.mark.parametrize("keys,match", [
    ({"id": CudaCol(np.zeros(8, "S8"))}, "string key"),
    ({"id": CudaCol(np.zeros(8, np.float32))}, "are not lowered"),
    ({"id": CudaCol(np.zeros(8, np.uint64))}, "are not lowered"),
])
def test_keys_the_device_cannot_encode_are_refused(keys, match):
    with pytest.raises(LoweringError, match=match):
        agg_set().ingest({**keys, "ts": CudaCol(np.zeros(8, np.int64)), "x": f32()})


def test_missing_entity_columns_are_refused_with_the_host_message():
    with pytest.raises(LoweringError, match=r"entity columns \['id'\] must all be in the ingested data"):
        agg_set().ingest({"ts": CudaCol(np.zeros(8, np.int64)), "x": f32()})


def test_reference_dtypes_is_refused():
    with pytest.raises(LoweringError, match="reference_dtypes=True"):
        bi.FeatureSet("s").ingest({"x": f32()}, reference_dtypes=True)


def test_device_column_batch_mirrors_column_batch():
    b = columnar.DeviceColumnBatch({"a": 1, "b": 2}, 5, index={"id": 3})
    assert b.names == ["a", "b"] and len(b) == 5 and b["b"] == 2 and b.index == {"id": 3}
    assert columnar.is_columnar(b)


def test_dlpack_only_columns_are_described_without_the_library():
    """shape, strides and dtype come from a capsule taken with stream=-1 (no synchronisation) and dropped at once"""
    col = DLPackOnly(np.zeros(8, np.float32))
    d = columnar.DeviceColumn(col, "x")
    assert str(d.dtype) == "float32" and d.n == 8 and d.ptr is None and col.streams == [-1]
    ts, n64 = DLPackOnly(np.zeros(8, np.int64)), DLPackOnly(np.zeros(8, np.int64))
    with pytest.raises(LoweringError, match="column 'n' is int64: only timestamps"):
        bi.FeatureSet("s", timestamp_key="ts").ingest({"ts": ts, "n": n64})
    assert ts.streams == n64.streams == [-1]
    with pytest.raises(LoweringError, match="has dtype float64"):
        bi.FeatureSet("s").ingest({"y": DLPackOnly(np.zeros(8))})
    with pytest.raises(ValueError, match="1-D"):
        bi.FeatureSet("s").ingest({"y": DLPackOnly(np.zeros((2, 4), np.float32))})
    with pytest.raises(ValueError, match="not C-contiguous"):
        bi.FeatureSet("s").ingest({"y": DLPackOnly(np.zeros(16, np.float32)[::2])})


def test_dlpack_only_float_keys_are_refused_before_the_library():
    with pytest.raises(LoweringError, match="are not lowered"):
        agg_set().ingest({"id": DLPackOnly(np.zeros(8, np.float32)), "ts": DLPackOnly(np.zeros(8, np.int64)),
                          "x": DLPackOnly(np.zeros(8, np.float32))})
