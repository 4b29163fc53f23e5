"""`GraphServer.run_batch` of rows in HBM, without a GPU: every refusal of a CUDA matrix and of CUDA columns is raised before
the library is touched (its entry points are replaced by ones that fail the test), with the stated type and message; host
arrays keep the host path; CUDA matrices, mappings of CUDA columns and `DeviceColumnBatch`es (index columns included) are
told apart; and the row ranges of `b2s_run_columns_device` start, end and place their outputs where the header says."""

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200 import plan as bplan
from mlrun_b200.feature_store import columnar
from mlrun_b200.lowering import LoweringError
from mlrun_b200.serving.host import GraphServer


class CudaArray:
    """an array that states a CUDA array interface (v3) over an address nothing reads"""

    def __init__(self, shape, dtype=np.float32, strides=None, typestr=None, data=0x7F00_0000_0000):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr or np.dtype(dtype).str, "data": (data, False),
                                         "version": 3, "strides": strides, "stream": None}


class OtherDevice:
    """DLPack on CUDA device 1"""

    def __dlpack_device__(self):
        return (2, 1)

    def __dlpack__(self, stream=None):
        raise AssertionError("the column must be refused before it is taken")


@pytest.fixture
def no_library(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("the library was called")

    monkeypatch.setattr(nat, "load", fail)
    monkeypatch.setattr(nat, "init", fail)
    monkeypatch.setattr(nat, "_inited", False)
    monkeypatch.delenv("LOCAL_RANK", raising=False)


@pytest.fixture
def server(no_library, monkeypatch):
    srv = GraphServer()

    def compile(*a, **k):
        raise AssertionError("compile() loads the library")

    monkeypatch.setattr(srv, "compile", compile)
    return srv


def col(n=8, dtype=np.float32, **k):
    return CudaArray((n,), dtype, **k)


def source(n=8, **extra):
    cols = {"a": col(n), "b": col(n, np.float64), "c": col(n, np.int64)}
    cols.update(extra)
    return cols


def error_of(fn):
    with pytest.raises(Exception) as err:
        fn()
    assert not isinstance(err.value, AssertionError), err.value
    return type(err.value), str(err.value)


# ---- CUDA columns ---------------------------------------------------------------------------------------------------------
def test_a_mixed_mapping_is_refused(server):
    with pytest.raises(ValueError, match=r"columns \['a'\] are CUDA columns and \['b'\] are host columns"):
        server.run_batch({"a": col(), "b": np.zeros(8, np.float32)}, names=["a", "b"])


def test_a_column_on_another_device_is_refused(server):
    with pytest.raises(ValueError, match="column 'z' is on CUDA device 1; the library runs on device 0"):
        server.run_batch(source(z=OtherDevice()), names=["a"])


@pytest.mark.parametrize("shape,strides,match", [((8,), (8,), "not C-contiguous"), ((2, 4), None, "expected a 1-D column")])
def test_non_contiguous_and_2d_columns_are_refused(server, shape, strides, match):
    with pytest.raises(ValueError, match=match):
        server.run_batch(source(z=CudaArray(shape, strides=strides)), names=["a"])


def test_columns_of_different_lengths_are_refused_as_pandas_refuses_them(server):
    with pytest.raises(ValueError) as host:
        pd.DataFrame({"a": np.zeros(8, np.float32), "b": np.zeros(7, np.float32)})
    assert error_of(lambda: server.run_batch({"a": col(8), "b": col(7)}, names=["a"])) == (ValueError, str(host.value))
    batch = columnar.DeviceColumnBatch({"a": col(8)}, 8, index={"id": col(7, np.int64)})
    assert error_of(lambda: server.run_batch(batch, names=["a"])) == (ValueError, str(host.value))


@pytest.mark.parametrize("names", [["a", "nope"], ["nope", "nada"]])
def test_a_missing_name_is_pandas_key_error(server, names):
    cols = source()
    host = error_of(lambda: pd.DataFrame({k: np.zeros(8) for k in cols})[names])
    assert error_of(lambda: server.run_batch(cols, names=names)) == host
    batch = columnar.DeviceColumnBatch({"a": col(), "b": col()}, 8, index={"c": col(8, np.int64)})
    assert error_of(lambda: server.run_batch(batch, names=names))[0] is KeyError


def test_a_selected_datetime_column_is_refused_by_name(server):
    cols = source(ts=col(typestr="<M8[ns]"))
    with pytest.raises(LoweringError, match="feature 'ts' is a datetime64\\[ns\\] column"):
        server.run_batch(cols, names=["a", "ts"])
    batch = columnar.DeviceColumnBatch({"a": col()}, 8, index={"ts": col(typestr="<M8[ns]")})
    with pytest.raises(LoweringError, match="feature 'ts' is a datetime64\\[ns\\] column"):
        server.run_batch(batch, names=["ts", "a"])
    # an unselected datetime column is no obstacle: the refusal that follows is the missing library, not the column
    with pytest.raises(AssertionError, match="compile"):
        server.run_batch(cols, names=["a", "b"])


@pytest.mark.parametrize("typestr", ["<f2", "<c8"])
def test_kinds_the_online_table_does_not_take_are_refused(server, typestr):
    with pytest.raises(LoweringError, match="feature 'z' has dtype"):
        server.run_batch(source(z=col(typestr=typestr)), names=["a", "z"])


# ---- CUDA matrices -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float16, np.int32])
def test_a_matrix_that_is_not_float32_is_refused_by_dtype(server, dtype):
    with pytest.raises(LoweringError, match=f"dtype {np.dtype(dtype)}.*dtype=\"float32\""):
        server.run_batch(CudaArray((8, 4), dtype), names=list("abcd"))


@pytest.mark.parametrize("shape,strides", [((8,), None), ((2, 4, 4), None), ((8, 4), (32, 8)), ((8, 5), None), ((8, 3), None)])
def test_a_matrix_of_the_wrong_shape_is_refused_as_check_rows_refuses_it(server, shape, strides):
    with pytest.raises(ValueError, match=r"rows must be a float32 \(B, 4\) array with unit inner stride"):
        server.run_batch(CudaArray(shape, strides=strides), names=list("abcd"))


def test_matrix_description_follows_the_producer():
    m = columnar.DeviceColumn(CudaArray((8, 40), strides=(256, 4)), "X", matrix=True)
    assert (m.shape, m.strides, m.ndim, m.dtype) == ((8, 40), (256, 4), 2, np.float32)
    m = columnar.DeviceColumn(CudaArray((8, 40)), "X", matrix=True)
    assert m.strides == (160, 4)
    bplan.check_rows(m, 40)


# ---- which path serves ---------------------------------------------------------------------------------------------------
class _Plan:
    n_in = 2

    def run(self, X, with_status=False):
        self.got = X
        return "host"


class _Compiled:
    def __init__(self):
        self.plan = _Plan()
        self.in_names = ["a", "b"]


def test_sources_take_their_own_paths(no_library, monkeypatch):
    srv = GraphServer()
    compiled = _Compiled()
    monkeypatch.setattr(srv, "compile", lambda names=None: compiled)
    monkeypatch.setattr(srv, "_run_device_matrix", lambda X, names, ws: "matrix")
    monkeypatch.setattr(srv, "_run_device_columns", lambda X, names, ws: "columns")
    host = np.arange(6, dtype=np.float64).reshape(3, 2)
    assert srv.run_batch(host, names=["a", "b"]) == "host"
    assert compiled.plan.got.dtype == np.float32 and compiled.plan.got.flags.c_contiguous
    assert srv.run_batch(CudaArray((3, 2))) == "matrix"
    assert srv.run_batch({"a": col(3), "b": col(3)}) == "columns"
    assert srv.run_batch(columnar.DeviceColumnBatch({"a": col(3)}, 3, index={"b": col(3, np.int64)})) == "columns"


def test_index_columns_of_a_batch_are_addressable(no_library):
    batch = columnar.DeviceColumnBatch({"a": col(), "b": col(8, np.uint8)}, 8, index={"id": col(8, np.int64)})
    cols = columnar.device_columns(batch)
    from mlrun_b200.feature_store.online import table_cols

    picked = table_cols(cols, ["id", "b"], "feature")
    assert [(c.name, dt, kind) for c, dt, kind in picked] == [("id", np.int64, nat.TCOL_INT), ("b", np.uint8, nat.TCOL_UINT)]


# ---- row ranges ------------------------------------------------------------------------------------------------------------
M = 1 << 20


@pytest.mark.parametrize("n,want", [
    (0, []),
    (1, [(0, 1)]),
    (M - 1, [(0, M - 1)]),
    (M, [(0, M)]),
    (M + 1, [(0, M), (M, 1)]),
    (2 * M + 3, [(0, M), (M, M), (2 * M, 3)]),
])
def test_row_ranges(n, want):
    out_row_bytes = 12
    ranges = bplan.column_ranges(n, out_row_bytes)
    assert [(r0, rows) for r0, rows, _off in ranges] == want
    assert [off for _r0, _rows, off in ranges] == [k * M * out_row_bytes for k in range(len(want))]
    assert sum(rows for _r0, rows, _off in ranges) == n
    assert all(rows <= bplan.RANGE_ROWS for _r0, rows, _off in ranges)
