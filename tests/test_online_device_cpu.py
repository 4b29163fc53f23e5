"""Online feature vectors of CUDA columns, without a GPU: every refusal of the device build and of CUDA query keys is raised
before the library is touched (its entry points are replaced by ones that fail the test), with the frame path's type and
message where it has one; and the decimal-text FNV-1a rule of composite keys, restated in numpy, equals `_hash_strings` on
the edge values of every signed int width."""

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import columnar
from mlrun_b200.feature_store import online as bo
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


@pytest.fixture
def no_library(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("the library was called")

    monkeypatch.setattr(nat, "load", fail)
    monkeypatch.setattr(nat, "init", fail)
    monkeypatch.setattr(nat, "_inited", False)
    monkeypatch.delenv("LOCAL_RANK", raising=False)


def cuda(a, **k):
    return CudaCol(a, **k)


def source(n=8, **extra):
    cols = {"id": cuda(np.zeros(n, np.int64)), "x": cuda(np.zeros(n, np.float32)), "y": cuda(np.zeros(n, np.float64))}
    cols.update(extra)
    return cols


def frame_of(cols):
    """the equal frame: the same names and dtypes (values do not matter to these refusals)"""
    return pd.DataFrame({k: np.zeros(c.__cuda_array_interface__["shape"][0], np.dtype(c.__cuda_array_interface__["typestr"]))
                         for k, c in cols.items()}).set_index("id")


def error_of(fn):
    with pytest.raises(Exception) as err:
        fn()
    assert not isinstance(err.value, AssertionError), err.value
    return type(err.value), str(err.value)


# ---- the vector's source ------------------------------------------------------------------------------------------------
def test_a_mixed_source_is_refused(no_library):
    with pytest.raises(ValueError, match="CUDA columns and .* host columns"):
        bo.FeatureVector("v", ["x"], ["id"], {"id": cuda(np.zeros(8, np.int64)), "x": np.zeros(8, np.float32)})


def test_a_column_on_another_device_is_refused(no_library):
    with pytest.raises(ValueError, match="CUDA device 1; the library runs on device 0"):
        bo.FeatureVector("v", ["x"], ["id"], source(z=OtherDevice()))


@pytest.mark.parametrize("shape,strides,match", [((8,), (8,), "not C-contiguous"), ((2, 4), None, "1-D")])
def test_non_contiguous_and_2d_columns_are_refused(no_library, shape, strides, match):
    with pytest.raises(ValueError, match=match):
        bo.FeatureVector("v", ["x"], ["id"], source(z=cuda(np.zeros(shape, np.float32), strides=strides)))


def test_columns_of_different_lengths_are_refused_as_pandas_refuses_them(no_library):
    with pytest.raises(ValueError) as host:
        pd.DataFrame({"id": np.zeros(8, np.int64), "x": np.zeros(7, np.float32)})
    assert error_of(lambda: bo.FeatureVector("v", ["x"], ["id"], {"id": cuda(np.zeros(8, np.int64)), "x": cuda(np.zeros(7, np.float32))})) \
        == (ValueError, str(host.value))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32, np.uint64, np.bool_, np.float32, np.float64])
def test_entity_keys_that_are_not_signed_ints_are_refused(no_library, dtype):
    with pytest.raises(LoweringError, match="signed int"):
        bo.FeatureVector("v", ["x"], ["id"], source(id=cuda(np.zeros(8, dtype))))
    with pytest.raises(LoweringError, match="signed int"):
        bo.FeatureVector("v", ["x"], ["id", "k"], source(k=cuda(np.zeros(8, dtype))))


def test_a_mapping_without_its_entity_columns_is_refused(no_library):
    with pytest.raises(LoweringError, match="no entity column 'k'"):
        bo.FeatureVector("v", ["x"], ["id", "k"], source())


def test_a_batch_without_entity_columns_is_refused(no_library):
    batch = columnar.DeviceColumnBatch({"x": cuda(np.zeros(8, np.float32))}, 8)
    with pytest.raises(LoweringError, match="no entity columns"):
        bo.FeatureVector("v", ["x"], ["id"], batch)


@pytest.mark.parametrize("typestr", ["<f2", "<c8", "<M8[ns]"])
def test_non_numeric_features_and_labels_are_refused_before_the_library(no_library, typestr):
    vec = bo.FeatureVector("v", ["x", "z"], ["id"], source(z=cuda(np.zeros(8, np.float32), typestr=typestr)))
    for policy in (None, {"*": 0.5}, {"*": "$mean"}):
        with pytest.raises(LoweringError, match="feature 'z' has dtype"):
            vec.get_online_feature_service(impute_policy=policy)
    with pytest.raises(LoweringError, match="feature 'z' has dtype"):
        vec.get_stats_table()
    vec = bo.FeatureVector("v", ["x", "z"], ["id"], source(z=cuda(np.zeros(8, np.float32), typestr=typestr)), label_column="z")
    with pytest.raises(LoweringError, match="label 'z' has dtype"):
        vec.get_online_feature_service()


@pytest.mark.parametrize("features", [["x", "nope"], ["nope", "nada"]])
@pytest.mark.parametrize("policy", [None, {"*": "$mean"}, {"x": 1.0}])
def test_a_missing_feature_is_the_frame_paths_key_error(no_library, features, policy):
    cols = source()
    host = error_of(lambda: bo.FeatureVector("v", features, ["id"], frame_of(cols)).get_online_feature_service(impute_policy=policy))
    got = error_of(lambda: bo.FeatureVector("v", features, ["id"], cols).get_online_feature_service(impute_policy=policy))
    assert got == host and got[0] is KeyError


def test_an_impute_policy_of_an_unknown_feature_is_the_frame_paths_error(no_library):
    cols = source()
    policy = {"*": "$mean", "nope": 1}
    host = error_of(lambda: bo.FeatureVector("v", ["x", "y"], ["id"], frame_of(cols)).get_online_feature_service(impute_policy=policy))
    got = error_of(lambda: bo.FeatureVector("v", ["x", "y"], ["id"], cols).get_online_feature_service(impute_policy=policy))
    assert got == host and got[0] is MLRunInvalidArgumentError


# ---- CUDA query keys ----------------------------------------------------------------------------------------------------
def service(index_keys=("id",), string_keys=False):
    """a service whose table is never reached: the refusals come first"""
    svc = bo.OnlineVectorService(bo.FeatureVector("v", ["x"], list(index_keys), source(k=cuda(np.zeros(8, np.int32)))))
    svc._string_keys = string_keys
    svc.table = None
    return svc


@pytest.mark.parametrize("dtype", [np.uint16, np.uint64, np.bool_, np.float64])
def test_cuda_query_keys_that_are_not_signed_ints_are_refused(no_library, dtype):
    with pytest.raises(LoweringError, match="signed int"):
        service().get_matrix(cuda(np.zeros(4, dtype)))
    with pytest.raises(LoweringError, match="signed int"):
        service(("id", "k"), True).get_matrix({"id": cuda(np.zeros(4, np.int64)), "k": cuda(np.zeros(4, dtype))})


def test_cuda_query_key_mappings_are_checked_before_the_library(no_library):
    with pytest.raises(LoweringError, match="no entity column 'k'"):
        service(("id", "k"), True).get_matrix({"id": cuda(np.zeros(4, np.int64))})
    with pytest.raises(ValueError, match="CUDA columns and .* host columns"):
        service(("id", "k"), True).get_matrix({"id": cuda(np.zeros(4, np.int64)), "k": np.zeros(4, np.int64)})
    with pytest.raises(ValueError, match="same length"):
        service(("id", "k"), True).get_matrix({"id": cuda(np.zeros(4, np.int64)), "k": cuda(np.zeros(5, np.int64))})
    with pytest.raises(ValueError, match="CUDA device 1"):
        service().get_matrix(OtherDevice())
    with pytest.raises(ValueError, match="1-D"):
        service().get_matrix(cuda(np.zeros((2, 2), np.int64)))


def test_composite_cuda_keys_for_an_integer_table_are_the_frame_paths_error(no_library):
    svc = service(("id", "k"), False)
    host = error_of(lambda: svc._encode_keys([(1, 2)]))
    got = error_of(lambda: svc.get_matrix({"id": cuda(np.zeros(4, np.int64)), "k": cuda(np.zeros(4, np.int64))}))
    assert got == host and got[0] is MLRunInvalidArgumentError


# ---- the decimal-text FNV-1a rule ---------------------------------------------------------------------------------------
_FNV_OFFSET, _FNV_PRIME = np.uint64(1469598103934665603), np.uint64(1099511628211)


def fnv_decimal_rows(cols):
    """keys_decimal_kernel in numpy: FNV-1a over "-" and the digits of each value's magnitude (taken in uint64, so
    INT64_MIN has one), most significant first, the columns joined by "." -- no string is made"""
    n = len(cols[0])
    h = np.full(n, _FNV_OFFSET, dtype=np.uint64)

    def fold(h, byte, where):
        return np.where(where, (h ^ np.uint64(byte)) * _FNV_PRIME, h)

    with np.errstate(over="ignore"):
        for j, col in enumerate(cols):
            v = np.asarray(col).astype(np.int64)
            if j:
                h = fold(h, ord("."), np.ones(n, bool))
            neg = v < 0
            u = v.view(np.uint64)
            u = np.where(neg, np.uint64(0) - u, u)
            h = fold(h, ord("-"), neg)
            p = np.ones(n, dtype=np.uint64)
            while True:
                more = u // p >= 10
                if not more.any():
                    break
                p = np.where(more, p * np.uint64(10), p)
            live = np.ones(n, bool)
            while live.any():
                d = u // p
                h = fold(h, ord("0") + d, live)
                u = np.where(live, u - d * p, u)
                live = live & (p != 1)
                p = np.where(p > 1, p // np.uint64(10), p)
    return h.view(np.int64)


def edge_values(dtype):
    info = np.iinfo(dtype)
    vals = {info.min, info.max, info.min + 1, info.max - 1, 0, -1, 1, 9, 10, -9, -10}
    for k in range(1, 19):
        for v in (10**k, 10**k - 1, -(10**k), -(10**k) + 1, 10**k + 1):
            if info.min <= v <= info.max:
                vals.add(v)
    return np.array(sorted(vals), dtype=dtype)


@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64])
def test_the_decimal_fnv_rule_equals_hash_strings_on_the_edge_values(dtype):
    a = edge_values(dtype)
    b = a[::-1].copy()
    c = np.roll(edge_values(np.int64), 3)[: len(a)] if len(edge_values(np.int64)) >= len(a) else np.resize(edge_values(np.int64), len(a))
    for cols in ([a], [a, b], [a, b, c]):
        text = [".".join(str(v) for v in row) for row in zip(*[x.tolist() for x in cols])]
        np.testing.assert_array_equal(fnv_decimal_rows(cols), bo._hash_strings(text))


def test_the_decimal_fnv_rule_is_what_the_frame_path_hashes_for_a_multiindex():
    a, b = edge_values(np.int64), edge_values(np.int32)
    b = np.resize(b, len(a))
    frame = pd.DataFrame({"x": np.zeros(len(a), np.float32)}, index=pd.MultiIndex.from_arrays([a, b], names=["u", "v"]))
    svc = bo.OnlineVectorService(bo.FeatureVector("v", ["x"], ["u", "v"], frame))
    np.testing.assert_array_equal(svc._encode_keys(frame.index, build=True), fnv_decimal_rows([a, b]))
