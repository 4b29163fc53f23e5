"""`GraphServer.run_batch` of rows in HBM, and `b2s_run_columns_device` under it, on the H100: `-m gpu`.

- The pack: a transform-only plan's output is the packed row, which must equal numpy's per-column astype(float32) bit for bit
  on every kind and width: NaN payloads of both signs from float64, overflow to +-inf, subnormals, integer extremes, bool.
- Every kernel family of tests/test_gpu_host_batches.py: run_batch of CUDA columns and of a CUDA matrix give the votes, status
  words and served kernel of b2s_run_device over the same rows, and so of the host batch of those rows (which, above 64 KiB,
  is served from device memory too).
- Ranges of 2^20 rows at the edges, with a column that holds the row number, read by a linear model.
- Zero-copy matrices: column slices, offset views and 4-byte row strides are served where they are, without a pack or scratch.
- Chains: get_offline_tensors' matrix, and a DeviceColumnBatch from FeatureSet.ingest, against the host chain's rows.
- Streams, lifetimes and the C-ABI's refusals.
"""

import ctypes as C
import gc
import io
import contextlib

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.plan import DevicePlan, column_ranges  # noqa: E402
from mlrun_b200.serving.compiler import CompiledGraph  # noqa: E402
from mlrun_b200.serving.host import GraphServer  # noqa: E402
from mlrun_b200.sharding import MergeComm  # noqa: E402
from tests.device_check import Rows, names, run_device  # noqa: E402
from tests.test_gpu_host_batches import KINDS, served  # noqa: E402
from tests.test_gpu_host_batches import _SERVED  # noqa: E402
from tests.test_gpu_linear_paths import Flow, scorers  # noqa: E402

M = 1 << 20
ERR_INVALID, ERR_UNSUPPORTED = -1, -6


@pytest.fixture(scope="module", autouse=True)
def device():
    nat.init(0)
    assert nat.device_info()["cc"] == (9, 0)
    yield
    for s in _SERVED.values():
        s.plan.close()
    _SERVED.clear()


def server_of(plan):
    """a GraphServer whose compiled graph is `plan` over f0 .. f{n_in - 1}"""
    srv = GraphServer()
    srv._compiled = CompiledGraph(plan, None, names(plan.n_in), ("", ""))
    return srv


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.view(np.uint32).tobytes() == b.view(np.uint32).tobytes()


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sync():
    torch.cuda.synchronize()
    nat.check(nat.load().b2s_device_sync())


# ---- the pack --------------------------------------------------------------------------------------------------------------
def edge_columns(n):
    rng = np.random.default_rng(5)
    f64 = rng.normal(size=n) * 10.0 ** rng.integers(-45, 45, n)
    nan_bits = np.array([0x7FF8_0000_0000_0001, 0xFFF8_0000_DEAD_BEEF, 0x7FF4_0000_0000_0000, 0xFFF0_0000_0000_0001,
                         0x7FFF_FFFF_FFFF_FFFF, 0x7FF8_1234_5678_9ABC], dtype=np.uint64).view(np.float64)
    edges64 = np.concatenate([nan_bits, [3.5e38, -3.5e38, 3.4028235677973366e38, 3.4028235e38, 1e-45, -1e-46, 7e-46, 1.4e-45,
                                         2.0 ** -149 * 1.5, 2.0 ** -126 * (1 - 2.0 ** -24), -0.0, np.inf, -np.inf,
                                         1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, 16777217.0]])
    f64[:len(edges64)] = edges64
    f32 = rng.normal(size=n).astype(np.float32)
    f32[:6] = np.array([0x7FC0_0001, 0xFFC0_1234, 0x7F80_0001, 0x0000_0001, 0x8000_0000, 0x007F_FFFF], dtype=np.uint32).view(np.float32)
    cols = {"f32": f32, "f64": f64}
    for dt in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64):
        info = np.iinfo(dt)
        a = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        a[:6] = np.array([info.min, info.max, 0, info.max - 1, info.min + 1, {8: 1, 16: 1, 32: 2**24 + 1, 64: 2**53 + 1}[info.bits]],
                         dtype=dt)
        cols[np.dtype(dt).name] = a
    cols["bool"] = rng.random(n) < 0.5
    return cols


KIND_OF = {"f": nat.TCOL_FLOAT, "i": nat.TCOL_INT, "u": nat.TCOL_UINT, "b": nat.TCOL_BOOL}


def table_cols(arrays):
    """(torch CUDA copies, [nat.TableCol]) of host arrays (unsigned and bool ones cross as signed ints of their width)"""
    dev = [cuda(a.view(f"i{a.dtype.itemsize}") if a.dtype.kind in "ub" else a) for a in arrays]
    sync()
    return dev, [nat.TableCol(t.data_ptr(), a.dtype.itemsize, KIND_OF[a.dtype.kind]) for t, a in zip(dev, arrays)]


@pytest.mark.parametrize("n", [1, 33, 100_003])
def test_the_pack_is_numpys_astype_float32(n):
    cols = edge_columns(max(n, 32))
    cols = {k: v[:n] for k, v in cols.items()}
    arrays = list(cols.values())
    plan = Flow(len(arrays)).program().build_plan([])  # transform-only: its output row is the packed row
    assert plan.kernel.startswith("rows_kernel<STORE")
    _dev, tcols = table_cols(arrays)
    out = torch.full((n + 1, len(arrays)), -7.0, device="cuda")
    sync()
    before = nat.launch_count()
    stats = plan.run_columns_device(tcols, n, out.data_ptr())
    sync()
    assert stats["kernels"] == 2 and stats["rows"] == n and nat.launch_count() - before == 2
    got = out.cpu().numpy()
    assert (got[n] == -7.0).all(), "a row past the end was written"
    with np.errstate(over="ignore", invalid="ignore"):
        want = np.stack([a.astype(np.float32) for a in arrays], axis=1)
    for j, name in enumerate(cols):
        assert same_bits(got[:n, j], want[:, j]), (name, np.argwhere(got[:n, j].view(np.uint32) != want[:, j].view(np.uint32))[:5])
    plan.close()


# ---- every kernel family ----------------------------------------------------------------------------------------------------
def mixed_columns(X):
    """X's columns as CUDA columns, every other one widened to float64 (astype(float32) gives the column back)"""
    return {f"f{j}": cuda(X[:, j] if j % 2 == 0 else X[:, j].astype(np.float64)) for j in range(X.shape[1])}


@pytest.mark.parametrize("kind", list(KINDS))
def test_every_kernel_family_serves_device_rows_as_it_serves_the_same_rows_in_hbm(kind):
    s = served(kind)
    srv = server_of(s.plan)
    cols = mixed_columns(s.X)
    sync()
    before = nat.launch_count()
    out, st = srv.run_batch(cols, with_status=True)
    assert isinstance(out, nat.DeviceArray) and isinstance(st, nat.DeviceArray)
    assert nat.launch_count() - before == 1 + s.k
    assert s.plan.last_kernel == s.dev_kernel, (kind, s.plan.last_kernel)
    assert same_bits(out.numpy(), s.dev_out) and (st.numpy() == s.dev_st).all(), kind

    X = cuda(s.X)
    sync()
    before = nat.launch_count()
    out, st = srv.run_batch(X, names=names(s.plan.n_in), with_status=True)
    assert nat.launch_count() - before == s.k
    assert s.plan.last_kernel == s.dev_kernel, (kind, s.plan.last_kernel)
    assert same_bits(out.numpy(), s.dev_out) and (st.numpy() == s.dev_st).all(), kind

    # above 64 KiB the host batch is copied in (or pipelined) first and served from device memory by the same family
    assert s.X.nbytes > 64 << 10
    host, host_st = srv.run_batch(s.X, with_status=True)
    assert same_bits(host, out.numpy()) and (host_st == st.numpy()).all(), kind


# ---- ranges ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, M - 1, M, M + 1, 2 * M + 3])
def test_ranges_place_every_row(n):
    """column 0 holds the row number and the model reads it: a wrong range offset names the row it moved"""
    plan = Flow(2).plan([("linear", dict(W=np.array([[1.0, 0.0]]), b=np.zeros(1), link=nat.LINK_IDENTITY, classes=None))])
    row = torch.arange(n, dtype=torch.int32, device="cuda")
    other = torch.zeros(n, dtype=torch.float64, device="cuda")
    out = torch.full((n + 1, 1), -7.0, device="cuda")
    status = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    sync()
    before = nat.launch_count()
    stats = plan.run_columns_device([nat.TableCol(row.data_ptr(), 4, nat.TCOL_INT), nat.TableCol(other.data_ptr(), 8, nat.TCOL_FLOAT)],
                                    n, out.data_ptr(), status.data_ptr())
    sync()
    ranges = column_ranges(n, 4)
    assert len(ranges) == (n + M - 1) // M
    assert stats["kernels"] == 2 * len(ranges) and nat.launch_count() - before == stats["kernels"]
    got, st = out.cpu().numpy(), status.cpu().numpy()
    bad = np.flatnonzero(got[:n, 0] != np.arange(n, dtype=np.float32))
    assert not len(bad), (bad[:5], got[bad[:5], 0])
    assert got[n, 0] == -7.0 and st[n] == -1 and (st[:n] == 0).all()
    plan.close()


# ---- zero-copy matrices ------------------------------------------------------------------------------------------------------
ZC_N = 70_001  # rows of 32 float32 values: 8.5 MiB


@pytest.fixture(scope="module")
def zc_plan():
    plan = Flow(32).plan(scorers(32, 2, seed=40))
    X = np.random.default_rng(40).normal(size=(ZC_N, 32)).astype(np.float32)
    X[::101, 7] = np.nan
    yield plan, X
    plan.close()


@pytest.mark.parametrize("how", ["contiguous", "column-slice", "offset-view", "stride-4-bytes"])
def test_cuda_matrices_are_scored_in_place(zc_plan, how):
    plan, X = zc_plan
    if how == "contiguous":
        t, stride, offset = cuda(X), 128, 0
    elif how == "column-slice":  # X[:, :32] of a 40-column matrix: 160-byte rows
        wide = np.zeros((ZC_N, 40), np.float32)
        wide[:, :32] = X
        t, stride, offset = cuda(wide)[:, :32], 160, 0
    elif how == "offset-view":  # rows start 4 bytes past a 16-byte boundary
        flat = torch.zeros(ZC_N * 32 + 1, device="cuda")
        flat[1:] = cuda(X).reshape(-1)
        t, stride, offset = flat[1:].view(ZC_N, 32), 128, 4
    else:  # 33-float rows: 132 bytes, a multiple of 4 and not of 16
        wide = np.zeros((ZC_N, 33), np.float32)
        wide[:, :32] = X
        t, stride, offset = cuda(wide)[:, :32], 132, 0
    want, want_st = run_device(plan, Rows(X, stride=stride, offset=offset))
    want_kernel = plan.last_kernel
    srv = server_of(plan)
    sync()
    live, before = nat.darray_live(), nat.launch_count()
    out, st = srv.run_batch(t, names=names(32), with_status=True)
    assert nat.darray_live() - live == 2, "only the outputs and status words were allocated"
    assert nat.launch_count() - before == 1, "one scoring launch and no pack"
    assert plan.last_kernel == want_kernel, (how, plan.last_kernel, want_kernel)
    assert want_kernel == ("rowthread/ldgsts" if how in ("offset-view", "stride-4-bytes") else "rowthread/tma")
    assert same_bits(out.numpy(), want) and (st.numpy() == want_st).all()
    host = srv.run_batch(X)
    assert same_bits(host, out.numpy())
    del out, st
    gc.collect()
    assert nat.darray_live() == live


def test_a_matrix_from_a_library_array_and_an_empty_matrix(zc_plan):
    plan, X = zc_plan
    srv = server_of(plan)
    arr = nat.DeviceArray(nat.darray_alloc(X.nbytes), X.shape, np.float32)
    nat.check(nat.load().b2s_memcpy_h2d(arr.ptr, X.ctypes.data, X.nbytes))
    assert same_bits(srv.run_batch(arr).numpy(), srv.run_batch(X))
    out, st = srv.run_batch(cuda(X[:0]), with_status=True)
    assert out.shape == (0, plan.out_cols) and st.shape == (0,)
    out, st = srv.run_batch({f"f{j}": cuda(X[:0, j]) for j in range(32)}, with_status=True)
    assert out.shape == (0, plan.out_cols) and st.shape == (0,)


# ---- chains ------------------------------------------------------------------------------------------------------------------
def linear_server(n_feat, impute=None, n_models=4, seed=0):
    from sklearn.linear_model import LinearRegression

    from mlrun_b200 import api

    rng = np.random.default_rng(seed)
    fn = api.new_function("scoring", kind="serving")
    step = fn.set_topology("flow", engine="sync")
    if impute is not None:
        step = step.to(api.Imputer(mapping=impute), name="imputer")
    step = step.to("*FeatureRowVotingEnsemble", name="ensemble", vote_type="regression", executor_type="array")
    for i in range(n_models):
        m = LinearRegression()
        m.coef_, m.intercept_, m.n_features_in_ = rng.normal(size=n_feat), float(rng.normal()), n_feat
        step.add_route(f"m{i + 1}", class_name="FeatureRowModelServer", model=m, model_path="")
    return fn.to_mock_server(namespace={"FeatureRowVotingEnsemble": api.FeatureRowVotingEnsemble,
                                        "FeatureRowModelServer": api.FeatureRowModelServer})


def chain_frames(n, keys, seed):
    rng = np.random.default_rng(seed)
    base = 1_600_000_000 * 10**9
    tx = {"card": rng.integers(0, keys, size=n).astype(np.int64),
          "when": (np.arange(n, dtype=np.int64) * 10**8 + base).view("datetime64[ns]")}
    for j in range(4):
        tx[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    tx["t1"][::17] = np.nan
    pick = np.sort(rng.choice(n, size=n // 4, replace=False))
    labels = {"card": tx["card"][pick], "when": tx["when"][pick], "label": rng.standard_normal(n // 4)}
    return tx, labels


def test_offline_tensors_are_scored_where_they_are():
    from mlrun_b200.feature_store import ingest as bi
    from mlrun_b200.feature_store import offline as boff

    tx, labels = chain_frames(20_000, 700, seed=8)
    results = []
    for device in (False, True):
        txn = bi.FeatureSet("transactions", entities=["card"], timestamp_key="when")
        txn.add_aggregation("t0", ["sum", "max", "avg"], ["1h"], "10m")
        lbs = bi.FeatureSet("labels", entities=["card"], timestamp_key="when")
        conv = (lambda d: {k: cuda(v.view(np.int64) if v.dtype.kind == "M" else v) for k, v in d.items()}) if device \
            else (lambda d: pd.DataFrame(d))
        with contextlib.redirect_stdout(io.StringIO()):
            batch = txn.ingest(conv(tx))
            sync()
            boff.register_offline_frame(txn, batch)
            boff.register_offline_frame(lbs, conv(labels))
            t = boff.get_offline_tensors(boff.FeatureVector("v", ["transactions.*"], label_feature="labels.label"),
                                         dtype="float32")
        results.append(t)
    th, td = results
    assert th.columns == td.columns
    srv = linear_server(len(td.columns), seed=3)
    host_out, host_st = srv.run_batch(th.features.numpy(), names=th.columns, with_status=True)
    out, st = srv.run_batch(td.features, names=td.columns, with_status=True)
    assert same_bits(out.numpy(), host_out) and (st.numpy() == host_st).all()
    assert host_st.any() and not host_st.all(), "some rows carry a NaN feature"
    for name in list(boff._OFFLINE):
        boff._OFFLINE.pop(name).close()


def test_an_ingested_device_batch_is_scored_with_its_index_columns():
    from mlrun_b200.feature_store import ingest as bi
    from mlrun_b200.feature_store import steps as bs

    rng = np.random.default_rng(9)
    n = 50_000
    cols = {"id": rng.integers(0, 300, n).astype(np.int64),
            "ts": np.sort(rng.integers(0, 3 * 24 * 3600 * 10**9, n)).astype(np.int64),
            "x": rng.normal(size=n).astype(np.float32), "c": rng.integers(0, 4, n).astype(np.int32),
            "y": rng.integers(-9, 9, n).astype(np.int32)}
    cols["x"][::13] = np.nan

    def feature_set():
        fs = bi.FeatureSet("tx", entities=["id"], timestamp_key="ts")
        fs.graph.to(bs.Imputer(mapping={"x": 0.25}), name="imputer").to(bs.OneHotEncoder(mapping={"c": [0, 1, 2]}), name="onehot")
        fs.add_aggregation("y", ["sum", "max"], ["1h"], "10m")
        return fs

    host_cols = {k: (v.view("datetime64[ns]") if k == "ts" else v) for k, v in cols.items()}
    with contextlib.redirect_stdout(io.StringIO()):
        host = feature_set().ingest(host_cols)
        dev = feature_set().ingest({k: cuda(v) for k, v in cols.items()})
    sync()
    picked = ["id"] + [k for k in host.columns if host.columns[k].dtype.kind != "M"]
    srv = linear_server(len(picked), impute={"x": 0.5}, seed=4)
    with np.errstate(over="ignore", invalid="ignore"):
        rows = np.stack([np.asarray(host.index["id"] if k == "id" else host.columns[k]).astype(np.float32) for k in picked], axis=1)
    host_out, host_st = srv.run_batch(rows, names=picked, with_status=True)
    before = nat.launch_count()
    out, st = srv.run_batch(dev, names=picked, with_status=True)
    assert nat.launch_count() - before == 2
    assert same_bits(out.numpy(), host_out) and (st.numpy() == host_st).all()


# ---- streams, lifetimes, refusals -------------------------------------------------------------------------------------------
def test_a_producers_side_stream_writes_are_awaited(zc_plan):
    plan, X = zc_plan
    srv = server_of(plan)
    want = srv.run_batch(X)
    src = {f"f{j}": cuda(X[:, j]) for j in range(32)}
    src_matrix = cuda(X)
    sync()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        cols = {k: torch.full((ZC_N,), -1.0, device="cuda") for k in src}
        torch.cuda._sleep(100_000_000)  # the copies below land well after the call was made
        for k, v in src.items():
            cols[k].copy_(v)
        got = srv.run_batch(cols)
    assert same_bits(got.numpy(), want)
    with torch.cuda.stream(side):
        t = torch.full((ZC_N, 32), -1.0, device="cuda")
        torch.cuda._sleep(100_000_000)
        t.copy_(src_matrix)
        got = srv.run_batch(t, names=names(32))
    assert same_bits(got.numpy(), want)


def test_outputs_go_through_dlpack_and_cai_and_are_freed(zc_plan):
    plan, X = zc_plan
    srv = server_of(plan)
    want = srv.run_batch(X)
    cols = {f"f{j}": cuda(X[:, j]) for j in range(32)}
    sync()
    gc.collect()
    live = nat.darray_live()
    out, st = srv.run_batch(cols, with_status=True)
    a = torch.from_dlpack(out)
    b = torch.as_tensor(st, device="cuda")
    assert same_bits(a.cpu().numpy(), want) and (b.cpu().numpy() == 0).sum() > 0
    del out, st
    gc.collect()
    assert nat.darray_live() == live + 2, "the consumers hold the arrays"
    del a, b
    gc.collect()
    assert nat.darray_live() == live

    target = nat.DeviceBuffer(4 * (ZC_N + 1) * plan.out_cols)
    plan.set_merge_targets([target.ptr], 0)
    try:
        with pytest.raises(nat.NativeError, match="error -6"):  # a refused call frees the outputs it had made
            srv.run_batch(cols, with_status=True)
    finally:
        plan.set_merge_targets([], 0)
    with pytest.raises(ValueError, match="same length"):
        srv.run_batch({**cols, "f1": cuda(X[:-1, 1])})
    gc.collect()
    assert nat.darray_live() == live


def test_c_abi_refusals_launch_nothing():
    plan = Flow(2).plan(scorers(2, 1, seed=2))
    lib = nat.load()
    a = torch.zeros(64, dtype=torch.float64, device="cuda")
    host = np.zeros(64, dtype=np.float64)
    out = torch.zeros(64, device="cuda")
    status = torch.zeros(64, dtype=torch.int32, device="cuda")
    sync()
    good = nat.TableCol(a.data_ptr(), 8, nat.TCOL_FLOAT)

    def call(p, cols, n=64, d_out=None, d_status=None):
        arr = (nat.TableCol * len(cols))(*cols)
        stats = nat.Stats()
        before = nat.launch_count()
        rc = lib.b2s_run_columns_device(p._h, arr, len(cols), n, out.data_ptr() if d_out is None else d_out,
                                        status.data_ptr() if d_status is None else d_status, C.byref(stats), None)
        sync()
        if rc:
            assert nat.launch_count() == before and stats.kernels == 0, "a refused call launched"
        else:
            assert nat.launch_count() - before == stats.kernels == (2 if n else 0)
        return rc

    assert call(plan, [good, good]) == 0
    assert call(plan, [good]) == ERR_INVALID                                                  # n_cols != n_in
    assert call(plan, [good, good, good]) == ERR_INVALID
    assert call(plan, [good, nat.TableCol(a.data_ptr(), 2, nat.TCOL_FLOAT)]) == ERR_INVALID   # width
    assert call(plan, [good, nat.TableCol(a.data_ptr(), 8, 7)]) == ERR_INVALID                # kind
    assert call(plan, [good, nat.TableCol(a.data_ptr(), 2, nat.TCOL_BOOL)]) == ERR_INVALID
    assert call(plan, [good, nat.TableCol(None, 8, nat.TCOL_FLOAT)]) == ERR_INVALID           # null
    assert call(plan, [good, nat.TableCol(a.data_ptr() + 4, 8, nat.TCOL_FLOAT)]) == ERR_INVALID  # misaligned
    assert call(plan, [good, nat.TableCol(host.ctypes.data, 8, nat.TCOL_FLOAT)]) == ERR_INVALID  # host memory
    assert call(plan, [good, good], d_out=out.data_ptr() + 2) == ERR_INVALID
    assert call(plan, [good, good], d_status=status.data_ptr() + 2) == ERR_INVALID
    assert call(plan, [good, good], n=-1) == ERR_INVALID
    unfinished = DevicePlan(2)
    assert call(unfinished, [good, good]) == ERR_INVALID
    unfinished.close()
    target = nat.DeviceBuffer(4 * 65)
    plan.set_merge_targets([target.ptr], 0)
    assert call(plan, [good, good]) == ERR_UNSUPPORTED
    assert call(plan, [good, good], n=0) == ERR_UNSUPPORTED
    plan.set_merge_targets([], 0)
    comm = MergeComm(0, 1, 64, plan.out_cols, exchange=None)
    comm.attach(plan)
    assert call(plan, [good, good]) == ERR_UNSUPPORTED
    assert call(plan, [good, good], n=0) == ERR_UNSUPPORTED
    comm.detach(plan)
    comm.close()
    assert call(plan, [good, good], n=0) == 0
    plan.close()
