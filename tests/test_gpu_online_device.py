"""Online feature vectors built from CUDA columns (b2s_table_create_device, b2s_table_stats_device,
b2s_table_label_keys_device, b2s_keys_hash_decimal_device) against the service built from the equal pandas frame: the
same lookups bit for bit, the same `get()` answers, the same refusals, statistics within the documented bound, and
enrichment from CUDA keys equal to enrichment from host keys.  Needs an H100."""

import ctypes as C

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import online as bo  # noqa: E402
from tests import api_b200  # noqa: E402

I64 = np.iinfo(np.int64)
I32 = np.iinfo(np.int32)
DTYPES = [np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.bool_]


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def feature_column(rng, dtype, n):
    """values of one dtype with its edges: NaN, +-inf, -0.0, values float32 rounds, ints beyond 2^24"""
    if dtype in (np.float32, np.float64):
        v = rng.normal(size=n) * 1e3
        v[rng.random(n) < 0.1] = np.nan
        v[rng.random(n) < 0.03] = np.inf
        v[rng.random(n) < 0.03] = -np.inf
        v[rng.random(n) < 0.03] = -0.0
        if dtype == np.float64:
            v[rng.random(n) < 0.05] = 1.0 + 2.0**-30  # rounds under float32
            v[rng.random(n) < 0.02] = 1e39  # overflows to inf
        return v.astype(dtype)
    if dtype == np.bool_:
        return rng.random(n) < 0.5
    info = np.iinfo(dtype)
    v = rng.integers(info.min, info.max, size=n, dtype=dtype, endpoint=True)
    if dtype == np.int64:
        v[: min(n, 3)] = [2**24 + 1, -(2**53) - 3, I64.max][: min(n, 3)]
    return v


def unique_ints(rng, dtype, n):
    info = np.iinfo(dtype)
    span = min(int(info.max) - int(info.min), 2**62)
    return (rng.choice(span, size=n, replace=False) + int(info.min)).astype(dtype) if n < span else None


def make_columns(n, n_feat, seed=0, keys=None, label=None):
    rng = np.random.default_rng(seed)
    cols = {"id": unique_ints(rng, np.int64, n) if keys is None else None}
    if keys is not None:
        cols = dict(keys)
    feats = []
    for j in range(n_feat):
        name = f"f{j}"
        cols[name] = feature_column(rng, DTYPES[j % len(DTYPES)], n)
        feats.append(name)
    if label is not None:
        cols["label"] = label
    return cols, feats


def to_cuda(cols):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in cols.items()}


def pair(cols, feats, index_keys=("id",), label=None, policy=None):
    """(frame service, device service) of the same rows"""
    frame = pd.DataFrame(cols).set_index(list(index_keys))
    feats = feats + (["label"] if label else [])
    hvec = bo.FeatureVector("v", feats, list(index_keys), frame, label_column=label)
    dvec = bo.FeatureVector("v", feats, list(index_keys), to_cuda(cols), label_column=label)
    return hvec.get_online_feature_service(impute_policy=policy), dvec.get_online_feature_service(impute_policy=policy)


def info(table):
    n, f, cap = C.c_int64(), C.c_int32(), C.c_int64()
    nat.check(nat.load().b2s_table_info(table._h, C.byref(n), C.byref(f), C.byref(cap)))
    return n.value, f.value, cap.value


def same_matrix(hs, ds, keys, d_keys):
    X, found = hs.get_matrix(keys)
    Y, dfound = ds.get_matrix(keys)
    np.testing.assert_array_equal(X.view(np.uint32), Y.view(np.uint32))
    np.testing.assert_array_equal(found, dfound)
    rows, f = ds.get_matrix(d_keys)
    assert isinstance(rows, nat.DeviceArray) and rows.shape == X.shape and f.dtype == np.int32
    np.testing.assert_array_equal(rows.numpy().view(np.uint32), X.view(np.uint32))
    np.testing.assert_array_equal(f.numpy().astype(bool), found)


def same_rows(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if w is None or g is None:
            assert g is None and w is None
            continue
        if isinstance(w, dict):
            assert list(g) == list(w)
            g, w = list(g.values()), list(w.values())
        np.testing.assert_array_equal(np.array(g, dtype=np.float64), np.array(w, dtype=np.float64))


def same_stats(hvec_stats, dvec_stats, exact=False):
    for k in ("count", "min", "max"):
        np.testing.assert_array_equal(dvec_stats[k].to_numpy(), hvec_stats[k].to_numpy())
    for k in ("mean", "std"):
        a = hvec_stats[k].to_numpy(dtype=np.float32)
        b = dvec_stats[k].to_numpy(dtype=np.float32)
        if exact:
            np.testing.assert_array_equal(b, a)
        else:
            ulp = np.spacing(np.abs(a)).astype(np.float32)
            ok = (np.isnan(a) & np.isnan(b)) | (np.abs(a.astype(np.float64) - b) <= ulp)
            assert ok.all(), (k, a[~ok], b[~ok])


# ---- sizes, widths and dtypes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,n_feat", [(1, 1), (2, 3), (8, 4), (9, 64), (16, 65), (17, 128), (32, 3), (33, 4), (2**20 + 1, 4)])
def test_device_table_equals_the_frame_table(n, n_feat):
    cols, feats = make_columns(n, n_feat, seed=n + n_feat)
    hs, ds = pair(cols, feats)
    assert info(hs.table) == info(ds.table)  # same keys, features and capacity
    rng = np.random.default_rng(1)
    ask = np.concatenate([cols["id"][rng.permutation(n)][:5000], np.array([I64.max - 7, 12345], dtype=np.int64)])
    same_matrix(hs, ds, ask, torch.from_numpy(ask).cuda())
    same_stats(hs.vector.get_stats_table(), ds.vector.get_stats_table())
    hs.close(), ds.close()


@pytest.mark.parametrize("policy", [None, {"*": "$mean"}, {"*": 0.5, "f1": "$max", "f2": -3}, {"f3": "$min"},
                                    {"*": "$std", "f0": "$count"}])
def test_get_and_impute_policies(policy):
    cols, feats = make_columns(500, 12, seed=3)
    hs, ds = pair(cols, feats, policy=policy)
    assert hs._impute_values == ds._impute_values
    ask = [[int(k)] for k in cols["id"][:40]] + [[123]] + [[int(k)] for k in cols["id"][100:110]]
    for as_list in (False, True):
        same_rows(ds.get(ask, as_list=as_list), hs.get(ask, as_list=as_list))
    hs.vector.with_indexes = ds.vector.with_indexes = True
    same_rows(ds.get([{"id": r[0]} for r in ask[:8]]), hs.get([{"id": r[0]} for r in ask[:8]]))
    hs.close(), ds.close()


# ---- keys ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.int8, np.int16, np.int32, np.int64])
def test_single_int_keys_of_every_width(dtype):
    rng = np.random.default_rng(5)
    n = 200 if dtype == np.int8 else 3000
    lo, hi = np.iinfo(dtype).min, np.iinfo(dtype).max
    rest = unique_ints(rng, dtype, n)
    keys = rng.permutation(np.concatenate([np.array([lo, hi], dtype=dtype), rest[(rest != lo) & (rest != hi)][: n - 2]]))
    cols, feats = make_columns(n, 5, seed=6, keys={"id": keys})
    hs, ds = pair(cols, feats, policy={"*": "$mean"})
    ask = np.concatenate([keys, np.array([np.iinfo(dtype).max], dtype=dtype)])[::-1].copy()
    same_matrix(hs, ds, ask.astype(np.int64), torch.from_numpy(ask).cuda())
    same_rows(ds.get([[int(k)] for k in ask[:50]]), hs.get([[int(k)] for k in ask[:50]]))


def edge_ints():
    vals = {I64.min, I64.max, 0, -1, I32.min, I32.max}
    for k in range(1, 19):
        vals |= {10**k, -(10**k), 10**k - 1}
    return np.array(sorted(vals), dtype=np.int64)


@pytest.mark.parametrize("n_cols", [2, 3])
def test_composite_keys_hash_as_the_frame_path_hashes(n_cols):
    e = edge_ints()
    grid = np.stack(np.meshgrid(*[e] * n_cols, indexing="ij"), -1).reshape(-1, n_cols)
    grid = grid[np.random.default_rng(7).permutation(len(grid))[:20000]]
    widths = [np.int64, np.int32, np.int16][:n_cols]
    keys = {}
    for j, w in enumerate(widths):
        col = grid[:, j]
        if w != np.int64:
            col = np.clip(col, np.iinfo(w).min, np.iinfo(w).max)
        keys[f"k{j}"] = col.astype(w)
    frame_keys = pd.DataFrame(keys).drop_duplicates()
    keys = {k: frame_keys[k].to_numpy() for k in frame_keys}
    cols, feats = make_columns(len(frame_keys), 4, seed=8, keys=keys)
    names = list(keys)
    hs, ds = pair(cols, feats, index_keys=names, policy={"*": 0.25})
    tuples = list(zip(*[keys[k].tolist() for k in names]))
    ask = tuples[::-1] + [tuple([5] * n_cols)]
    d_ask = {k: torch.from_numpy(np.array([t[j] for t in ask], dtype=keys[k].dtype)).cuda() for j, k in enumerate(names)}
    same_matrix(hs, ds, ask, d_ask)
    same_rows(ds.get([list(t) for t in ask[:30]]), hs.get([list(t) for t in ask[:30]]))


@pytest.mark.parametrize("where", ["first", "last", "interior"])
@pytest.mark.parametrize("composite", [False, True])
def test_duplicate_keys_are_refused_with_the_frame_paths_message(where, composite):
    n = 5000
    rng = np.random.default_rng(9)
    ids = unique_ints(rng, np.int64, n)
    at = {"first": (0, 1), "last": (n - 2, n - 1), "interior": (1200, 3100)}[where]
    ids[at[1]] = ids[at[0]]
    ids[4000] = ids[2000]  # a later repeat: the message names the first
    keys = {"id": ids, "k": np.zeros(n, np.int32)} if composite else {"id": ids}
    cols, feats = make_columns(n, 3, seed=10, keys=keys)
    index_keys = list(keys)
    frame = pd.DataFrame(cols).set_index(index_keys)
    errs = []
    for src in (frame, to_cuda(cols)):
        with pytest.raises(Exception) as err:
            bo.FeatureVector("v", feats, index_keys, src).get_online_feature_service()
        errs.append((type(err.value), str(err.value)))
    assert errs[0] == errs[1], errs
    if not composite:  # the first row that repeats a key, and the row it repeats
        first, row = at if at[1] < 4000 else (2000, 4000)
        assert errs[0][1].endswith(f"duplicate entity key {ids[row]} (rows {first} and {row})"), errs[0][1]


# ---- labels -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64, np.int8, np.bool_])
def test_truthy_labels(dtype):
    n = 4000
    cols, feats = make_columns(n, 4, seed=11)
    for f in feats:
        cols[f][:300] = 0  # all-zero rows: the label decides whether get() reports them
    rng = np.random.default_rng(12)
    lab = rng.integers(0, 3, size=n).astype(dtype)
    if dtype in (np.float32, np.float64):
        lab[rng.random(n) < 0.2] = np.nan
        lab[::7] = -0.0
    cols["label"] = lab
    hs, ds = pair(cols, feats, label="label")
    np.testing.assert_array_equal(ds._label_alive, hs._label_alive)
    ask = [[int(k)] for k in cols["id"][:400]]
    same_rows(ds.get(ask), hs.get(ask))
    same_rows(ds.get(ask, as_list=True), hs.get(ask, as_list=True))


# ---- statistics ---------------------------------------------------------------------------------------------------------
def test_stats_bit_equal_on_an_exact_workload_and_within_one_ulp_otherwise():
    rng = np.random.default_rng(13)
    n = 100_000
    k = rng.integers(-(2**14) + 1, 2**14, size=(n - 100) // 2)
    exact = {}
    for j, c in enumerate([0.0, 3.0, -1000.0, 100.25]):
        # c + k / 1024 in float32 exactly; every float64 partial sum is exact, the mean is c, the squares are exact too
        v = np.concatenate([k, -k, np.full(100, np.nan)])[rng.permutation(n)].astype(np.float64) / 1024 + c
        exact[f"e{j}"] = v.astype(np.float32)
    cols = {"id": unique_ints(rng, np.int64, n), **exact}
    hs, ds = pair(cols, list(exact))
    same_stats(hs.vector.get_stats_table(), ds.vector.get_stats_table(), exact=True)
    for seed in range(3):
        cols, feats = make_columns(300_000, 16, seed=20 + seed)
        hs, ds = pair(cols, feats)
        same_stats(hs.vector.get_stats_table(), ds.vector.get_stats_table())


def test_stats_of_columns_without_two_finite_values():
    n = 50
    cols = {"id": np.arange(n, dtype=np.int64), "a": np.full(n, np.nan, np.float32),
            "b": np.where(np.arange(n) == 3, 1.5, np.inf).astype(np.float32)}
    hs, ds = pair(cols, ["a", "b"])
    pd.testing.assert_frame_equal(ds.vector.get_stats_table(), hs.vector.get_stats_table())


# ---- enrichment ---------------------------------------------------------------------------------------------------------
def enriched_server(vec, policy, trees=False):
    from sklearn.ensemble import GradientBoostingRegressor
    from sklearn.linear_model import LinearRegression

    api_b200.register_feature_vector("store://dvec", vec)
    fn = api_b200.new_function("enrich-dev", kind="serving")
    graph = fn.set_topology("router", api_b200.EnrichmentVotingEnsemble(feature_vector_uri="store://dvec", impute_policy=policy,
                                                                        vote_type="regression", executor_type="array"))
    rng = np.random.default_rng(14)
    F = len(vec.features)
    for i in range(2 if trees else 4):
        if trees:
            X = rng.normal(size=(300, F)).astype(np.float32)
            m = GradientBoostingRegressor(n_estimators=6, max_depth=3, random_state=i).fit(X, X[:, 0] + i)
        else:
            m = LinearRegression()
            m.coef_, m.intercept_, m.n_features_in_ = rng.normal(size=F), 0.5 * i, F
        graph.add_route(f"m{i}", class_name="SKLearnModelServer", model=m, model_path="")
    return fn.to_mock_server(namespace={"SKLearnModelServer": api_b200.SKLearnModelServer})


@pytest.mark.parametrize("trees", [False, True])
def test_run_enriched_from_cuda_keys_equals_host_keys(trees):
    n = 20000
    cols, feats = make_columns(n, 8, seed=15)
    policy = {"*": "$mean"}
    frame = pd.DataFrame(cols).set_index(["id"])
    hserver = enriched_server(bo.FeatureVector("v", feats, ["id"], frame), policy, trees)
    dserver = enriched_server(bo.FeatureVector("v", feats, ["id"], to_cuda(cols)), policy, trees)
    ask = cols["id"][np.random.default_rng(16).integers(0, n, size=50000)]
    ask[::11] = 99  # not an entity
    want, want_st = hserver.run_enriched(ask, with_status=True)
    for server in (hserver, dserver):
        before = nat.launch_count()
        out, st = server.run_enriched(torch.from_numpy(ask).cuda(), with_status=True)
        launches = nat.launch_count() - before
        assert launches == (6 if trees else 2)  # the keys, then one fused launch, or the lookup, trees3's three and mark_unknown
        assert isinstance(out, nat.DeviceArray) and isinstance(st, nat.DeviceArray)
        np.testing.assert_array_equal(out.numpy().view(np.uint32), want.view(np.uint32))
        np.testing.assert_array_equal(st.numpy(), want_st)
        assert (st.numpy()[::11] & nat.ROW_UNKNOWN_KEY).all()
    got, got_st = dserver.run_enriched(ask, with_status=True)  # host keys on a device-built table
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(got_st, want_st)


# ---- launches, streams and lifetimes ------------------------------------------------------------------------------------
def test_launch_counts_of_the_build():
    cols, feats = make_columns(1000, 6, seed=17, label=np.ones(1000, np.float32))
    dvec = bo.FeatureVector("v", feats + ["label"], ["id"], to_cuda(cols), label_column="label")
    before = nat.launch_count()
    svc = dvec.get_online_feature_service()
    assert nat.launch_count() - before == 1 + 3 + 1  # keys, pack + insert + check, label keys
    svc.close()
    dvec._stats = None
    before = nat.launch_count()
    svc = dvec.get_online_feature_service(impute_policy={"*": "$mean"})
    assert nat.launch_count() - before == 3 + 1 + 3 + 1  # statistics, keys, build, label keys
    keys = {"a": torch.arange(100, device="cuda"), "b": torch.arange(100, device="cuda", dtype=torch.int32)}
    comp = {**{k: v.cpu().numpy() for k, v in keys.items()}, "x": np.ones(100, np.float32)}
    csvc = bo.FeatureVector("c", ["x"], ["a", "b"], to_cuda(comp)).get_online_feature_service()
    before = nat.launch_count()
    rows, found = csvc.get_matrix(keys)
    assert nat.launch_count() - before == 2 and found.numpy().all()  # the decimal hash, the lookup


def test_a_callers_stream_and_later_writes():
    n = 200_000
    cols, feats = make_columns(n, 4, seed=18)
    frame = pd.DataFrame(cols).set_index(["id"])
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):  # DLPack orders the library behind the stream that is current when a column is taken
        dev = {k: torch.empty(len(v), dtype=torch.from_numpy(v[:1]).dtype, device="cuda") for k, v in cols.items()}
        torch.cuda._sleep(20_000_000)  # the copies below land after a delay on the producer's stream
        for k, v in cols.items():
            dev[k].copy_(torch.from_numpy(v).pin_memory(), non_blocking=True)
        dvec = bo.FeatureVector("v", feats, ["id"], dev)
        ds = dvec.get_online_feature_service(impute_policy={"*": "$max"})
    hs = bo.FeatureVector("v", feats, ["id"], frame).get_online_feature_service(impute_policy={"*": "$max"})
    torch.cuda.synchronize()
    for t in dev.values():
        t.zero_() if t.dtype != torch.bool else t.fill_(False)  # the table holds its own copy
    torch.cuda.synchronize()
    ask = cols["id"][::-3].copy()
    same_matrix(hs, ds, ask, torch.from_numpy(ask).cuda())


def test_device_arrays_are_released():
    cols, feats = make_columns(5000, 8, seed=19)
    live = nat.darray_live()
    hs, ds = pair(cols, feats, policy={"*": "$mean"})
    rows, found = ds.get_matrix(torch.from_numpy(cols["id"]).cuda())
    del rows, found
    hs.close(), ds.close()
    assert nat.darray_live() == live


# ---- the C-ABI ----------------------------------------------------------------------------------------------------------
def test_misaligned_and_host_pointers_are_refused_before_any_launch():
    lib = nat.load()
    n = 64
    keys = nat.DeviceBuffer(8 * n + 16)
    vals = nat.DeviceBuffer(8 * n + 16)
    host = np.zeros(n, np.int64)
    out = C.c_void_p()
    stats = np.empty((5, 1), np.float32)
    col = nat.TableCol(vals.ptr, 4, nat.TCOL_FLOAT)
    bad = [
        lambda: lib.b2s_table_create_device(keys.ptr + 4, n, C.byref(col), 1, None, C.byref(out)),
        lambda: lib.b2s_table_create_device(host.ctypes.data, n, C.byref(col), 1, None, C.byref(out)),
        lambda: lib.b2s_table_create_device(keys.ptr, n, C.byref(nat.TableCol(vals.ptr + 2, 4, nat.TCOL_FLOAT)), 1, None, C.byref(out)),
        lambda: lib.b2s_table_create_device(keys.ptr, n, C.byref(nat.TableCol(vals.ptr, 3, nat.TCOL_INT)), 1, None, C.byref(out)),
        lambda: lib.b2s_table_stats_device(C.byref(nat.TableCol(host.ctypes.data, 8, nat.TCOL_INT)), 1, n, nat._p(stats, C.c_float), None),
        lambda: lib.b2s_table_label_keys_device(keys.ptr + 4, n, C.byref(col), nat._p(host, C.c_int64), C.byref(C.c_int64()), None),
        lambda: lib.b2s_keys_hash_decimal_device((nat.KeyCol * 2)(nat.KeyCol(vals.ptr + 4, 8, 1), nat.KeyCol(vals.ptr, 8, 1)), 2, n,
                                                 keys.ptr, None),
        lambda: lib.b2s_keys_hash_decimal_device((nat.KeyCol * 1)(nat.KeyCol(vals.ptr, 4, 0)), 1, n, keys.ptr, None),
        lambda: lib.b2s_table_mark_unknown_device(keys.ptr + 2, vals.ptr, n, None),
    ]
    for call in bad:
        before = nat.launch_count()
        assert call() == -1, lib.b2s_last_error()
        assert nat.launch_count() == before
