"""Real-time feature enrichment on the device (b2s_table_* + the Enrichment routers) vs the oracle.  Needs an H100."""

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store import online as bo  # noqa: E402
from oracle import enrichment as oe  # noqa: E402
from tests import api_b200, api_oracle  # noqa: E402

RTOL, ATOL = 1e-5, 1e-5


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def _vectors(n_keys=500, n_feat=12, seed=1, key_kind="str", label=None):
    """the same online rows as a product FeatureVector (frame) and an oracle FeatureVector (dict table)"""
    rng = np.random.default_rng(seed)
    feat = [f"f{i}" for i in range(n_feat)]
    vals = rng.normal(size=(n_keys, n_feat)).astype(np.float32)
    vals[rng.random(vals.shape) < 0.08] = np.nan
    vals[rng.random(vals.shape) < 0.02] = np.inf
    vals[rng.random(vals.shape) < 0.01] = -np.inf
    vals[5] = 0.0
    vals[6] = np.nan
    if key_kind == "str":
        keys = [f"ent-{i * 7919 % 100003}" for i in range(n_keys)]
    elif key_kind == "int":
        keys = [int(k) for k in rng.choice(10**12, size=n_keys, replace=False) - 5 * 10**11]
    else:
        keys = [(f"u{i % 37}", i) for i in range(n_keys)]
    index_keys = ["ticker"] if key_kind != "tuple" else ["user", "seq"]
    if key_kind == "tuple":
        frame = pd.DataFrame(vals, columns=feat, index=pd.MultiIndex.from_tuples(keys, names=index_keys))
    else:
        frame = pd.DataFrame(vals, columns=feat, index=pd.Index(keys, name="ticker"))
    bvec = bo.FeatureVector("vec", feat, index_keys, frame, label_column=label)
    stats = bvec.get_stats_table()
    table = {(k if isinstance(k, tuple) else (k,)): {feat[j]: float(vals[i, j]) for j in range(n_feat)} for i, k in enumerate(keys)}
    ovec = oe.FeatureVector("vec", feat, index_keys, table, stats, label_column=label)
    return bvec, ovec, keys, vals, feat


def _same_rows(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if w is None or g is None:
            assert g is None and w is None
            continue
        if isinstance(w, dict):
            assert list(g) == list(w)
            g, w = list(g.values()), list(w.values())
        np.testing.assert_array_equal(np.array(g, dtype=np.float64), np.array(w, dtype=np.float64))


@pytest.mark.parametrize("key_kind", ["str", "int", "tuple"])
@pytest.mark.parametrize("policy", [None, {"*": "$mean"}, {"*": 0.5, "f1": "$max", "f2": -3}, {"f3": "$min"}])
def test_online_service_get_matches_the_reference_semantics(key_kind, policy):
    bvec, ovec, keys, vals, feat = _vectors(key_kind=key_kind)
    bsvc = bvec.get_online_feature_service(impute_policy=policy)
    osvc = ovec.get_online_feature_service(impute_policy=policy)
    unknown = "nope" if key_kind == "str" else (123 if key_kind == "int" else ("zz", 1))
    ask = keys[:40] + [unknown] + keys[100:110]
    rows = [list(k) if isinstance(k, tuple) else [k] for k in ask]
    _same_rows(bsvc.get(rows, as_list=True), osvc.get(rows, as_list=True))
    dict_rows = [dict(zip(bvec.index_keys, r)) for r in rows[:8]]
    _same_rows(bsvc.get(dict_rows), osvc.get(dict_rows))
    with pytest.raises(ValueError, match="must be a list of lists or list of dicts"):
        bsvc.get("GOOG")
    with pytest.raises(ValueError, match="same size of the index_keys"):
        bsvc.get([[1, 2, 3]])
    bsvc.close()


def test_impute_policy_errors_and_matrix_lookup():
    bvec, ovec, keys, vals, feat = _vectors(n_keys=2000, n_feat=16, seed=3)
    with pytest.raises(ValueError, match="in impute_policy but not in feature vector"):
        bvec.get_online_feature_service(impute_policy={"nope": 1})
    svc = bvec.get_online_feature_service(impute_policy={"*": "$mean"})
    X, found = svc.get_matrix(keys[::-1] + ["ghost"])
    assert found[:-1].all() and not found[-1]
    stats = bvec.get_stats_table()
    want = vals[::-1].copy()
    mean = stats["mean"].to_numpy(dtype=np.float32)
    bad = ~np.isfinite(want)
    want[bad] = np.broadcast_to(mean, want.shape)[bad]
    np.testing.assert_array_equal(X[:-1], want)
    np.testing.assert_array_equal(X[-1], mean)  # unknown key: all-NaN row, imputed
    with pytest.raises(ValueError, match="share a 64-bit hash|duplicated"):
        dup = pd.DataFrame(vals[:2], columns=feat, index=pd.Index(["a", "a"], name="ticker"))
        bo.FeatureVector("d", feat, ["ticker"], dup).get_online_feature_service()


def _enriched_server(api, vec, policy, n_models, coefs):
    from sklearn.linear_model import LinearRegression

    api.register_feature_vector("store://vec", vec)
    fn = api.new_function("enrich", kind="serving")
    graph = fn.set_topology("router", api.EnrichmentVotingEnsemble(feature_vector_uri="store://vec", impute_policy=policy,
                                                                    vote_type="regression", executor_type="array"))
    for i in range(n_models):
        m = LinearRegression()
        m.coef_, m.intercept_, m.n_features_in_ = np.asarray(coefs[i], dtype=np.float64), 0.25 * i, len(coefs[i])
        graph.add_route(f"m{i}", class_name="SKLearnModelServer", model=m, model_path="")
    return fn.to_mock_server(namespace={"SKLearnModelServer": api.SKLearnModelServer})


def test_enrichment_router_per_event_and_fused_batch():
    bvec, ovec, keys, vals, feat = _vectors(n_keys=3000, n_feat=16, seed=4)
    coefs = np.random.default_rng(5).normal(size=(4, 16))
    policy = {"*": "$mean"}
    bserver = _enriched_server(api_b200, bvec, policy, 4, coefs)
    oserver = _enriched_server(api_oracle, ovec, policy, 4, coefs)
    ask = [[k] for k in keys[10:42] if k not in (keys[5],)]
    got = bserver.test("/v2/models/infer", body={"inputs": ask})
    want = oserver.test("/v2/models/infer", body={"inputs": ask})
    np.testing.assert_allclose(got["outputs"], want["outputs"], rtol=RTOL, atol=ATOL)
    assert got["model_name"] == want["model_name"]
    # batched engine path: keys -> gather kernel -> fused scoring plan, nothing returns to the host in between
    out, status = bserver.run_enriched(keys + ["ghost"], with_status=True)
    ref = oserver.test("/v2/models/infer", body={"inputs": [[k] for k in keys if k != keys[5]]})["outputs"]
    mask = np.array([k != keys[5] for k in keys])
    np.testing.assert_allclose(out[:-1, 0][mask], ref, rtol=RTOL, atol=ATOL)
    assert (status[:-1] == 0).all() and status[-1] == 4


def test_enrich_host_equals_lookup_then_plan_for_pinned_and_pageable_keys():
    """b2s_table_enrich_host (one call: keys -> gather -> plan -> votes + status) against the two-call form
    (b2s_table_lookup_host, then b2s_run_host on the rows it returned); staging grows across calls; unknown keys without an
    impute value reach the models as NaN, so they carry both status bits"""
    bvec, _ovec, keys, vals, feat = _vectors(n_keys=5000, n_feat=16, seed=9, key_kind="int")
    coefs = np.random.default_rng(10).normal(size=(4, 16))
    for policy in ({"*": "$mean"}, None):
        server = _enriched_server(api_b200, bvec, policy, 4, coefs)
        plan = server.compile().plan
        table = server.graph._object._feature_service.table
        rng = np.random.default_rng(11)
        for n in (1, 33, 4096, 70001, 5):
            ask = np.asarray(keys, dtype=np.int64)[rng.integers(0, len(keys), size=n)]
            ask[::13] = 7  # not an entity
            rows, found = table.lookup(ask)
            want, want_st = plan.run(rows, with_status=True)
            for pinned in (False, True):
                k = ask
                if pinned:
                    k = nat.pinned_empty((n,), np.int64)
                    k[:] = ask
                got, st, stats = table.enrich(plan, k, with_stats=True)
                np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
                np.testing.assert_array_equal(st, want_st | np.where(found, 0, nat.ROW_UNKNOWN_KEY))
                assert stats["rows"] == n and stats["nonfinite_rows"] == int((want_st & 1).sum())
                assert stats["kernels"] == 1  # the scoring kernel gathered its own rows (b2s_table_enrich_device)
            assert (st[::13] & nat.ROW_UNKNOWN_KEY).all() and not (st[1::13] & nat.ROW_UNKNOWN_KEY).any()
            if policy is None:
                assert (st[::13] & nat.ROW_NONFINITE_INPUT).all()
    with pytest.raises(nat.NativeError):
        other = _enriched_server(api_b200, _vectors(n_keys=50, n_feat=12, seed=3, key_kind="int")[0], None, 1, coefs[:1, :12])
        table.enrich(other.compile().plan, np.array([1], dtype=np.int64))


def test_enrich_device_one_launch_and_the_fallback_of_tree_plans():
    """b2s_table_enrich_device on device-resident keys: one launch, same bits as gather-then-score; a tree ensemble is
    not covered by the gather loader (B2S_ERR_UNSUPPORTED -> enrich_host gathers first: the lookup, the three trees3
    launches and mark_unknown, five launches in the stats and in the library's count)"""
    from sklearn.ensemble import GradientBoostingRegressor

    bvec, _ovec, keys, vals, feat = _vectors(n_keys=4000, n_feat=16, seed=12, key_kind="int")
    coefs = np.random.default_rng(13).normal(size=(4, 16))
    server = _enriched_server(api_b200, bvec, {"*": "$mean", "f3": 1.5}, 4, coefs)
    plan = server.compile().plan
    table = server.graph._object._feature_service.table
    n = 10000
    ask = np.asarray(keys, dtype=np.int64)[np.random.default_rng(14).integers(0, len(keys), size=n)]
    ask[::17] = -3
    rows, found = table.lookup(ask)
    want, want_st = plan.run(rows, with_status=True)
    d_keys, d_out, d_st = nat.DeviceBuffer(n * 8), nat.DeviceBuffer(n * plan.out_cols * 4), nat.DeviceBuffer(n * 4)
    nat.check(nat.load().b2s_memcpy_h2d(d_keys.ptr, ask.ctypes.data, n * 8))
    before = nat.launch_count()
    assert table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr) is True
    assert nat.launch_count() - before == 1
    nat.load().b2s_device_sync()
    got, st = np.empty_like(want), np.empty(n, dtype=np.int32)
    nat.check(nat.load().b2s_memcpy_d2h(got.ctypes.data, d_out.ptr, got.nbytes))
    nat.check(nat.load().b2s_memcpy_d2h(st.ctypes.data, d_st.ptr, st.nbytes))
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(st, want_st | np.where(found, 0, nat.ROW_UNKNOWN_KEY))

    # a tree ensemble behind the same router: not fusable, same results through the fallback (lookup, the three trees3
    # launches, mark_unknown)
    api_b200.register_feature_vector("store://vec", bvec)
    fn = api_b200.new_function("enrich-trees", kind="serving")
    graph = fn.set_topology("router", api_b200.EnrichmentVotingEnsemble(feature_vector_uri="store://vec", impute_policy={"*": 0.0},
                                                                        vote_type="regression", executor_type="array"))
    rng = np.random.default_rng(15)
    Xf = rng.normal(size=(400, 16)).astype(np.float32)
    for i in range(2):
        m = GradientBoostingRegressor(n_estimators=8, max_depth=3, random_state=i).fit(Xf, Xf[:, i] * 2 + Xf[:, 5])
        graph.add_route(f"t{i}", class_name="SKLearnModelServer", model=m, model_path="")
    tserver = fn.to_mock_server(namespace={"SKLearnModelServer": api_b200.SKLearnModelServer})
    tplan = tserver.compile().plan
    assert tplan.kernel.startswith("t3_prep_kernel + trees3_kernel<"), tplan.kernel
    ttable = tserver.graph._object._feature_service.table
    assert ttable.enrich_device(tplan, d_keys.ptr, n, d_out.ptr, d_st.ptr) is False
    rows, found = ttable.lookup(ask)
    want, want_st = tplan.run(rows, with_status=True)
    before = nat.launch_count()
    got, st, stats = ttable.enrich(tplan, ask, with_stats=True)
    assert stats["kernels"] == 5 and nat.launch_count() - before == 5
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(st, want_st | np.where(found, 0, nat.ROW_UNKNOWN_KEY))
