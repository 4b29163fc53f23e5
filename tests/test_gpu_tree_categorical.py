"""xgboost and LightGBM models with categorical splits on every kernel that serves them.  Needs an H100: `-m gpu`.

Plans with a categorical node run on trees3 (`trees3_kernel<D,MISS,U,CAT=true>`, depth <= 8) or on `rows_kernel<TREES>`,
like numeric ones.  Each case checks the output against the float64 walk of the packed model (tests/tree_cat_fixtures.py)
with the score bound of tests/test_gpu_tree_paths.py, against the libraries' decision functions (the oracle), and asserts
`plan.kernel` and `plan.last_kernel`.  Labels and status words are compared exactly.
"""

import ctypes as C
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import tree_formats  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from mlrun_b200.plan import DevicePlan  # noqa: E402
from tests import device_emulator as emu  # noqa: E402
from tests import tree_cat_fixtures as fx  # noqa: E402
from tests.device_check import U32, U64, Rows, assert_kernel, check_close, names, run_device  # noqa: E402

CARDS = {0: 40, 3: 8, 5: 1001, 6: 33}


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def xgb_model(depth, n_feat=8, seed=0, n_trees=12, cards=CARDS, **kw):
    doc = fx.random_xgb_cat_model(n_trees=n_trees, depth=depth, n_feat=n_feat, cat_cards=cards, seed=seed, p_leaf=0.1, **kw)
    return doc, tree_formats.pack_xgboost_json(json.dumps(doc))


def lgbm_model(depth, n_feat=8, seed=0, n_trees=12, cards=CARDS, **kw):
    doc = fx.random_lgbm_cat_dump(n_trees=n_trees, depth=depth, n_feat=n_feat, cat_cards=cards, seed=seed, p_leaf=0.1, **kw)
    return doc, tree_formats.pack_lightgbm_dump(doc)


def max_depth(t):
    best = 0
    for ti in range(t.n_trees):
        base, stack = t.tree_offset[ti], [(0, 0)]
        while stack:
            nd, d = stack.pop()
            best = max(best, d)
            if t.feature[base + nd] >= 0:
                stack += [(t.left[base + nd], d + 1), (t.right[base + nd], d + 1)]
    return best


def check_scores(out, packed, X, ok):
    """identity-link output column vs the float64 walk: |out - ref| <= 2^-24 |ref| + (n_terms + 2) 2^-52 S"""
    sc, S, n_terms = fx.packed_walk(packed, X)
    check_close(out[ok], sc[ok, 0], (n_terms[0] + 2) * U64 * S[ok, 0], "scores")
    return sc[:, 0]


def inputs(n, n_feat=8, seed=0, cards=CARDS, nan_frac=0.05):
    X = fx.cat_inputs(n, n_feat, cards, seed=seed, nan_frac=nan_frac)
    # every edge value in every categorical column
    k = len(fx.EDGE_VALUES)
    for f in cards:
        X[:min(k, n), f] = fx.EDGE_VALUES[:min(k, n)]
    return X


# ------------------------------------------------------------------------------------------ trees3
@pytest.mark.parametrize("depth", [2, 3, 4, 5, 6, 7, 8])
def test_trees3_categorical_nan_routing(sms, depth):
    """trees3_kernel<D, NaN routing, categorical>: an xgboost and a LightGBM document side by side (both route NaN)"""
    xdoc, xm = xgb_model(depth, seed=depth)
    ldoc, lm = lgbm_model(depth, seed=depth + 100)
    assert max(max_depth(xm), max_depth(lm)) == depth
    X = inputs(4000, seed=depth)
    plan = ColumnProgram(names(8)).build_plan([("trees", xm), ("trees", lm)])
    assert_kernel(plan, f"trees3_kernel<D={depth},NaN routing,categorical>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3_cat"
    ok = ~np.isinf(X).any(axis=1)
    np.testing.assert_array_equal(st != 0, ~ok)
    check_scores(out[:, 0], xm, X, ok)
    check_scores(out[:, 1], lm, X, ok)
    np.testing.assert_allclose(out[ok, 0], fx.xgboost_predict(xdoc, X[ok]), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out[ok, 1], fx.lightgbm_predict(ldoc, X[ok]), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("depth", [2, 3, 4, 5, 6, 7, 8])
def test_trees3_categorical_floats_beside_a_linear_model(sms, depth):
    """trees3_kernel<D, floats, categorical>: a linear model in the plan turns NaN routing off; NaN rows are flagged"""
    doc, m = (xgb_model if depth % 2 else lgbm_model)(depth, seed=depth + 200)
    assert max_depth(m) == depth
    rng = np.random.default_rng(depth)
    lin = {"W": rng.normal(size=(1, 8)), "b": np.array([0.25]), "link": nat.LINK_IDENTITY, "classes": None}
    X = inputs(3000, seed=depth + 1)
    plan = ColumnProgram(names(8)).build_plan([("trees", m), ("linear", lin)])
    assert_kernel(plan, f"trees3_kernel<D={depth},floats,categorical>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3_cat"
    ok = np.isfinite(X).all(axis=1)
    assert (~ok).any()
    np.testing.assert_array_equal(st != 0, ~ok)
    check_scores(out[:, 0], m, X, ok)


def test_trees3_categorical_row_counts(sms):
    doc, m = lgbm_model(6, seed=7, n_trees=30)
    big = 3 * 64 * sms + 77
    X = inputs(big, seed=8)
    rows = Rows(X)
    plan = ColumnProgram(names(8)).build_plan([("trees", m)])
    assert_kernel(plan, "trees3_kernel<D=6,NaN routing,categorical>")
    sc = fx.packed_walk(m, X)
    for n in (1, 2, 63, 64, 65, 1000, big):
        out, st = run_device(plan, rows, n)
        assert plan.last_kernel == "trees3_cat"
        ok = ~np.isinf(X[:n]).any(axis=1)
        np.testing.assert_array_equal(st != 0, ~ok)
        check_close(out[ok, 0], sc[0][:n][ok, 0], (sc[2][0] + 2) * U64 * sc[1][:n][ok, 0], f"{n} rows")


def test_trees3_categorical_classifiers_and_vote(sms):
    """a binary xgboost and a 3-class LightGBM model: labels exact on the rows whose margin no rounding can flip"""
    _, xb = xgb_model(5, seed=31, objective="binary:logistic")
    _, lc = lgbm_model(5, seed=32, objective="multiclass", num_class=3)
    X = inputs(3000, seed=33)
    plan = ColumnProgram(names(8)).build_plan([("trees", xb), ("trees", lc)])
    assert_kernel(plan, "trees3_kernel<D=5,NaN routing,categorical>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3_cat"
    ok = ~np.isinf(X).any(axis=1)
    for j, m in enumerate((xb, lc)):
        sc, S, n_terms = fx.packed_walk(m, X)
        eps = (n_terms + 2) * U64 * S
        if sc.shape[1] == 1:
            sure = np.abs(sc[:, 0]) > 2 * eps[:, 0]
        else:
            srt = np.sort(sc, axis=1)
            sure = (srt[:, -1] - srt[:, -2]) > 2 * eps.max(axis=1)
        sure &= ok
        assert sure.sum() >= 0.99 * ok.sum()
        np.testing.assert_array_equal(out[sure, j], fx.packed_predict(m, X)[sure])


def test_trees3_categorical_imputer_fill_is_a_code(sms):
    """an Imputer in front: NaN in a categorical column becomes category 3 before the walk"""
    doc, m = lgbm_model(5, seed=41)
    X = inputs(2000, seed=42, nan_frac=0.2)
    prog = ColumnProgram(names(8))
    prog.imputer({"f0": 3.0, "f5": 1000.0})
    plan = prog.build_plan([("trees", m)])
    assert_kernel(plan, "trees3_kernel<D=5,NaN routing,categorical>")
    out, st = run_device(plan, X)
    E = X.copy()
    E[np.isnan(E[:, 0]), 0] = 3.0
    E[np.isnan(E[:, 5]), 5] = 1000.0
    ok = ~np.isinf(E).any(axis=1)
    np.testing.assert_array_equal(st != 0, ~ok)
    check_scores(out[:, 0], m, E, ok)
    np.testing.assert_allclose(out[ok, 0], fx.lightgbm_predict(doc, E[ok]), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------ rows_kernel<TREES>
def test_deep_categorical_trees_on_rows_kernel():
    """depth 10 (LightGBM's num_leaves=31 with max_depth=-1 grows past 8): rows_kernel<TREES>; NaN rows are flagged"""
    doc, m = lgbm_model(10, seed=51, n_trees=8)
    xdoc, xm = xgb_model(10, seed=52, n_trees=8)
    assert max_depth(m) == 10
    X = inputs(4000, seed=53, nan_frac=0.01)
    plan = ColumnProgram(names(8)).build_plan([("trees", m), ("trees", xm)])
    assert_kernel(plan, "rows_kernel<TREES,NS=1> (categorical splits)")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "rows_cat"
    ok = np.isfinite(X).all(axis=1)
    assert ok.any() and (~ok).any()
    np.testing.assert_array_equal(st != 0, ~ok)
    check_scores(out[:, 0], m, X, ok)
    check_scores(out[:, 1], xm, X, ok)
    np.testing.assert_allclose(out[ok, 0], fx.lightgbm_predict(doc, X[ok]), rtol=1e-5, atol=1e-5)


def test_categorical_trees_behind_a_onehot_encoder():
    """a OneHotEncoder in front: the trees read the expanded row (rows_kernel<TREES>)"""
    prog = ColumnProgram(names(8))
    prog.one_hot({"f7": [0, 1, 2]})
    X = inputs(3000, seed=61)
    X[:, 7] = np.random.default_rng(62).integers(0, 4, size=len(X))
    E = emu.transform(prog, X)
    n_out = E.shape[1]
    cards = {0: 40, 5: 1001}
    np.testing.assert_array_equal(E[:, [0, 5]], X[:, [0, 5]])  # the categorical columns pass through in place
    doc, m = xgb_model(5, n_feat=n_out, seed=63, cards=cards)
    plan = prog.build_plan([("trees", m)])
    assert_kernel(plan, "rows_kernel<TREES,NS=1> (categorical splits)")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "rows_cat"
    ok = np.isfinite(E).all(axis=1)
    np.testing.assert_array_equal(st != 0, ~ok)
    check_scores(out[:, 0], m, E, ok)


def test_sets_too_large_for_trees3_fall_back_to_rows_kernel():
    """one set of 59 375 words (codes up to 1.9 million) does not fit a trees3 CTA's shared memory"""
    doc, m = xgb_model(4, seed=71)
    # grow one set: categories up to 1 900 000 on the first categorical node of the first tree
    tree = next(t for t in doc["learner"]["gradient_booster"]["model"]["trees"] if t["categories_nodes"])
    j = 0
    seg, size = tree["categories_segments"][j], tree["categories_sizes"][j]
    cats = tree["categories"][seg:seg + size] + [1_900_000]
    tree["categories"] = tree["categories"][:seg] + cats + tree["categories"][seg + size:]
    tree["categories_sizes"][j] = len(cats)
    tree["categories_segments"] = [s + (1 if k > j else 0) for k, s in enumerate(tree["categories_segments"])]
    m = tree_formats.pack_xgboost_json(doc)
    assert len(m.cat_words) > 59_000
    X = inputs(2000, seed=72, nan_frac=0.0)
    X[:50, tree["split_indices"][tree["categories_nodes"][j]]] = 1_900_000.0
    plan = ColumnProgram(names(8)).build_plan([("trees", m)])
    assert_kernel(plan, "rows_kernel<TREES,NS=1> (categorical splits)")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "rows_cat"
    ok = np.isfinite(X).all(axis=1)
    check_scores(out[:, 0], m, X, ok)
    np.testing.assert_allclose(out[ok, 0], fx.xgboost_predict(doc, X[ok]), rtol=1e-5, atol=1e-5)


def test_wide_plan_on_rows_kernel():
    """420 columns leave trees3 no room: rows_kernel<TREES> walks the categorical splits"""
    n_in = 420
    doc, m = lgbm_model(6, n_feat=n_in, seed=81, n_trees=10)
    X = inputs(1000, n_feat=n_in, seed=82)
    plan = ColumnProgram(names(n_in)).build_plan([("trees", m)])
    assert_kernel(plan, "rows_kernel<TREES,NS=1> (categorical splits)")
    rows = Rows(X)
    for n in (1, 777, 1000):
        out, st = run_device(plan, rows, n)
        assert plan.last_kernel == "rows_cat"
        ok = np.isfinite(X[:n]).all(axis=1)
        np.testing.assert_array_equal(st != 0, ~ok)
        check_scores(out[:, 0], m, X[:n], ok)


# ------------------------------------------------------------------------------------------ served end to end
def test_served_through_model_servers():
    """a VotingEnsemble of categorical LightGBM and xgboost models, and a single FeatureRowModelServer, through run_batch
    and run_events, equal to the oracle's predict"""
    from mlrun_b200 import api

    xdoc, _ = xgb_model(5, seed=91)
    ldoc, _ = lgbm_model(5, seed=92)
    X = inputs(512, seed=93, nan_frac=0.0)
    X = X[np.isfinite(X).all(axis=1)]
    want = (fx.xgboost_predict(xdoc, X) + fx.lightgbm_predict(ldoc, X)) / 2
    fn = api.new_function("cat", kind="serving")
    graph = fn.set_topology("router", api.FeatureRowVotingEnsemble(vote_type="regression"))
    graph.add_route("m1", class_name="XGBoostModelServer", model=xdoc, model_path="")
    graph.add_route("m2", class_name="LGBMModelServer", model=ldoc, model_path="")
    server = fn.to_mock_server(namespace={"XGBoostModelServer": api.XGBoostModelServer, "LGBMModelServer": api.LGBMModelServer})
    out, status = server.run_batch(X, names=names(8), with_status=True)
    assert "categorical" in server.compile(names(8)).plan.kernel
    np.testing.assert_allclose(out[:, 0], want, rtol=1e-5, atol=1e-5)
    assert not status.any()
    bodies = [{f"f{j}": float(X[i, j]) for j in range(8)} for i in range(16)]
    resp = server.run_events(bodies)
    np.testing.assert_allclose([r["outputs"][0] for r in resp], want[:16], rtol=1e-5, atol=1e-5)

    fn1 = api.new_function("cat1", kind="serving")
    g1 = fn1.set_topology("router")
    g1.add_route("m", class_name="FeatureRowModelServer", model=ldoc, model_path="")
    s1 = fn1.to_mock_server(namespace={"FeatureRowModelServer": api.FeatureRowModelServer})
    out1 = s1.run_batch(X, names=names(8))
    np.testing.assert_allclose(out1[:, 0], fx.lightgbm_predict(ldoc, X), rtol=1e-5, atol=1e-5)
    resp1 = s1.run_events(bodies)
    np.testing.assert_allclose([r["outputs"][0] for r in resp1], fx.lightgbm_predict(ldoc, X[:16]), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------ the new entry point, numeric
def _add_through_cat_entry(plan, t):
    lib = plan._lib
    nat.check(lib.b2s_plan_add_tree_model_cat(
        plan._h, t.n_trees, nat._p(t.tree_offset, C.c_int32), nat._p(t.feature, C.c_int32), nat._p(t.threshold, C.c_float),
        nat._p(t.left, C.c_int32), nat._p(t.right, C.c_int32), nat._p(t.leaf_value, C.c_double),
        nat._p(t.tree_slot, C.c_int32), nat._p(t.tree_scale, C.c_double), nat._p(t.init, C.c_double), t.n_scores, t.link,
        None, 0, t.cmp_mode, nat._p(t.default_left, C.c_uint8), nat.NAN_DEFAULT_CHILD,
        nat._p(np.full(t.n_nodes, -1, dtype=np.int32), C.c_int32), None, 0, None, 0, nat.CAT_NONNEG))
    plan.n_models += 1


@pytest.mark.parametrize("depth", [6, 10])
def test_numeric_model_through_the_new_entry_point_is_bit_identical(depth):
    from tests import tree_fixtures as tf

    doc = tf.random_xgb_model(n_trees=20, depth=depth, n_feat=8, seed=depth, p_leaf=0.05)
    t = tree_formats.pack_xgboost_json(doc)
    X = tf.grid_inputs(3000, 8, seed=depth + 1)
    a = DevicePlan(8).add_trees(t).finalize()
    b = DevicePlan(8)
    _add_through_cat_entry(b, t)
    b.finalize()
    assert a.kernel == b.kernel and "categorical" not in b.kernel
    out_a, st_a = run_device(a, X)
    out_b, st_b = run_device(b, X)
    assert a.last_kernel == b.last_kernel
    np.testing.assert_array_equal(out_a.view(np.uint32), out_b.view(np.uint32))
    np.testing.assert_array_equal(st_a, st_b)


def test_bound_is_not_vacuous():
    """the score bound is far below the smallest leaf difference of the documents used here"""
    _, m = lgbm_model(6, seed=1)
    X = inputs(500, seed=2)
    sc, S, n_terms = fx.packed_walk(m, X)
    assert ((n_terms[0] + 2) * U64 * S[:, 0] + U32 * np.abs(sc[:, 0])).max() < 1e-5
