"""Tree plans on every kernel that can serve them, against plain float64 references.  Needs an H100: `-m gpu`.

A tree plan runs on one of two kernel families, chosen when the plan is finalized (b2s_plan_finalize):
  * t3_prep_kernel + trees3_kernel<D,MISS,U> + t3_vote_kernel: identity schema (+ Imputer), depth <= 8, <= 8 linear score
    columns, the part tables fit;
  * rows_kernel<TREES,NS>: everything else -- trees deeper than 8 levels (unconstrained scikit-learn forests), trees behind
    a OneHotEncoder or MapValues, more than 8 linear score columns, rows too wide for trees3's transposed tiles.
Every case asserts `plan.kernel` and, after the run, `plan.last_kernel`, so a plan that moves to another kernel fails.

Scores: every tree path accumulates in fp64 and rounds once to float32 on output.  Per element
    |out - ref| <= 2^-24 |ref| + (n_terms + 2) 2^-52 S,     S = |init| + sum |scale * leaf| along the row's paths
(n_terms: the trees of the score plus the init; for a linear scorer the columns plus the intercept, S = sum |x w| + |b|).
A mean vote adds one fp64 rounding per model.  `test_float32_accumulation_breaks_the_bound` checks that a float32
accumulator of the same trees does not fit this bound.  Labels, votes and status words are compared exactly; classifier
labels on the rows whose two best scores are further apart than twice the bound (at least 99 % of the rows).
"""

import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing, tree_formats  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from oracle import tree_libs  # noqa: E402
from tests import device_emulator as emu  # noqa: E402
from tests import tree_fixtures as fx  # noqa: E402
from tests.device_check import (ROW_BAD_LABEL, U32, U64, Ref, Rows, assert_kernel, check_close,  # noqa: E402
                                check_plan_output, names, run_device, run_host, tree_scores)


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def build(prog, models, vote=None):
    return prog.build_plan(models, vote=vote)


# ------------------------------------------------------------------------------------------ fitted models
def regression_data(n_feat, n=3000, seed=0, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, n_feat)).astype(np.float32)
    y = 2 * X[:, 0] + np.sin(3 * X[:, 1 % n_feat]) + X[:, 2 % n_feat] * X[:, 3 % n_feat] + 0.3 * rng.normal(size=n)
    if nan_frac:
        X[rng.random(X.shape) < nan_frac] = np.nan
    return X, y


def class_labels(X, K, seed=0, labels=None):
    rng = np.random.default_rng(seed + 1000)
    Xf = np.nan_to_num(X)
    z = Xf[:, 0] * 1.5 + Xf[:, 1 % X.shape[1]] + 0.5 * rng.normal(size=len(X))
    idx = np.clip(((z - z.min()) / (z.max() - z.min() + 1e-9) * K).astype(int), 0, K - 1)
    idx[:K] = np.arange(K)  # every class present
    return idx if labels is None else np.asarray(labels)[idx]


def gbr(n_feat, depth, n_trees, seed=0, **kw):
    from sklearn.ensemble import GradientBoostingRegressor

    X, y = regression_data(n_feat, seed=seed)
    return GradientBoostingRegressor(n_estimators=n_trees, max_depth=depth, random_state=seed, **kw).fit(X, y)


def gbc(n_feat, depth, n_trees, K, seed=0, labels=None):
    from sklearn.ensemble import GradientBoostingClassifier

    X, _ = regression_data(n_feat, seed=seed)
    return GradientBoostingClassifier(n_estimators=n_trees, max_depth=depth, random_state=seed).fit(X, class_labels(X, K, seed, labels))


def pk(model):
    return packing.pack_model(model)


def xgb(depth, n_feat, seed, n_trees=20, **kw):
    doc = fx.random_xgb_model(n_trees=n_trees, depth=depth, n_feat=n_feat, seed=seed, **kw)
    return doc, ("trees", tree_formats.pack_xgboost_json(json.dumps(doc)))


def lgbm(depth, n_feat, seed, n_trees=20):
    dump = fx.random_lgbm_dump(n_trees=n_trees, depth=depth, n_feat=n_feat, seed=seed)
    return dump, ("trees", tree_formats.pack_lightgbm_dump(dump))


def max_depth(packed):
    t = packed[1]
    best = 0
    for ti in range(t.n_trees):
        base, stack = t.tree_offset[ti], [(0, 0)]
        while stack:
            nd, d = stack.pop()
            best = max(best, d)
            if t.feature[base + nd] >= 0:
                stack += [(t.left[base + nd], d + 1), (t.right[base + nd], d + 1)]
    return best


def on_thresholds(X, models, seed, frac=0.3):
    """a copy of X in which a fraction of the rows carry, in every column, the threshold of some split on that column:
    walks then meet x == threshold, where `<=` and `<` part ways"""
    rng = np.random.default_rng(seed)
    X = X.copy()
    rows = np.flatnonzero(rng.random(len(X)) < frac)
    for _kind, t in models:
        split = t.feature >= 0
        f, thr = t.feature[split], emu.device_thresholds(t)[split]
        for _ in range(X.shape[1]):
            s = rng.integers(0, len(f), size=len(rows))
            X[rows, f[s]] = thr[s]
    return X


# ------------------------------------------------------------------------------------------ the bound itself
def test_float32_accumulation_breaks_the_bound():
    """the score bound is tight enough to catch a float32 accumulator: 100 depth-6 trees of a GradientBoostingRegressor"""
    model = gbr(16, 6, 100, seed=5)
    t = pk(model)[1]
    X = np.random.default_rng(6).normal(size=(4000, 16)).astype(np.float32)
    sc64, S, n_terms = tree_scores(t, X)
    np.testing.assert_allclose(sc64[:, 0], model.predict(X.astype(np.float64)), rtol=1e-12, atol=1e-12)
    sc32, _, _ = tree_scores(t, X, acc=np.float32)
    tol = U32 * np.abs(sc64[:, 0]) + (n_terms[0] + 2) * U64 * S[:, 0]
    assert (np.abs(sc32[:, 0] - sc64[:, 0]) > tol).mean() > 0.05


# ------------------------------------------------------------------------------------------ trees3: walks, loaders, shapes
@pytest.mark.parametrize("depth", [2, 3, 4, 5, 6, 7, 8])
def test_trees3_float_walk(sms, depth):
    """trees3_kernel<D, floats>: scikit-learn models of max_depth D"""
    models = [pk(gbr(16, depth, 12, seed=depth)), pk(gbr(16, depth, 7, seed=depth + 50, subsample=0.7))]
    assert max(max_depth(m) for m in models) == depth
    X = on_thresholds(np.random.default_rng(depth).normal(size=(5000, 16)).astype(np.float32), models, seed=depth)
    plan = build(ColumnProgram(names(16)), models)
    assert_kernel(plan, f"trees3_kernel<D={depth},floats>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3"  # 16 columns: no tensor map
    check_plan_output(out, st, models, X)
    want = np.stack([gbr(16, depth, 12, seed=depth).predict(X.astype(np.float64))], axis=1)
    check_close(out[:, :1], want, Ref(models, X).bound[:, :1], "sklearn")


@pytest.mark.parametrize("depth", [2, 3, 4, 5, 6, 7, 8])
def test_trees3_nan_routing_walk(sms, depth):
    """trees3_kernel<D, NaN routing>: xgboost (odd D) and LightGBM (even D) documents; inputs from the threshold grid, so
    x == threshold, +-0, +-1e-40 and -inf thresholds meet NaN on every tree"""
    X = fx.grid_inputs(4000, 12, seed=100 + depth)
    if depth % 2:
        doc, model = xgb(depth, 12, seed=depth, p_leaf=0.1)
        want = tree_libs.xgboost_predict(doc, X[:400])
    else:
        doc, model = lgbm(depth, 12, seed=depth)
        want = tree_libs.lightgbm_predict(doc, X[:400])
    assert max_depth(model) == depth
    plan = build(ColumnProgram(names(12)), [model])
    assert_kernel(plan, f"trees3_kernel<D={depth},NaN routing>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3"
    ref = check_plan_output(out, st, [model], X, routes_nan=True)
    assert not st.any()
    # xgboost itself adds the leaves in float32, LightGBM in float64
    check_close(out[:400, 0], want, (2.0 ** 28 if depth % 2 else 1.0) * ref.bound[:400, 0], "library")


LOADERS = [(64, "device", "trees3/tma"), (64, "host", "trees3/tma"), (20, "device", "trees3"), (13, "device", "trees3"),
           (64, "small", "trees3")]


@pytest.mark.parametrize("miss", [False, True], ids=["floats", "nan"])
@pytest.mark.parametrize("n_in,how,kernel", LOADERS, ids=["tma", "tma-pageable", "cp16", "cp4", "small-host"])
def test_trees3_prep_loaders(sms, n_in, how, kernel, miss):
    """t3_prep_kernel's loaders under both MISS values: TMA boxes (n_in a multiple of 32; also a large pageable host batch),
    16-byte cp.async (a multiple of 4), 4-byte copies (odd n_in), and a small host batch read from mapped memory"""
    if miss:
        _, model = xgb(5, n_in, seed=n_in)
        X = fx.grid_inputs(70000 if how == "host" else (200 if how == "small" else 9000), n_in, seed=n_in)
    else:
        model = pk(gbr(n_in, 5, 15, seed=n_in))
        X = np.random.default_rng(n_in).normal(size=(70000 if how == "host" else (200 if how == "small" else 9000), n_in))
        X = X.astype(np.float32)
        X[7, n_in - 1] = np.nan
        X[8, 0] = -np.inf
    plan = build(ColumnProgram(names(n_in)), [model])
    assert_kernel(plan, "trees3_kernel<D=5", "NaN routing" if miss else "floats")
    out, st = run_device(plan, X) if how == "device" else run_host(plan, X)
    assert plan.last_kernel == kernel
    check_plan_output(out, st, [model], X, routes_nan=miss)


def test_trees3_row_counts(sms):
    """1, 63, 64, 65 rows, and 3 * 64 * SMs + 77: every CTA then walks more than two tiles, so the two-deep tile ring and
    the partial-sum buffer waits turn over"""
    models = [pk(gbr(32, 6, 30, seed=1)), pk(gbr(32, 4, 40, seed=2))]
    n_max = 3 * 64 * sms + 77
    X = np.random.default_rng(9).normal(size=(n_max, 32)).astype(np.float32)
    X[n_max - 1, 3] = np.nan
    rows = Rows(X)
    plan = build(ColumnProgram(names(32)), models, vote=(nat.VOTE_MEAN, [0.3, 0.7]))
    assert_kernel(plan, "trees3_kernel<D=6,floats>")
    for n in (1, 63, 64, 65, n_max):
        out, st = run_device(plan, rows, n)
        assert plan.last_kernel == "trees3/tma"
        check_plan_output(out, st, models, X[:n], vote=(nat.VOTE_MEAN, [0.3, 0.7]))


def test_trees3_imputer_before_nan_routing():
    """an Imputer in front of NaN-routing trees: imputed columns are filled first, NaN in the others takes each node's
    default child (scikit-learn forests fitted on data with NaN)"""
    from sklearn.ensemble import RandomForestRegressor

    Xf, y = regression_data(12, seed=21, nan_frac=0.1)
    model = RandomForestRegressor(n_estimators=16, max_depth=7, random_state=0).fit(Xf, y)
    packed = pk(model)
    assert packed[1].nan_ok
    X = fx.grid_inputs(6000, 12, seed=22, nan_frac=0.2, with_inf=True)
    mapping = {f"f{i}": 0.25 * i - 1.0 for i in range(0, 12, 3)}
    prog = ColumnProgram(names(12))
    prog.imputer(mapping)
    plan = build(prog, [packed])
    assert_kernel(plan, "trees3_kernel<D=7,NaN routing>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3"
    Xi = emu.transform(prog, X)
    assert np.isnan(Xi).any()
    ref = check_plan_output(out, st, [packed], Xi, routes_nan=True)
    ok = ~np.isinf(Xi).any(axis=1)
    check_close(out[ok, 0], model.predict(Xi[ok].astype(np.float64)), ref.bound[ok, 0], "sklearn")


@pytest.mark.parametrize("n_lin,big", [(1, False), (3, False), (3, True), (8, False), (8, True)])
def test_trees3_linear_part(sms, n_lin, big):
    """the linear part of a mixed ensemble at 1, 3 and 8 score columns, beside small tree tables (its feature slices live
    in the partial-sum buffers) and large ones (the slices alias the tree tables)"""
    from sklearn.linear_model import LogisticRegression

    K = 2 if n_lin == 1 else n_lin
    X, _ = regression_data(32, seed=30 + n_lin)
    lab = class_labels(X, K, seed=n_lin)
    lin = pk(LogisticRegression(max_iter=400).fit(X, lab))
    trees = [pk(gbc(32, 8 if big else 3, 16 if big else 4, K, seed=s)) for s in range(2)]
    models = [lin] + trees
    Xt = np.random.default_rng(31).normal(size=(7000, 32)).astype(np.float32)
    for vote in (None, (nat.VOTE_MAJORITY, [0.5, 0.3, 0.2])):
        plan = build(ColumnProgram(names(32)), models, vote=vote)
        assert_kernel(plan, "trees3_kernel")
        out, st = run_device(plan, Xt)
        assert plan.last_kernel == "trees3/tma"
        check_plan_output(out, st, models, Xt, vote=vote)


def test_nine_linear_columns_leave_trees3():
    """9 linear score columns exceed the linear part (8): the plan runs on rows_kernel"""
    from sklearn.linear_model import LogisticRegression

    X, _ = regression_data(16, seed=40)
    lab = class_labels(X, 9, seed=40)
    models = [pk(LogisticRegression(max_iter=400).fit(X, lab)), pk(gbc(16, 3, 3, 9, seed=1))]
    plan = build(ColumnProgram(names(16)), models)
    assert_kernel(plan, "rows_kernel<TREES,NS=16>")
    Xt = np.random.default_rng(41).normal(size=(3000, 16)).astype(np.float32)
    out, st = run_device(plan, Xt)
    assert plan.last_kernel == "rows"
    check_plan_output(out, st, models, Xt)


LINK_VOTES = [(link, vote) for link in ("identity", "binary_ge", "argmax") for vote in ("none", "mean", "majority")
              if not (vote == "mean" and link != "identity")]  # VotingEnsemble averages regressors only


@pytest.mark.parametrize("link,vote", LINK_VOTES)
def test_trees3_links_and_votes(link, vote):
    """links x votes on trees3, with non-contiguous class labels; a negative label under a majority vote flags its row"""
    if link == "identity":
        models = [pk(gbr(16, 4, 10, seed=s)) for s in range(3)]
    elif link == "binary_ge":
        models = [pk(gbc(16, 4, 10, 2, seed=s, labels=[-2, 5] if s == 1 else [3, 7])) for s in range(3)]
    else:
        models = [pk(gbc(16, 4, 6, 3, seed=s, labels=[3, 7, 11] if s != 1 else [-1, 7, 11])) for s in range(3)]
    w = [0.5, 0.2, 0.3]
    v = None if vote == "none" else ((nat.VOTE_MEAN if vote == "mean" else nat.VOTE_MAJORITY), w)
    X = np.random.default_rng(50).normal(size=(6000, 16)).astype(np.float32)
    X[11, 2] = np.inf
    plan = build(ColumnProgram(names(16)), models, vote=v)
    assert_kernel(plan, "trees3_kernel<D=4,floats>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3"
    ref = check_plan_output(out, st, models, X, vote=v)
    if vote == "majority" and link != "identity":
        assert (ref.pred < 0).any() and ((st & ROW_BAD_LABEL) != 0).any()


@pytest.mark.parametrize("shape,vote", [("4x10", "none"), ("4x10", "majority"), ("2x20", "none")])
def test_trees3_more_than_32_scores_in_one_plan(sms, shape, vote):
    """a plan may hold up to 16 models of up to 32 scores each: 4 x 10-class (40 score columns) and 2 x 20-class
    GradientBoostingClassifiers stay on trees3, whose vote holds one model's scores at a time"""
    M, K = (4, 10) if shape == "4x10" else (2, 20)
    models = [pk(gbc(16, 3, 3, K, seed=s)) for s in range(M)]
    v = None if vote == "none" else (nat.VOTE_MAJORITY, [1.0 / M] * M)
    plan = build(ColumnProgram(names(16)), models, vote=v)
    assert_kernel(plan, "trees3_kernel<D=3,floats>", f"{M * K} parts")
    X = np.random.default_rng(60).normal(size=(5000, 16)).astype(np.float32)
    out, st = run_device(plan, X)
    assert plan.last_kernel == "trees3"
    check_plan_output(out, st, models, X, vote=v)


# ------------------------------------------------------------------------------------------ rows_kernel<TREES,NS>: wide rows
def wide_rows(n, n_in, seed, models):
    X = on_thresholds(np.random.default_rng(seed).normal(size=(n, n_in)).astype(np.float32), models, seed)
    X[n // 3, 2] = np.nan
    X[n // 2, n_in - 1] = np.inf
    return X


@pytest.mark.parametrize("case", ["420-cp16", "419-cp4", "416-d7", "408-ns4"])
def test_wide_rows_on_rows_kernel(case):
    """plans trees3 cannot hold (two transposed tiles of rows this wide leave no room for a table) run on
    rows_kernel<TREES>: 420 columns (16-byte loads), 419 (4-byte), 416 at depth 7, and a majority vote of a binary depth-8
    classifier and a 3-class one over 408 columns (NS = 4).  At these widths the kernel's shared-memory budget leaves one
    tile stage, and a single model's tile shrinks from 256 to 128 rows: code that only wide rows reach"""
    n_in = int(case.split("-")[0])
    vote = None
    if case == "408-ns4":
        models = [pk(gbc(n_in, 8, 1, 2, seed=1)), pk(gbc(n_in, 1, 1, 3, seed=2))]
        assert max_depth(models[0]) == 8
        vote = (nat.VOTE_MAJORITY, [0.6, 0.4])
        want_kernel = "rows_kernel<TREES,NS=4>"
    else:
        models = [pk(gbr(n_in, 7 if n_in == 416 else 6, 6 if n_in == 416 else 10, seed=n_in))]
        assert max_depth(models[0]) == (7 if n_in == 416 else 6)  # one level less would fit trees3 at 416 columns
        want_kernel = "rows_kernel<TREES,NS=1>"
    plan = build(ColumnProgram(names(n_in)), models, vote=vote)
    assert_kernel(plan, want_kernel)
    X = wide_rows(1000, n_in, n_in, models)
    rows = Rows(X)
    for n in (1, 65, 777, 1000):
        out, st = run_device(plan, rows, n)
        assert plan.last_kernel == "rows"
        check_plan_output(out, st, models, X[:n], vote=vote)


# ------------------------------------------------------------------------------------------ rows_kernel<TREES,NS>
@pytest.mark.parametrize("name,K,ns", [("RandomForestRegressor", 0, 1), ("ExtraTreesRegressor", 0, 1),
                                       ("DecisionTreeRegressor", 0, 1), ("RandomForestClassifier", 2, 4),
                                       ("RandomForestClassifier", 3, 4), ("RandomForestClassifier", 5, 8),
                                       ("RandomForestClassifier", 9, 16), ("RandomForestClassifier", 17, 32),
                                       ("RandomForestClassifier", 20, 32), ("RandomForestClassifier", 32, 32)])
def test_unconstrained_sklearn_trees_on_rows_kernel(name, K, ns):
    """max_depth=None grows trees far deeper than 8 levels: rows_kernel<TREES,NS>, NS = 1 / 4 / 8 / 16 / 32 (17 to 32
    classes need NS = 32).  Forests of 16 fully grown trees have 0/1 leaf probabilities: every scaled sum is exact, so every
    row's label is compared, ties included"""
    import sklearn.ensemble as ens
    import sklearn.tree as tree

    cls = getattr(ens, name, None) or getattr(tree, name)
    kw = {} if name.startswith("Decision") else {"n_estimators": 16}
    X, y = regression_data(16, n=3000, seed=K + 70)
    model = cls(random_state=0, **kw).fit(X, class_labels(X, K, seed=K) if K else y)
    packed = pk(model)
    assert max_depth(packed) > 8
    plan = build(ColumnProgram(names(16)), [packed])
    assert_kernel(plan, f"rows_kernel<TREES,NS={ns}>")
    Xt = on_thresholds(np.random.default_rng(K + 71).normal(size=(5000, 16)).astype(np.float32), [packed], seed=K)
    Xt[3, 1] = np.inf
    out, st = run_device(plan, Xt)
    assert plan.last_kernel == "rows"
    ok = np.isfinite(Xt).all(axis=1)
    np.testing.assert_array_equal(st != 0, ~ok)
    if K:
        np.testing.assert_array_equal(out[ok, 0], model.predict(Xt[ok].astype(np.float64)))
    else:
        ref = check_plan_output(out, st, [packed], Xt)
        check_close(out[ok, 0], model.predict(Xt[ok].astype(np.float64)), ref.bound[ok, 0], "sklearn")


def test_depth10_xgboost_document_on_rows_kernel():
    """a depth-10 xgboost document: `x < t` as `x <= prev(t)` and NaN (-inf) thresholds on the generic walk; its NaN rows
    are flagged there (NaN routing is honoured on trees3 only)"""
    doc, model = xgb(10, 8, seed=3, n_trees=12, p_leaf=0.05)
    assert max_depth(model) == 10
    X = fx.grid_inputs(5000, 8, seed=4, nan_frac=0.01)
    plan = build(ColumnProgram(names(8)), [model])
    assert_kernel(plan, "rows_kernel<TREES,NS=1>")
    out, st = run_device(plan, X)
    assert plan.last_kernel == "rows"
    ok = np.isfinite(X).all(axis=1)
    assert ok.any() and (~ok).any()
    ref = check_plan_output(out, st, [model], X, ok=ok)
    # xgboost itself adds the leaves in float32
    check_close(out[ok, 0][:500], tree_libs.xgboost_predict(doc, X[ok][:500]), 2.0 ** 28 * ref.bound[ok, 0][:500], "xgboost")


def categorical_rows(n, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, 6)).astype(np.float32)
    X[:, 4] = rng.choice(np.array([0, 1, 2, 3, 7, np.inf, -np.inf, np.nan], dtype=np.float32), n)
    X[:, 5] = rng.choice(np.array([10, 20, 30, 99, np.nan], dtype=np.float32), n)
    X[5, 0] = np.nan
    return X


@pytest.mark.parametrize("steps", ["onehot", "mapvalues", "imputer+onehot"])
def test_trees_behind_feature_steps_on_rows_kernel(steps):
    """trees behind a OneHotEncoder / MapValues read the expanded row; categorical edge values (+-Inf, NaN,
    out-of-vocabulary) become all-zero one-hot columns, so only non-finite numeric columns flag a row"""
    from sklearn.ensemble import GradientBoostingRegressor

    prog = ColumnProgram(names(6))
    if "imputer" in steps:
        prog.imputer({"f0": 0.5, "f5": 20.0})
    if "onehot" in steps:
        prog.one_hot({"f4": [0, 1, 2, 3], "f5": [10, 20, 30]})
    else:
        prog.map_values({"f0": {"ranges": {1: ["-inf", 0], 2: [0, "inf"]}}, "f1": {"ranges": {5: [-1, 1]}},
                         "f4": {0: 10, 1: 11, 2: 12}, "f5": {10: -1, 20: 1}})
    Xfit = categorical_rows(4000, seed=80)
    Efit = emu.transform(prog, Xfit)
    yfit = np.nan_to_num(Efit).sum(axis=1) + np.sin(np.nan_to_num(Efit[:, 0]))
    keep = np.isfinite(Efit).all(axis=1)
    model = GradientBoostingRegressor(n_estimators=20, max_depth=4, random_state=0).fit(Efit[keep], yfit[keep])
    packed = pk(model)
    plan = build(prog, [packed])
    assert_kernel(plan, "rows_kernel<TREES,NS=1>")
    X = categorical_rows(3000, seed=81)
    out, st = run_device(plan, X)
    assert plan.last_kernel == "rows"
    E = emu.transform(prog, X)
    ref = check_plan_output(out, st, [packed], E)
    ok = np.isfinite(E).all(axis=1)
    check_close(out[ok, 0], model.predict(E[ok].astype(np.float64)), ref.bound[ok, 0], "sklearn")


def test_mixed_ensemble_with_many_linear_columns_on_rows_kernel():
    """a 17-class LogisticRegression beside a 17-class forest: 17 linear score columns, NS = 32"""
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.linear_model import LogisticRegression

    X, _ = regression_data(16, seed=90)
    lab = class_labels(X, 17, seed=90)
    models = [pk(LogisticRegression(max_iter=300).fit(X, lab)),
              pk(RandomForestClassifier(n_estimators=4, max_depth=6, random_state=0).fit(X, lab))]
    Xt = np.random.default_rng(91).normal(size=(4000, 16)).astype(np.float32)
    for vote in (None, (nat.VOTE_MAJORITY, [0.7, 0.3])):
        plan = build(ColumnProgram(names(16)), models, vote=vote)
        assert_kernel(plan, "rows_kernel<TREES,NS=32>")
        out, st = run_device(plan, Xt)
        assert plan.last_kernel == "rows"
        check_plan_output(out, st, models, Xt, vote=vote)


@pytest.mark.parametrize("M", [3, 5, 16])
def test_many_models_on_rows_kernel(M):
    """3, 5 and 16 deep forests: the per-row prediction table is padded to a power of two of models and the tile shrinks
    to 16 rows at 16 models"""
    from sklearn.ensemble import RandomForestRegressor

    X, y = regression_data(10, n=1500, seed=M)
    models = [pk(RandomForestRegressor(n_estimators=3, random_state=s).fit(X, y + s)) for s in range(M)]
    w = list(np.random.default_rng(M).random(M))
    Xt = np.random.default_rng(M + 1).normal(size=(2500, 10)).astype(np.float32)
    for vote in (None, (nat.VOTE_MEAN, w)):
        plan = build(ColumnProgram(names(10)), models, vote=vote)
        assert_kernel(plan, "rows_kernel<TREES,NS=1>")
        out, st = run_device(plan, Xt)
        assert plan.last_kernel == "rows"
        check_plan_output(out, st, models, Xt, vote=vote)


# ------------------------------------------------------------------------------------------ the NaN contract of the fallbacks
def test_nan_routing_models_flag_nan_rows_on_rows_kernel():
    """b2s_plan_add_tree_model_ex: NaN routing is honoured on trees3 only; elsewhere a NaN row is flagged, never answered
    differently.  A scikit-learn forest fitted on NaN (rows_kernel: depth > 8) and an xgboost document over 420 columns
    (rows_kernel: too wide for trees3): NaN rows get status bit 1, Inf rows too, every other row matches the reference"""
    from sklearn.ensemble import RandomForestRegressor

    Xf, y = regression_data(12, seed=95, nan_frac=0.1)
    forest = pk(RandomForestRegressor(n_estimators=8, random_state=0).fit(Xf, y))
    assert forest[1].nan_ok and max_depth(forest) > 8
    _, wide = xgb(6, 420, seed=96, n_trees=10)
    for packed, n_in, kernel, ran in ((forest, 12, "rows_kernel<TREES,NS=1>", "rows"),
                                      (wide, 420, "rows_kernel<TREES,NS=1>", "rows")):
        plan = build(ColumnProgram(names(n_in)), [packed])
        assert_kernel(plan, kernel)
        X = fx.grid_inputs(3000, n_in, seed=n_in, nan_frac=0.0005 if n_in > 100 else 0.02)
        X[::97, n_in // 2] = np.inf
        X[1::89, 0] = -np.inf
        out, st = run_device(plan, X)
        assert plan.last_kernel == ran
        ok = np.isfinite(X).all(axis=1)
        assert (np.isnan(X).any(axis=1) & ~np.isinf(X).any(axis=1)).any() and ok.sum() > 100
        check_plan_output(out, st, [packed], X, ok=ok)


# ------------------------------------------------------------------------------------------ one model on both tree kernels
def test_same_model_on_trees3_and_rows_kernel():
    """the same packed ensemble on trees3 (16 columns), rows_kernel over rows too wide for trees3 (padded with unused zero
    columns to 420) and rows_kernel behind a OneHotEncoder on an unused column: each within the bound of the reference,
    and of each other"""
    models = [pk(gbr(16, 6, 10, seed=11)), pk(gbr(16, 5, 8, seed=12))]
    X = on_thresholds(np.random.default_rng(13).normal(size=(4000, 16)).astype(np.float32), models, seed=13)
    ref = Ref(models, X)
    outs = {}
    plan = build(ColumnProgram(names(16)), models)
    assert_kernel(plan, "trees3_kernel<D=6,floats>")
    outs["trees3"] = run_device(plan, X)[0]
    Xw = np.zeros((4000, 420), dtype=np.float32)
    Xw[:, :16] = X
    plan = build(ColumnProgram(names(420)), models)
    assert_kernel(plan, "rows_kernel<TREES,NS=1>")
    outs["rows/wide"] = run_device(plan, Xw)[0]
    assert plan.last_kernel == "rows"
    Xo = np.concatenate([X, np.zeros((4000, 1), dtype=np.float32)], axis=1)
    prog = ColumnProgram(names(17))
    prog.one_hot({"f16": [5.0]})
    plan = build(prog, models)
    assert_kernel(plan, "rows_kernel<TREES,NS=1>")
    outs["rows"] = run_device(plan, Xo)[0]
    assert plan.last_kernel == "rows"
    for k, out in outs.items():
        check_close(out, ref.pred, ref.bound, k)
    for a in outs:
        for b in outs:
            check_close(outs[a], outs[b].astype(np.float64), 2 * ref.bound + U32 * np.abs(ref.pred), f"{a} vs {b}")
