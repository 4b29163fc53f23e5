"""Categorical splits of xgboost and LightGBM models, without a GPU: the oracle against hand-worked cases, the exporters'
canonical form against the oracle, and the refusals."""

import ctypes as C

import numpy as np
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200 import tree_formats
from mlrun_b200.packing import UnsupportedModel
from tests import tree_cat_fixtures as fx

NAN = float("nan")
# x, then the leaf reached for the literal one-node documents below (1.0: left leaf, 2.0: right leaf)
#            x        xgboost  LightGBM
LITERAL = [(NAN,      1.0,     2.0),   # xgboost: default child (left); LightGBM: always right
           (-1.0,     1.0,     2.0),   # invalid code: xgboost left, LightGBM right
           (-0.5,     1.0,     1.0),   # xgboost: x < 0 is invalid; LightGBM: trunc -> code 0, in its set -> left
           (-0.0,     1.0,     1.0),   # code 0: not in xgboost's set (left), in LightGBM's (left)
           (0.0,      1.0,     1.0),
           (1.0,      2.0,     2.0),   # in xgboost's set (right); not in LightGBM's (right)
           (2.7,      1.0,     2.0),   # code 2: in neither
           (3.9,      2.0,     1.0),   # code 3: in both
           (31.0,     1.0,     2.0),   # word boundary: 31 in neither, 32 in both, 33 in neither
           (32.0,     2.0,     1.0),
           (33.0,     1.0,     2.0),
           (999.0,    1.0,     2.0),   # a set spanning 32 words
           (1000.0,   2.0,     1.0),
           (5000.0,   1.0,     2.0),   # past the end of the bitset
           (3e9,      1.0,     2.0)]   # beyond int32: outside the set


def _xgb_doc(trees, objective="reg:squarederror", base_score=0.0, num_class=0):
    return {"learner": {"gradient_booster": {"name": "gbtree", "model": {
        "trees": trees, "tree_info": [0] * len(trees), "gbtree_model_param": {"num_trees": str(len(trees))}}},
        "learner_model_param": {"base_score": repr(base_score), "num_class": str(num_class), "num_feature": "2"},
        "objective": {"name": objective}}}


def _xgb_one_cat_node(categories, default_left=1):
    return _xgb_doc([{"left_children": [1, -1, -1], "right_children": [2, -1, -1], "split_conditions": [0.0, 1.0, 2.0],
                      "split_indices": [0, 0, 0], "default_left": [default_left, 0, 0], "split_type": [1, 0, 0],
                      "categories": categories, "categories_nodes": [0], "categories_segments": [0],
                      "categories_sizes": [len(categories)]}])


def _lgbm_doc(root, objective="regression"):
    return {"num_class": 1, "num_tree_per_iteration": 1, "max_feature_idx": 1, "objective": objective,
            "tree_info": [{"tree_index": 0, "tree_structure": root}]}


def _lgbm_one_cat_node(threshold, default_left=True, missing_type="None"):
    return _lgbm_doc({"split_feature": 0, "decision_type": "==", "threshold": threshold, "default_left": default_left,
                      "missing_type": missing_type, "left_child": {"leaf_value": 1.0}, "right_child": {"leaf_value": 2.0}})


XGB_SET = [1, 3, 32, 1000]
LGBM_SET = "0||3||32||1000"


def _column(xs):
    X = np.zeros((len(xs), 2), dtype=np.float32)
    X[:, 0] = xs
    return X


@pytest.mark.parametrize("default_left", [0, 1])
def test_xgboost_oracle_literal(default_left):
    X = _column([c[0] for c in LITERAL])
    want = np.array([c[1] for c in LITERAL])
    want[0] = 1.0 if default_left else 2.0  # NaN follows the default child
    doc = _xgb_one_cat_node(XGB_SET, default_left)
    np.testing.assert_array_equal(fx.xgboost_predict(doc, X), want)
    # the exporter's canonical form takes the same branches
    np.testing.assert_array_equal(fx.packed_predict(tree_formats.pack_xgboost_json(doc), X), want)


@pytest.mark.parametrize("default_left,missing_type", [(True, "None"), (False, "NaN"), (True, "NaN")])
def test_lightgbm_oracle_literal(default_left, missing_type):
    X = _column([c[0] for c in LITERAL])
    want = np.array([c[2] for c in LITERAL])  # NaN goes right whatever default_left and missing_type say
    doc = _lgbm_one_cat_node(LGBM_SET, default_left, missing_type)
    np.testing.assert_array_equal(fx.lightgbm_predict(doc, X), want)
    np.testing.assert_array_equal(fx.packed_predict(tree_formats.pack_lightgbm_dump(doc), X), want)


def test_mixed_numeric_and_categorical_literal():
    # xgboost: root f1 < 0.5 -> node 1 (categories [2]: not listed -> leaf 10, listed -> leaf 20); else leaf 5
    xgb = _xgb_doc([{"left_children": [1, 3, -1, -1, -1], "right_children": [2, 4, -1, -1, -1],
                     "split_conditions": [0.5, 0.0, 5.0, 10.0, 20.0], "split_indices": [1, 0, 0, 0, 0],
                     "default_left": [0, 0, 0, 0, 0], "split_type": [0, 1, 0, 0, 0], "categories": [2],
                     "categories_nodes": [1], "categories_segments": [0], "categories_sizes": [1]}])
    # LightGBM: root f1 <= 0.5 -> categorical node ("1||2" -> leaf 10, else leaf 20); else leaf 5
    lgbm = _lgbm_doc({"split_feature": 1, "decision_type": "<=", "threshold": 0.5, "missing_type": "None", "default_left": True,
                      "left_child": {"split_feature": 0, "decision_type": "==", "threshold": "1||2", "missing_type": "None",
                                     "default_left": False, "left_child": {"leaf_value": 10.0}, "right_child": {"leaf_value": 20.0}},
                      "right_child": {"leaf_value": 5.0}})
    X = np.array([[2, 0], [1, 0], [2, 1], [NAN, 0], [1, 0.5], [-0.5, 0]], dtype=np.float32)
    want_xgb = [20.0, 10.0, 5.0, 20.0, 5.0, 10.0]  # row 3: NaN takes node 1's default child (right)
    want_lgbm = [10.0, 10.0, 5.0, 20.0, 10.0, 20.0]
    np.testing.assert_array_equal(fx.xgboost_predict(xgb, X), want_xgb)
    np.testing.assert_array_equal(fx.lightgbm_predict(lgbm, X), want_lgbm)
    np.testing.assert_array_equal(fx.packed_predict(tree_formats.pack_xgboost_json(xgb), X), want_xgb)
    np.testing.assert_array_equal(fx.packed_predict(tree_formats.pack_lightgbm_dump(lgbm), X), want_lgbm)


def test_canonical_form():
    """xgboost keeps its children; LightGBM's swap, and NaN takes LightGBM's right child (canonical left)"""
    px = tree_formats.pack_xgboost_json(_xgb_one_cat_node([1, 33], default_left=0))
    assert px.cat_mode == nat.CAT_NONNEG and px.node_cat.tolist() == [0, -1, -1]
    assert px.cat_offsets.tolist() == [0, 2] and px.cat_words.tolist() == [1 << 1, 1 << 1]
    assert (px.left[0], px.right[0], px.default_left[0]) == (1, 2, 0)
    pl = tree_formats.pack_lightgbm_dump(_lgbm_one_cat_node("0||31", default_left=False, missing_type="NaN"))
    assert pl.cat_mode == nat.CAT_TRUNC and pl.node_cat.tolist() == [0, -1, -1]
    assert pl.cat_offsets.tolist() == [0, 1] and pl.cat_words.tolist() == [1 | (1 << 31)]
    assert pl.leaf_value[pl.left[0]] == 2.0 and pl.leaf_value[pl.right[0]] == 1.0 and pl.default_left[0] == 1


def test_numeric_models_keep_the_old_form():
    from tests import tree_fixtures as tf

    assert tree_formats.pack_xgboost_json(tf.random_xgb_model(seed=1)).node_cat is None
    assert tree_formats.pack_lightgbm_dump(tf.random_lgbm_dump(seed=1)).node_cat is None
    assert tree_formats.pack_xgboost_json(fx.random_xgb_cat_model(seed=1, p_cat=0.0)).node_cat is None


CASES = [("reg:squarederror", 0, "regression", 1), ("binary:logistic", 0, "binary", 1), ("multi:softprob", 3, "multiclass", 3)]


@pytest.mark.parametrize("xgb_obj,xgb_nc,lgbm_obj,lgbm_nc", CASES)
@pytest.mark.parametrize("seed", [0, 1])
def test_exporters_match_the_oracle(xgb_obj, xgb_nc, lgbm_obj, lgbm_nc, seed):
    cards = {0: 40, 2: 8, 5: 1001}
    X = fx.cat_inputs(300, 8, cards, seed=seed + 10)
    xdoc = fx.random_xgb_cat_model(n_trees=6, depth=5, cat_cards=cards, seed=seed, objective=xgb_obj, num_class=xgb_nc)
    px = tree_formats.pack_xgboost_json(xdoc)
    assert px.node_cat is not None and (px.node_cat >= 0).any()
    ref, _ = fx.xgboost_margins(xdoc, X)
    got = fx.packed_scores(px, X)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6)
    np.testing.assert_array_equal(fx.packed_predict(px, X), fx.xgboost_predict(xdoc, X))
    ldoc = fx.random_lgbm_cat_dump(n_trees=6, depth=5, cat_cards=cards, seed=seed, objective=lgbm_obj, num_class=lgbm_nc)
    pl = tree_formats.pack_lightgbm_dump(ldoc)
    ref, _ = fx.lightgbm_raw(ldoc, X)
    np.testing.assert_allclose(fx.packed_scores(pl, X), ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_array_equal(fx.packed_predict(pl, X), fx.lightgbm_predict(ldoc, X))


def test_get_dump_refuses_categorical_nodes():
    dump = [{"nodeid": 0, "depth": 0, "split": "f0", "split_condition": [1, 3], "yes": 2, "no": 1, "missing": 2,
             "children": [{"nodeid": 1, "leaf": 1.0}, {"nodeid": 2, "leaf": 2.0}]}]
    with pytest.raises(UnsupportedModel, match="save_model"):
        tree_formats.pack_xgboost_dump(dump)


def test_negative_category_in_a_document_is_refused():
    with pytest.raises(UnsupportedModel, match="negative category"):
        tree_formats.pack_xgboost_json(_xgb_one_cat_node([-3, 2]))


# ------------------------------------------------------------------------------------------ the C-ABI's checks
def _cat_call(lib, plan, packed, node_cat=None, cat_offsets=None, n_sets=None, cat_words=None, n_words=None, cat_mode=None):
    t = packed
    node_cat = np.ascontiguousarray(t.node_cat if node_cat is None else node_cat, dtype=np.int32)
    offs = np.ascontiguousarray(t.cat_offsets if cat_offsets is None else cat_offsets, dtype=np.int32)
    words = np.ascontiguousarray(t.cat_words if cat_words is None else cat_words, dtype=np.uint32)
    return lib.b2s_plan_add_tree_model_cat(
        plan, t.n_trees, nat._p(t.tree_offset, C.c_int32), nat._p(t.feature, C.c_int32), nat._p(t.threshold, C.c_float),
        nat._p(t.left, C.c_int32), nat._p(t.right, C.c_int32), nat._p(t.leaf_value, C.c_double),
        nat._p(t.tree_slot, C.c_int32), nat._p(t.tree_scale, C.c_double), nat._p(t.init, C.c_double), t.n_scores, t.link,
        None, 0, t.cmp_mode, nat._p(t.default_left, C.c_uint8), nat.NAN_DEFAULT_CHILD,
        nat._p(node_cat, C.c_int32), nat._p(offs, C.c_int32), len(offs) - 1 if n_sets is None else n_sets,
        nat._p(words, C.c_uint32), len(words) if n_words is None else n_words, t.cat_mode if cat_mode is None else cat_mode)


def _lib_or_skip():
    try:
        return nat.load()
    except Exception as e:  # the library is built by build(); plan building itself needs no device
        pytest.skip(f"libb200serve.so not built: {e}")


def test_c_abi_rejects_malformed_categorical_input():
    lib = _lib_or_skip()
    packed = tree_formats.pack_xgboost_json(_xgb_one_cat_node([1, 40]))  # one set of two words
    leaf_cat = packed.node_cat.copy()
    leaf_cat[1] = 0
    bad = {
        "set index out of range": dict(node_cat=[1, -1, -1]),
        "set index below -1": dict(node_cat=[-2, -1, -1]),
        "offsets not monotone": dict(cat_offsets=[0, 2, 1], n_sets=2, node_cat=[0, -1, -1]),
        "offsets past cat_words": dict(cat_offsets=[0, 3]),
        "negative first offset": dict(cat_offsets=[-1, 2]),
        "categorical leaf": dict(node_cat=leaf_cat),
        "unknown cat_mode": dict(cat_mode=7),
    }
    for what, kw in bad.items():
        h = C.c_void_p()
        nat.check(lib.b2s_plan_create(2, C.byref(h)))
        try:
            assert _cat_call(lib, h, packed, **kw) == -1, what  # B2S_ERR_INVALID
            assert lib.b2s_last_error(), what
        finally:
            lib.b2s_plan_destroy(h)
    h = C.c_void_p()
    nat.check(lib.b2s_plan_create(2, C.byref(h)))
    try:
        assert _cat_call(lib, h, packed) == 0, lib.b2s_last_error()
    finally:
        lib.b2s_plan_destroy(h)
