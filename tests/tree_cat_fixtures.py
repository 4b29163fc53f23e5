"""Categorical splits of xgboost and LightGBM (tests only; neither library is in the image).

`xgboost_margins` / `lightgbm_raw` restate the libraries' published decision functions over their own serialised models,
one row at a time, in plain Python -- the oracle of the categorical tests.  Parity with the libraries themselves is
unpinned (DESIGN.md section 2):

  xgboost  common::Decision (src/common/categorical.h), used from GetNextNode (src/predictor/predict_fn.h):  NaN -> the
           node's default child; x < 0 or too large for int32 -> left; otherwise the category trunc(x) goes right when it is
           listed in the node's `categories` and left when it is not.  Numeric nodes: left when x < split_condition.
  LightGBM 4.x Tree::CategoricalDecision (include/LightGBM/tree.h):  NaN -> right (whatever missing_type and default_left
           say); trunc(x) < 0 (or too large for int32) -> right; a category listed in the node's threshold "a||b||c" goes
           left, any other right.  Numeric nodes: Tree::NumericalDecision as in oracle/tree_libs.py.

`packed_predict` is the float64 walk of the canonical PackedTrees (include/b200serve.h, b2s_plan_add_tree_model_cat), and
`random_xgb_cat_model` / `random_lgbm_cat_dump` write seeded documents mixing numeric and categorical nodes.
"""

import json
import math

import numpy as np

from mlrun_b200 import _native as nat
from tests.device_emulator import device_thresholds

INT32_LIMIT = 2.0 ** 31


def _doc(d):
    return json.loads(d) if isinstance(d, (str, bytes, bytearray)) else d


# ------------------------------------------------------------------------------------------ oracle: xgboost
def _xgb_cats(tree):
    cats = {}
    for j, nid in enumerate(tree.get("categories_nodes", [])):
        seg, size = tree["categories_segments"][j], tree["categories_sizes"][j]
        cats[int(nid)] = {int(c) for c in tree["categories"][seg:seg + size]}
    return cats


def xgboost_margins(model_json, X):
    """(B, n_groups) float64 margins of a `save_model` JSON document with numeric and categorical nodes"""
    doc = _doc(model_json)
    learner = doc["learner"]
    booster = learner["gradient_booster"]
    model = booster["gbtree"]["model"] if "gbtree" in booster else booster["model"]
    lmp = learner["learner_model_param"]
    groups = max(int(lmp.get("num_class", "0") or 0), 1)
    base_score = float(lmp.get("base_score", "0.5"))
    objective = learner["objective"]["name"]
    base_margin = math.log(base_score / (1.0 - base_score)) if objective == "binary:logistic" else base_score
    tree_info = model.get("tree_info") or [0] * len(model["trees"])
    X = np.asarray(X, dtype=np.float32)
    cats = [_xgb_cats(t) for t in model["trees"]]
    out = np.zeros((len(X), groups), dtype=np.float64)
    for r, row in enumerate(X):
        psum = [0.0] * groups
        for ti, tree in enumerate(model["trees"]):
            left, right = tree["left_children"], tree["right_children"]
            cond, feat, dleft = tree["split_conditions"], tree["split_indices"], tree["default_left"]
            split_type = tree.get("split_type") or [0] * len(left)
            nid = 0
            while left[nid] != -1:
                fvalue = float(row[feat[nid]])
                if math.isnan(fvalue):
                    nid = left[nid] if dleft[nid] else right[nid]
                elif split_type[nid] == 1:
                    go_left = fvalue < 0 or fvalue >= INT32_LIMIT or int(fvalue) not in cats[ti].get(nid, ())
                    nid = left[nid] if go_left else right[nid]
                else:
                    nid = left[nid] if np.float32(fvalue) < np.float32(cond[nid]) else right[nid]
            g = tree_info[ti] if groups > 1 else 0
            psum[g] += float(np.float32(cond[nid]))
        for g in range(groups):
            out[r, g] = float(np.float32(base_margin)) + psum[g]
    return out, objective


def xgboost_predict(model_json, X):
    margins, objective = xgboost_margins(model_json, X)
    if objective.startswith("multi:"):
        return np.argmax(margins, axis=1)
    if objective.startswith("binary:"):
        return (margins[:, 0] > 0).astype(int)
    return margins[:, 0]


# ------------------------------------------------------------------------------------------ oracle: LightGBM
def lightgbm_raw(dump, X):
    doc = _doc(dump)
    num_class = int(doc.get("num_class", 1))
    per_iter = int(doc.get("num_tree_per_iteration", num_class))
    X = np.asarray(X, dtype=np.float32)
    out = np.zeros((len(X), max(per_iter, 1)), dtype=np.float64)
    for r, row in enumerate(X):
        for ti, info in enumerate(doc["tree_info"]):
            node = info["tree_structure"]
            while "split_feature" in node:
                fval = float(row[node["split_feature"]])
                if node.get("decision_type", "<=") == "==":
                    if math.isnan(fval) or fval >= INT32_LIMIT or int(fval) < 0:  # int(): toward zero, as static_cast<int>
                        go_left = False
                    else:
                        go_left = int(fval) in {int(c) for c in str(node["threshold"]).split("||") if c != ""}
                else:
                    missing = node.get("missing_type", "None")
                    if math.isnan(fval) and missing != "NaN":
                        fval = 0.0
                    if missing == "NaN" and math.isnan(fval):
                        go_left = bool(node.get("default_left", False))
                    else:
                        go_left = fval <= float(node["threshold"])
                node = node["left_child"] if go_left else node["right_child"]
            out[r, ti % per_iter if per_iter > 1 else 0] += float(node.get("leaf_value", 0.0))
    return out, str(doc.get("objective", "regression")).split(" ")[0]


def lightgbm_predict(dump, X):
    raw, objective = lightgbm_raw(dump, X)
    if objective.startswith("multiclass"):
        return np.argmax(raw, axis=1)
    if objective in ("binary", "cross_entropy"):
        return (raw[:, 0] > 0).astype(int)
    return raw[:, 0]


# ------------------------------------------------------------------------------------------ the packed (canonical) form
def packed_walk(t, X):
    """float64 walk of a PackedTrees over float32 rows: numeric nodes as the device stores them, categorical nodes by the
    canonical rule (right iff x is a valid code whose bit is set; NaN -> default_left).  -> scores (B, K), S = |init| +
    sum of |leaf| along the paths (B, K), terms per score (K,)"""
    X = np.asarray(X, dtype=np.float32)
    B = X.shape[0]
    thr = device_thresholds(t)
    dleft = t.default_left if t.nan_ok else None
    node_cat = t.node_cat if t.node_cat is not None else np.full(t.n_nodes, -1, dtype=np.int32)
    offs = t.cat_offsets if t.cat_offsets is not None else np.zeros(1, dtype=np.int32)
    words = np.concatenate([t.cat_words, [0]]).astype(np.int64) if t.cat_words is not None else np.zeros(1, dtype=np.int64)
    sc = np.tile(np.asarray(t.init, dtype=np.float64), (B, 1))
    S = np.tile(np.abs(t.init), (B, 1))
    rows = np.arange(B)
    with np.errstate(invalid="ignore"):
        for ti in range(t.n_trees):
            base = int(t.tree_offset[ti])
            node = np.zeros(B, dtype=np.int64)
            active = t.feature[base + node] >= 0
            while active.any():
                i = base + node
                f = t.feature[i]
                x = X[rows, np.where(f >= 0, f, 0)].astype(np.float64)
                s = node_cat[i]
                cat = s >= 0
                sidx = np.where(cat, s, 0)
                nbits = 32.0 * (offs[np.minimum(sidx + 1, len(offs) - 1)] - offs[sidx])
                valid = (x >= 0) if t.cat_mode == nat.CAT_NONNEG else (x > -1)
                in_range = cat & valid & (x < nbits)
                c = np.where(in_range, np.trunc(np.where(in_range, x, 0)), 0).astype(np.int64)
                w = words[np.where(in_range, offs[sidx] + (c >> 5), len(words) - 1)]
                right = np.where(cat, in_range & (((w >> (c & 31)) & 1) == 1), ~(x <= thr[i]))
                if dleft is not None:
                    right = np.where(np.isnan(x), dleft[i] == 0, right)
                node = np.where(active, np.where(right, t.right[i], t.left[i]), node)
                active = t.feature[base + node] >= 0
            v = t.tree_scale[ti] * t.leaf_value[base + node]
            k = t.tree_slot[ti]
            sc[:, k] += v
            S[:, k] += np.abs(v)
    return sc, S, np.bincount(t.tree_slot, minlength=t.n_scores) + 1


def packed_scores(t, X):
    return packed_walk(t, X)[0]


def packed_predict(t, X):
    sc = packed_scores(t, X)
    if t.link == nat.LINK_IDENTITY:
        return sc[:, 0]
    if t.link == nat.LINK_ARGMAX:
        idx = np.argmax(sc, axis=1)
    elif t.link == nat.LINK_BINARY_GE:
        idx = (sc[:, 0] >= 0).astype(int)
    else:
        idx = (sc[:, 0] > 0).astype(int)
    return t.classes[idx] if t.classes is not None else idx


# ------------------------------------------------------------------------------------------ seeded documents
# category edge values: NaN, invalid codes, -0.0 and (-1, 0) (code 0 only for LightGBM), truncation, word boundaries,
# a code past every set, values beyond int32
EDGE_VALUES = np.array([np.nan, -1.0, -0.5, -0.0, 0.0, 2.7, 31.0, 32.0, 33.0, 31.9, 63.0, 64.0, 999.0, 1000.0, 1023.0,
                        5000.0, 3e9, -3e9, 1.0, 3.0], dtype=np.float32)


def cat_inputs(n_rows, n_feat, cat_cards, seed, nan_frac=0.1):
    """rows whose categorical columns (cat_cards: {column: cardinality}) hold codes and edge values"""
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n_rows, n_feat)).astype(np.float32)
    for f, card in cat_cards.items():
        col = rng.integers(0, card + 8, size=n_rows).astype(np.float32)
        edge = rng.random(n_rows) < 0.25
        col[edge] = rng.choice(EDGE_VALUES, size=int(edge.sum()))
        X[:, f] = col
    X[rng.random((n_rows, n_feat)) < nan_frac] = np.nan
    return X


def _shape(rng, depth, p_leaf):
    nodes, frontier = [None], [(0, 0)]
    while frontier:
        nid, d = frontier.pop(0)
        if d >= depth or (d > 0 and rng.random() < p_leaf):
            continue
        li, ri = len(nodes), len(nodes) + 1
        nodes.extend([None, None])
        nodes[nid] = (li, ri)
        frontier.extend([(li, d + 1), (ri, d + 1)])
    return nodes


def _subset(rng, card):
    k = int(rng.integers(1, max(2, card // 2) + 1))
    return sorted(int(c) for c in rng.choice(card, size=min(k, card), replace=False))


def random_xgb_cat_model(n_trees=8, depth=4, n_feat=8, cat_cards=None, seed=0, objective="reg:squarederror", num_class=0,
                         base_score=0.5, p_leaf=0.2, p_cat=0.6):
    """a `save_model` document; nodes on the columns of cat_cards split on categories with probability p_cat"""
    rng = np.random.default_rng(seed)
    cat_cards = {0: 40, 1: 1001} if cat_cards is None else cat_cards
    trees, tree_info = [], []
    groups = max(num_class, 1)
    for t in range(n_trees * groups):
        shape = _shape(rng, depth, p_leaf)
        n = len(shape)
        left, right, cond, feat, dleft, stype = [-1] * n, [-1] * n, [0.0] * n, [0] * n, [0] * n, [0] * n
        cat_nodes, cats, segs, sizes = [], [], [], []
        for i, kids in enumerate(shape):
            if kids is None:
                cond[i] = float(np.float32(rng.normal() * 0.3))
                continue
            left[i], right[i] = kids
            dleft[i] = int(rng.random() < 0.5)
            if cat_cards and rng.random() < p_cat:
                f = int(rng.choice(list(cat_cards)))
                feat[i], stype[i] = f, 1
                codes = _subset(rng, cat_cards[f])
                cat_nodes.append(i), segs.append(len(cats)), sizes.append(len(codes))
                cats.extend(codes)
            else:
                feat[i] = int(rng.integers(0, n_feat))
                cond[i] = float(np.float32(rng.normal()))
        trees.append({"left_children": left, "right_children": right, "split_conditions": cond, "split_indices": feat,
                      "default_left": dleft, "split_type": stype, "categories": cats, "categories_nodes": cat_nodes,
                      "categories_segments": segs, "categories_sizes": sizes, "id": t,
                      "tree_param": {"num_nodes": str(n), "num_feature": str(n_feat)}})
        tree_info.append(t % groups)
    return {"learner": {"gradient_booster": {"name": "gbtree", "model": {
        "trees": trees, "tree_info": tree_info,
        "gbtree_model_param": {"num_trees": str(len(trees)), "num_parallel_tree": "1"}}},
        "learner_model_param": {"base_score": repr(float(base_score)), "num_class": str(num_class), "num_feature": str(n_feat)},
        "objective": {"name": objective}}, "version": [1, 7, 0]}


def random_lgbm_cat_dump(n_trees=8, depth=4, n_feat=8, cat_cards=None, seed=0, objective="regression", num_class=1,
                         p_leaf=0.2, p_cat=0.6):
    """a `dump_model()` document with decision_type "==" nodes on the columns of cat_cards"""
    rng = np.random.default_rng(seed)
    cat_cards = {0: 40, 1: 1001} if cat_cards is None else cat_cards
    infos = []
    for t in range(n_trees * max(num_class, 1)):
        shape = _shape(rng, depth, p_leaf)

        def build(i, shape=shape):
            if shape[i] is None:
                return {"leaf_index": i, "leaf_value": float(rng.normal() * 0.3)}
            node = {"split_index": i, "default_left": bool(rng.random() < 0.5),
                    "missing_type": str(rng.choice(["None", "NaN"]))}
            if cat_cards and rng.random() < p_cat:
                f = int(rng.choice(list(cat_cards)))
                node.update(split_feature=f, decision_type="==", threshold="||".join(str(c) for c in _subset(rng, cat_cards[f])))
            else:
                node.update(split_feature=int(rng.integers(0, n_feat)), decision_type="<=", threshold=float(rng.normal()))
            node.update(left_child=build(shape[i][0]), right_child=build(shape[i][1]))
            return node

        infos.append({"tree_index": t, "num_leaves": sum(1 for s in shape if s is None), "shrinkage": 0.1, "tree_structure": build(0)})
    return {"name": "tree", "version": "v4", "num_class": num_class, "num_tree_per_iteration": max(num_class, 1),
            "max_feature_idx": n_feat - 1, "objective": objective if num_class <= 1 else f"{objective} num_class:{num_class}",
            "average_output": False, "tree_info": infos}
