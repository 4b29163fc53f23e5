"""xgboost / LightGBM tree ensembles -> PackedTrees (the device format of mlrun_b200.plan).

The reference serves these libraries through the same predict call as scikit-learn:
`XGBoostModelServer = PickleModelServer` (mlrun/frameworks/xgboost/__init__.py:30 -> `self.model.predict(x)`,
frameworks/_ml_common/pkl_model_server.py:52-60) and `LGBMModelServer.predict` (frameworks/lgbm/model_server.py:142-159).
Neither library is installed in the build image, so the exporters read the libraries' own *serialised* models -- the
JSON a user gets from `Booster.save_model("m.json")` / `Booster.get_dump(dump_format="json")` / `Booster.dump_model()` --
and restate the published walk (parity with the libraries themselves is unpinned, DESIGN.md section 2):

  xgboost   (src/tree/tree_model.h RegTree::GetNext / predict_fn.h):  go to the "yes" (left) child when x < split_condition,
            a missing value (NaN) goes to the node's default ("missing") child; margins are base_margin + sum of leaves;
            reg:squarederror -> margin; binary:logistic -> margin > 0; multi:softmax/softprob -> argmax over class margins
            (trees round-robin over classes, `tree_info`).
  LightGBM  (include/LightGBM/tree.h Tree::NumericalDecision):  left when x <= threshold; missing_type "NaN": NaN takes
            `default_left`; missing_type "None": NaN is read as 0.0 (so it goes left iff 0 <= threshold); "Zero" splits
            are not lowered.  Leaf values already include the shrinkage.

`x < t` becomes `x <= prev_float32(t)` inside b2s_plan_add_tree_model_ex (cmp_mode B2S_CMP_LT); LightGBM's float64
thresholds are rounded toward -inf to float32 exactly like scikit-learn's (packing.threshold_to_f32).

Categorical splits.  xgboost (`save_model` JSON: split_type 1, the node's categories in `categories` at
`categories_segments` / `categories_sizes` of its entry in `categories_nodes`; common::Decision in
src/common/categorical.h, used from GetNextNode in src/predictor/predict_fn.h) and LightGBM 4.x (`dump_model()`:
decision_type "==", threshold "0||3||17"; Tree::CategoricalDecision in include/LightGBM/tree.h) decide as follows:

                    xgboost                                 LightGBM 4.x
  NaN               the node's default child                always LightGBM's right child
  category of x     trunc(x)                                trunc(x) (x in (-1, 0) is category 0)
  invalid code      x < 0 -> left                           trunc(x) < 0 -> right
  in the node's set -> right                                -> left
  otherwise         -> left (also past the end of the set)  -> right

A value too large for int32 counts as outside the set (undefined behaviour in LightGBM).  LightGBM <= 3 read NaN as
category 0 under missing_type None; that rule is not reproduced.  The exporters normalise both into one device form:
*a categorical node sends x right iff x is a valid code whose bit is set*.  LightGBM nodes get their children swapped and
their NaN default set to the side of LightGBM's right child.  The one per-library difference left is the model's
`cat_mode`: a valid code is x >= 0 (nat.CAT_NONNEG, xgboost) or x > -1 (nat.CAT_TRUNC, LightGBM).  Sets are bitsets of
32-bit words: code c is bit c % 32 of word c // 32 of the node's set (PackedTrees.node_cat / cat_offsets / cat_words).
`get_dump` documents do not carry the sets and keep being refused.
"""

import json
import math

import numpy as np

from . import _native as nat
from .packing import UnsupportedModel, threshold_to_f32
from .plan import PackedTrees


def _cat_bitset(codes):
    """category codes -> the canonical set: 32-bit words, code c is bit c % 32 of word c // 32"""
    codes = [int(c) for c in codes]
    if any(c < 0 for c in codes):
        raise UnsupportedModel(f"negative category code in a categorical split: {min(codes)}")
    words = np.zeros(max(codes) // 32 + 1 if codes else 0, dtype=np.uint32)
    for c in codes:
        words[c >> 5] |= np.uint32(1 << (c & 31))
    return words


class _Acc:
    def __init__(self):
        self.feature, self.threshold, self.left, self.right, self.leaf, self.default_left = [], [], [], [], [], []
        self.offset, self.slot, self.scale = [0], [], []
        self.node_cat, self.sets = [], []  # per node -1 or an index into sets (canonical bitsets)

    def add_set(self, codes):
        self.sets.append(_cat_bitset(codes))
        return len(self.sets) - 1

    def add_tree(self, feature, threshold, left, right, leaf, default_left, slot, scale=1.0, node_cat=None):
        self.feature.append(np.asarray(feature, dtype=np.int32))
        self.threshold.append(np.asarray(threshold, dtype=np.float32))
        self.left.append(np.asarray(left, dtype=np.int32))
        self.right.append(np.asarray(right, dtype=np.int32))
        self.leaf.append(np.asarray(leaf, dtype=np.float64))
        self.default_left.append(np.asarray(default_left, dtype=np.uint8))
        self.node_cat.append(np.full(len(feature), -1, dtype=np.int32) if node_cat is None else np.asarray(node_cat, dtype=np.int32))
        self.offset.append(self.offset[-1] + len(feature))
        self.slot.append(int(slot))
        self.scale.append(float(scale))

    def finish(self, init, link, classes, cmp_mode, n_features=None, cat_mode=nat.CAT_NONNEG):
        cat = {}
        if self.sets:  # a model without a categorical node keeps node_cat None (b2s_plan_add_tree_model_ex, as before)
            cat = dict(node_cat=np.concatenate(self.node_cat),
                       cat_offsets=np.cumsum([0] + [len(w) for w in self.sets]).astype(np.int32),
                       cat_words=np.concatenate(self.sets).astype(np.uint32), cat_mode=cat_mode)
        packed = PackedTrees(
            tree_offset=np.asarray(self.offset, dtype=np.int32), feature=np.concatenate(self.feature),
            threshold=np.concatenate(self.threshold), left=np.concatenate(self.left), right=np.concatenate(self.right),
            leaf_value=np.concatenate(self.leaf), tree_slot=np.asarray(self.slot, dtype=np.int32),
            tree_scale=np.asarray(self.scale, dtype=np.float64), init=np.asarray(init, dtype=np.float64), link=link,
            classes=classes, cmp_mode=cmp_mode, default_left=np.concatenate(self.default_left), nan_ok=True, **cat)
        packed.n_features = n_features
        return packed


def _bfs_order(root, children_of):
    """nodes of a nested tree in an order where children follow their parent (what the C-ABI requires)"""
    order, queue = [], [root]
    while queue:
        node = queue.pop(0)
        order.append(node)
        queue.extend(children_of(node))
    return order


# ------------------------------------------------------------------------------------------ xgboost
_XGB_IDENTITY = {"reg:squarederror", "reg:linear", "reg:absoluteerror", "reg:pseudohubererror", "reg:quantileerror",
                 "reg:squaredlogerror"}


def _xgb_objective_head(objective, base_score, num_class):
    """-> (init margins, link, n_scores)"""
    if objective in _XGB_IDENTITY:
        return [base_score], nat.LINK_IDENTITY, 1
    if objective in ("binary:logistic", "binary:logitraw", "binary:hinge"):
        if objective == "binary:logistic":
            if not 0.0 < base_score < 1.0:
                raise UnsupportedModel(f"binary:logistic with base_score {base_score}")
            margin = math.log(base_score / (1.0 - base_score))
        else:
            margin = base_score
        return [margin], nat.LINK_BINARY_GT, 1  # XGBClassifier.predict: proba > 0.5  <=>  margin > 0
    if objective in ("multi:softmax", "multi:softprob"):
        if num_class < 2:
            raise UnsupportedModel("multi-class objective without num_class")
        return [base_score] * num_class, nat.LINK_ARGMAX, num_class
    raise UnsupportedModel(f"xgboost objective {objective!r} is not lowered (identity, binary and softmax heads are)")


def pack_xgboost_json(model_json, classes=None):
    """the model as written by `Booster.save_model("model.json")` / `save_raw("json")` (str, bytes or parsed dict)"""
    doc = json.loads(model_json) if isinstance(model_json, (str, bytes, bytearray)) else model_json
    learner = doc["learner"]
    booster = learner["gradient_booster"]
    if booster.get("name", "gbtree") not in ("gbtree", "dart"):
        raise UnsupportedModel(f"xgboost booster {booster.get('name')!r} is not a tree ensemble")
    weight_drop = booster.get("weight_drop")  # dart: per-tree output scale
    model = booster["gbtree"]["model"] if "gbtree" in booster else booster["model"]
    lmp = learner["learner_model_param"]
    num_class = int(lmp.get("num_class", "0") or 0)
    base_score = float(lmp.get("base_score", "0.5"))
    n_features = int(lmp.get("num_feature", "0") or 0) or None
    objective = learner["objective"]["name"]
    init, link, n_scores = _xgb_objective_head(objective, base_score, num_class)
    if int(model.get("gbtree_model_param", {}).get("num_parallel_tree", "1") or 1) > 1:
        pass  # a boosted random forest is still a sum of trees
    acc = _Acc()
    tree_info = model.get("tree_info") or [0] * len(model["trees"])
    for ti, tree in enumerate(model["trees"]):
        left = np.asarray(tree["left_children"], dtype=np.int64)
        right = np.asarray(tree["right_children"], dtype=np.int64)
        cond = np.asarray(tree["split_conditions"], dtype=np.float64)
        feat = np.asarray(tree["split_indices"], dtype=np.int64)
        dleft = np.asarray(tree["default_left"], dtype=np.int64)
        split_type = tree.get("split_type") or [0] * len(left)
        # categorical nodes: the categories that go right (common::Decision returns "left" when the bit is not set) --
        # already the canonical direction, so children and default child are kept
        cat_codes = {}
        for j, nid in enumerate(tree.get("categories_nodes", [])):
            seg, size = int(tree["categories_segments"][j]), int(tree["categories_sizes"][j])
            cat_codes[int(nid)] = tree["categories"][seg:seg + size]
        # re-number so that children follow their parent (xgboost's ids do after pruning too, but the ABI demands it)
        order = _bfs_order(0, lambda i: [] if left[i] < 0 else [int(left[i]), int(right[i])])
        new_id = {old: new for new, old in enumerate(order)}
        is_leaf = np.array([left[i] < 0 for i in order])
        node_cat = []
        for i, lf in zip(order, is_leaf):
            if lf or int(split_type[i]) == 0:
                node_cat.append(-1)
            elif int(split_type[i]) == 1:
                node_cat.append(acc.add_set(cat_codes.get(i, [])))
            else:
                raise UnsupportedModel(f"xgboost split_type {split_type[i]} is not lowered")
        acc.add_tree(
            feature=[-1 if lf else int(feat[i]) for i, lf in zip(order, is_leaf)],
            threshold=[0.0 if lf else cond[i] for i, lf in zip(order, is_leaf)],
            left=[0 if lf else new_id[int(left[i])] for i, lf in zip(order, is_leaf)],
            right=[0 if lf else new_id[int(right[i])] for i, lf in zip(order, is_leaf)],
            leaf=[cond[i] if lf else 0.0 for i, lf in zip(order, is_leaf)],  # a leaf keeps its value in split_conditions
            default_left=[0 if lf else int(dleft[i] != 0) for i, lf in zip(order, is_leaf)],
            slot=int(tree_info[ti]) if n_scores > 1 else 0,
            scale=float(weight_drop[ti]) if weight_drop else 1.0, node_cat=node_cat)
    cls = None
    if link != nat.LINK_IDENTITY:
        cls = np.arange(2 if n_scores == 1 else n_scores, dtype=np.int32) if classes is None else np.asarray(classes, dtype=np.int32)
    return acc.finish(init, link, cls, nat.CMP_LT, n_features, nat.CAT_NONNEG)


def pack_xgboost_dump(trees, objective="reg:squarederror", base_score=0.5, num_class=0, classes=None, n_features=None):
    """`Booster.get_dump(dump_format="json")`: a list with one nested {"nodeid", "split": "f3", "split_condition",
    "yes", "no", "missing", "children"} / {"nodeid", "leaf"} document per tree (strings or parsed dicts)"""
    init, link, n_scores = _xgb_objective_head(objective, float(base_score), int(num_class))
    acc = _Acc()
    for ti, tree in enumerate(trees):
        root = json.loads(tree) if isinstance(tree, (str, bytes, bytearray)) else tree
        order = _bfs_order(root, lambda n: n.get("children", []))
        new_id = {n["nodeid"]: i for i, n in enumerate(order)}
        feat, thr, left, right, leaf, dleft = [], [], [], [], [], []
        for n in order:
            if "leaf" in n:
                feat.append(-1), thr.append(0.0), left.append(0), right.append(0), leaf.append(float(n["leaf"])), dleft.append(0)
                continue
            if isinstance(n.get("split_condition"), list) or "categories" in n:  # xgboost dumps a category set as a list
                raise UnsupportedModel("categorical splits are not lowered from get_dump documents: they do not carry the "
                                       "category sets; export the model with Booster.save_model(\"model.json\") instead")
            name = str(n["split"])
            if not (name.startswith("f") and name[1:].isdigit()):
                raise UnsupportedModel(f"feature {name!r}: dump the model without a feature map (names f0, f1, ...)")
            feat.append(int(name[1:])), thr.append(float(n["split_condition"]))
            left.append(new_id[n["yes"]]), right.append(new_id[n["no"]]), leaf.append(0.0)
            dleft.append(1 if n.get("missing", n["yes"]) == n["yes"] else 0)
        acc.add_tree(feat, thr, left, right, leaf, dleft, slot=(ti % n_scores) if n_scores > 1 else 0)
    cls = None
    if link != nat.LINK_IDENTITY:
        cls = np.arange(2 if n_scores == 1 else n_scores, dtype=np.int32) if classes is None else np.asarray(classes, dtype=np.int32)
    return acc.finish(init, link, cls, nat.CMP_LT, n_features)


# ------------------------------------------------------------------------------------------ LightGBM
def pack_lightgbm_dump(dump, classes=None):
    """`Booster.dump_model()` (dict or its JSON text)"""
    doc = json.loads(dump) if isinstance(dump, (str, bytes, bytearray)) else dump
    objective = str(doc.get("objective", "regression")).split(" ")[0]
    num_class = int(doc.get("num_class", 1))
    per_iter = int(doc.get("num_tree_per_iteration", num_class))
    if objective in ("binary", "cross_entropy"):
        init, link, n_scores = [0.0], nat.LINK_BINARY_GT, 1
    elif objective in ("multiclass", "multiclassova"):
        init, link, n_scores = [0.0] * num_class, nat.LINK_ARGMAX, num_class
    elif objective in ("regression", "regression_l1", "huber", "fair", "quantile", "mape"):
        init, link, n_scores = [0.0], nat.LINK_IDENTITY, 1
    else:
        raise UnsupportedModel(f"LightGBM objective {objective!r} is not lowered")
    if doc.get("average_output"):
        raise UnsupportedModel("random-forest mode (average_output) is not lowered")
    acc = _Acc()
    for ti, info in enumerate(doc["tree_info"]):
        root = info["tree_structure"]
        order = _bfs_order(root, lambda n: [] if "leaf_value" in n or "split_feature" not in n else [n["left_child"], n["right_child"]])
        ids = {id(n): i for i, n in enumerate(order)}
        feat, thr, left, right, leaf, dleft, node_cat = [], [], [], [], [], [], []
        for n in order:
            if "split_feature" not in n:
                feat.append(-1), thr.append(0.0), left.append(0), right.append(0), leaf.append(float(n.get("leaf_value", 0.0))), dleft.append(0)
                node_cat.append(-1)
                continue
            decision = n.get("decision_type", "<=")
            if decision == "==":
                # Tree::CategoricalDecision: the listed categories go left, everything else (NaN, negative codes, codes not
                # listed) right.  Canonical form: the set sends right, so the children swap, and NaN takes the canonical left
                thr_text = n["threshold"]
                parts = thr_text.split("||") if isinstance(thr_text, str) else []
                if not parts or not all(c.isdigit() for c in parts):
                    raise UnsupportedModel(f"categorical split with threshold {thr_text!r}: expected category codes 'a||b||c'")
                codes = [int(c) for c in parts]
                feat.append(int(n["split_feature"])), thr.append(0.0)
                left.append(ids[id(n["right_child"])]), right.append(ids[id(n["left_child"])]), leaf.append(0.0), dleft.append(1)
                node_cat.append(acc.add_set(codes))
                continue
            if decision != "<=":
                raise UnsupportedModel(f"LightGBM decision_type {decision!r} is not lowered")
            node_cat.append(-1)
            missing = n.get("missing_type", "None")
            t64 = float(n["threshold"])
            if missing == "NaN":
                dl = bool(n.get("default_left", False))
            elif missing == "None":
                dl = 0.0 <= t64  # NaN is read as 0.0 (Tree::NumericalDecision)
            else:
                raise UnsupportedModel(f"missing_type {missing!r} (zero-as-missing) is not lowered")
            feat.append(int(n["split_feature"])), thr.append(float(threshold_to_f32([t64])[0]))
            left.append(ids[id(n["left_child"])]), right.append(ids[id(n["right_child"])]), leaf.append(0.0), dleft.append(int(dl))
        acc.add_tree(feat, thr, left, right, leaf, dleft, slot=(ti % per_iter) if n_scores > 1 else 0, node_cat=node_cat)
    cls = None
    if link != nat.LINK_IDENTITY:
        cls = np.arange(2 if n_scores == 1 else n_scores, dtype=np.int32) if classes is None else np.asarray(classes, dtype=np.int32)
    n_features = int(doc["max_feature_idx"]) + 1 if "max_feature_idx" in doc else None
    return acc.finish(init, link, cls, nat.CMP_LE, n_features, nat.CAT_TRUNC)


# ------------------------------------------------------------------------------------------ live objects
def pack_library_model(model):
    """a live xgboost / LightGBM object (what the reference's model servers unpickle): serialise it with the library's own
    writer and read that.  -> PackedTrees, or None when `model` is not from one of these libraries."""
    name = type(model).__name__
    module = type(model).__module__.split(".")[0]
    if module == "xgboost":
        booster = model.get_booster() if hasattr(model, "get_booster") else model
        classes = getattr(model, "classes_", None)
        return pack_xgboost_json(bytes(booster.save_raw(raw_format="json")), classes=classes)
    if module == "lightgbm":
        booster = model.booster_ if hasattr(model, "booster_") else model
        classes = getattr(model, "classes_", None)
        return pack_lightgbm_dump(booster.dump_model(), classes=classes)
    if name in ("XGBRegressor", "XGBClassifier", "LGBMRegressor", "LGBMClassifier"):
        raise UnsupportedModel(f"{name} from module {module!r}")
    return None


def pack_serialised(doc):
    """a parsed JSON document of either library -> PackedTrees"""
    if isinstance(doc, dict) and "learner" in doc:
        return pack_xgboost_json(doc)
    if isinstance(doc, dict) and "tree_info" in doc:
        return pack_lightgbm_dump(doc)
    raise UnsupportedModel("not an xgboost save_model JSON nor a LightGBM dump_model document")
