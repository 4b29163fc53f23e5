"""Fit the tree ensembles of BASELINE configs[2] (SURVEY.md 8(d) config 3) ONCE and commit them as fixtures.

    python -m tests.golden.gen_trees_cfg3          # ~6 min on 8 cores; writes tests/golden/trees_cfg3_{reg,cls}.pkl.xz
                                                   # and trees_cfg4_reg.pkl.xz (the 64-feature tree scorers of configs[3])

4 x GradientBoostingRegressor(n_estimators=100, max_depth=6, random_state=30+i) and 4 x GradientBoostingClassifier (3
classes: terciles of y) fit on 20 000 synthetic rows of 128 float32 features, all features considered at every split,
y = 2*x0 + sin(x1) + x2*x3 + eps.  Fitting takes ~1.2 s per tree, far too long for a test or a bench run, so the fitted
scikit-learn estimators are stored (cloudpickle + xz; per-node training statistics and split-node values that predict() never
reads are zeroed so that each file compresses to less than 1 MB).  The oracle at test time is still scikit-learn's own predict() on these very objects.
"""

import lzma
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
N_FIT, N_FEAT, N_TREES, DEPTH, N_MODELS = 20000, 128, 100, 6, 4
N_FEAT_CFG4 = 64  # BASELINE configs[3] (SURVEY 8(d) config 4): "8 linear+tree models (as cfg 2/3, depth 6, 100 trees, 64 feat)"


def fit_data(n_feat=N_FEAT):
    frng = np.random.default_rng(103 if n_feat == N_FEAT else 104)
    Xf = frng.normal(size=(N_FIT, n_feat)).astype(np.float32)
    y = 2 * Xf[:, 0] + np.sin(Xf[:, 1]) + Xf[:, 2] * Xf[:, 3] + 0.1 * frng.normal(size=N_FIT)
    return Xf, y


def _slim(tree):
    """zero the training statistics of a fitted sklearn Tree and the values of its split nodes (predict / apply read the
    values of leaves only)"""
    state = tree.__getstate__()
    nodes = state["nodes"].copy()
    for field in ("impurity", "n_node_samples", "weighted_n_node_samples"):
        nodes[field] = 0
    state["nodes"] = nodes
    values = state["values"].copy()
    values[nodes["left_child"] != -1] = 0
    state["values"] = values
    tree.__setstate__(state)


def fit_one(kind, i):
    from sklearn.ensemble import GradientBoostingClassifier, GradientBoostingRegressor

    Xf, y = fit_data(N_FEAT_CFG4 if kind == "cfg4" else N_FEAT)
    if kind in ("reg", "cfg4"):
        m = GradientBoostingRegressor(n_estimators=N_TREES, max_depth=DEPTH, random_state=30 + i, subsample=0.8).fit(Xf, y)
    else:
        labels = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3]))
        m = GradientBoostingClassifier(n_estimators=N_TREES, max_depth=DEPTH, random_state=30 + i, subsample=0.8).fit(Xf, labels)
    for est in m.estimators_.ravel():
        _slim(est.tree_)
    m.train_score_ = np.zeros(0)
    if hasattr(m, "oob_improvement_"):
        m.oob_improvement_ = np.zeros(0)
        m.oob_scores_ = np.zeros(0)
    return m


def main():
    import cloudpickle
    from joblib import Parallel, delayed

    t0 = time.time()
    only = sys.argv[1:]  # e.g. `python -m tests.golden.gen_trees_cfg3 cfg4` regenerates one set
    jobs = [(k, i) for k in ("reg", "cls", "cfg4") if not only or k in only for i in range(N_MODELS)]
    models = Parallel(n_jobs=min(8, os.cpu_count() or 1))(delayed(fit_one)(k, i) for k, i in jobs)
    for kind in ("reg", "cls", "cfg4"):
        mine = [m for (k, _i), m in zip(jobs, models) if k == kind]
        if not mine:
            continue
        path = os.path.join(HERE, f"trees_cfg3_{kind}.pkl.xz" if kind != "cfg4" else "trees_cfg4_reg.pkl.xz")
        with lzma.open(path, "wb", preset=9) as fp:
            cloudpickle.dump(mine, fp)
        print(path, os.path.getsize(path), "bytes")
    print("fit wall %.0fs" % (time.time() - t0), file=sys.stderr)


if __name__ == "__main__":
    main()
