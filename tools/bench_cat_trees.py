"""Cost of categorical splits on the trees3 walk: a seeded LightGBM-shaped ensemble with categorical splits against the
same tree shapes with numeric splits only, in one process, alternating, timed with CUDA events.

Workload: 4 models x 100 trees of depth 6 over 128 features, 16 of them categorical (cardinality 8 to 1000); 256 Ki rows.
The numeric twin replaces every categorical node by a `<=` split on the same column, so both plans walk trees of the same
shape.  Prints one JSON line with the card's name and power limit (read in the same run).

    python tools/bench_cat_trees.py [--rows 262144] [--reps 5] [--iters 50]
"""

import argparse
import copy
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import tree_formats  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from tests import tree_cat_fixtures as fx  # noqa: E402

N_FEAT, N_MODELS, N_TREES, DEPTH = 128, 4, 100, 6


def cards(seed):
    rng = np.random.default_rng(seed)
    cols = rng.choice(N_FEAT, size=16, replace=False)
    return {int(c): int(k) for c, k in zip(cols, np.geomspace(8, 1000, 16).round())}


def numeric_twin(doc):
    """the same trees with every categorical node turned into `x <= card / 2` on its column"""
    doc = copy.deepcopy(doc)

    def walk(n):
        if "split_feature" not in n:
            return
        if n.get("decision_type") == "==":
            codes = [int(c) for c in n["threshold"].split("||")]
            n["decision_type"], n["threshold"], n["missing_type"] = "<=", float(np.median(codes)) + 0.5, "NaN"
        walk(n["left_child"])
        walk(n["right_child"])

    for info in doc["tree_info"]:
        walk(info["tree_structure"])
    return doc


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    nat.init(0)
    cc = cards(1)
    docs = [fx.random_lgbm_cat_dump(n_trees=N_TREES, depth=DEPTH, n_feat=N_FEAT, cat_cards=cc, seed=10 + i, p_leaf=0.0, p_cat=16 / N_FEAT * 4)
            for i in range(N_MODELS)]
    plans = {}
    for kind, ds in (("categorical", docs), ("numeric", [numeric_twin(d) for d in docs])):
        models = [("trees", tree_formats.pack_lightgbm_dump(d)) for d in ds]
        plans[kind] = ColumnProgram([f"f{i}" for i in range(N_FEAT)]).build_plan(
            models, vote=(nat.VOTE_MEAN, [1.0 / N_MODELS] * N_MODELS))
    cat_nodes = sum(int((tree_formats.pack_lightgbm_dump(d).node_cat >= 0).sum()) for d in docs)
    all_nodes = sum(int((tree_formats.pack_lightgbm_dump(d).feature >= 0).sum()) for d in docs)
    X = fx.cat_inputs(args.rows, N_FEAT, cc, seed=3, nan_frac=0.01)
    bufs = [nat.DeviceBuffer(X.nbytes).upload(X) for _ in range(2)]
    outs = {k: nat.DeviceBuffer(args.rows * 4) for k in plans}
    for k, p in plans.items():
        p.time_device([b.ptr for b in bufs], args.rows, N_FEAT * 4, outs[k].ptr, 5)  # warm-up
    ms = {k: [] for k in plans}
    for _ in range(args.reps):
        for k, p in plans.items():
            ms[k].append(p.time_device([b.ptr for b in bufs], args.rows, N_FEAT * 4, outs[k].ptr, args.iters) / args.iters)
    res = {"gpu": gpu_info(), "rows": args.rows, "models": N_MODELS, "trees": N_TREES, "depth": DEPTH,
           "categorical_nodes_share": cat_nodes / all_nodes}
    for k, p in plans.items():
        res[k] = {"kernel": p.kernel, "ms": ms[k], "events_per_s": [args.rows / (t * 1e-3) for t in ms[k]]}
    assert "categorical" in plans["categorical"].kernel and "categorical" not in plans["numeric"].kernel
    # node visits per row: every tree is complete (p_leaf = 0), so each walk visits DEPTH nodes
    visits = N_MODELS * N_TREES * DEPTH
    cat_visits = visits * res["categorical_nodes_share"]
    d_ns = (np.median(ms["categorical"]) - np.median(ms["numeric"])) * 1e6 / args.rows
    res["extra_ns_per_row"] = d_ns
    res["extra_ns_per_categorical_visit"] = d_ns / cat_visits if cat_visits else None
    print(json.dumps(res))


if __name__ == "__main__":
    main()
