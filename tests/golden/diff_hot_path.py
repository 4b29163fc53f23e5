"""The checker of the CUDA kernels -- oracle/batch.py, the vectorised float64 restatement -- against the REAL reference running
the hot path one event at a time (build container only): seeded random metric-shaped workloads (Imputer -> OneHotEncoder ->
1..6 linear models -> mean vote; 4..24 numeric and 0..6 categorical columns, different seeds, NaN and out-of-vocabulary
rates) through the reference's sync flow, one MockEvent per row; and tree-ensemble routers (regression: mean vote,
classification: majority vote; 2..5 models) with one event carrying the batch.  rtol 1e-12 for regression (the per-event path
adds the same float64 terms in a different association), exact for labels.

    python -m tests.golden.diff_hot_path             # live, needs the reference sources importable (tests/golden/_refshim.py)
    python -m tests.golden.diff_hot_path --record    # live, and store the reference's outputs in ref_hot_path.json.xz
    python -m tests.golden.diff_hot_path --golden    # against the stored outputs: runs anywhere
"""
import json
import lzma
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402

from mlrun_b200.synthetic import flow3_workload, tree_workload  # noqa: E402
from oracle import batch as obatch  # noqa: E402


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_hot_path.json.xz")


def cases():
    """the 64 seeded workloads, in order: (kind, case, workload, request path or model kind)"""
    rnd = random.Random(31)
    for case in range(40):
        n_models = rnd.choice([1, 1, 2, 4, 6])
        wl = flow3_workload(n_rows=rnd.randint(20, 60), n_num=rnd.randint(4, 24), n_cat=rnd.randint(0, 6), seed=100 + case, n_models=n_models)
        yield "flow3", case, wl, "/" if n_models == 1 else "/v2/models/infer"
    for case in range(24):
        kind = rnd.choice(["regression", "classification"])
        wl = tree_workload(n_rows=rnd.randint(16, 80), n_feat=rnd.randint(4, 24), n_models=rnd.randint(2, 5), n_trees=rnd.randint(3, 12),
                           depth=rnd.randint(2, 5), seed=200 + case, kind=kind, n_fit=400)
        yield "trees", case, wl, kind


def reference_outputs():
    """what the real reference returns for every case (one MockEvent per row for the flows, one batch event for the trees)"""
    from tests.golden import api_reference as ref

    outs = []
    for what, _case, wl, arg in cases():
        if what == "flow3":
            server = wl.build_server(ref, engine="sync")
            got = []
            for row in wl.rows_as_dicts():
                out = server.test(path=arg, body=row)["outputs"]
                got.append(out[0] if isinstance(out, list) else out)
            outs.append([float(v) for v in got])
        else:
            out = wl.build_server(ref).test("/v2/models/infer", body={"inputs": wl.X.astype(np.float64).tolist()})["outputs"]
            outs.append([float(v) for v in out] if arg == "regression" else [v.item() if hasattr(v, "item") else v for v in out])
    return outs


def check(want_all):
    n_events = 0
    for (what, case, wl, arg), got in zip(cases(), want_all, strict=True):
        if what == "flow3":
            want = obatch.flow3(wl)["out"]
            np.testing.assert_allclose(np.asarray(got, dtype=np.float64), want, rtol=1e-12, atol=1e-12, err_msg=f"flow3 case {case}")
        else:
            want = obatch.tree_ensemble(wl)["out"]
            if arg == "regression":
                np.testing.assert_allclose(np.asarray(got, dtype=np.float64), want, rtol=1e-12, atol=1e-12, err_msg=f"trees case {case}")
            else:
                assert list(got) == want.tolist(), f"trees case {case}: labels differ"
        n_events += len(got)
    return n_events


def main():
    if "--golden" in sys.argv:  # the reference's outputs as recorded by --record: no reference tree needed
        with lzma.open(GOLDEN, "rt") as f:
            n_events = check(json.load(f))
        print("the batched oracle equals the real reference's per-event path (recorded outputs) on", n_events, "events of 64 random workloads")
        return 0
    want = reference_outputs()
    if "--record" in sys.argv:
        with lzma.open(GOLDEN, "wt") as f:
            json.dump(want, f)
    n_events = check(want)
    print("the batched oracle equals the real reference's per-event path on", n_events, "events of 64 random workloads")
    return 0


if __name__ == "__main__":
    sys.exit(main())
