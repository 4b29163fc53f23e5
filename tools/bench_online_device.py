"""The online table two ways, alternated in one run: 16 Mi keys x 32 float32 features plus an int label, impute_policy
{"*": "$mean"}.

- build: a pandas frame -> FeatureVector -> get_online_feature_service (to_numpy, numpy statistics, the sequential host
  insert, the upload), against torch CUDA columns -> the same (statistics, keys, pack, insert, check and label keys on the
  device)
- enrich: GraphServer.run_enriched of 1 Mi keys on a 4-model linear EnrichmentVotingEnsemble over the device-built table,
  from host int64 keys (outputs on the host) against from the same keys in a CUDA tensor (outputs in HBM)

Each time is the host clock from the call to a torch.cuda.synchronize() after it.  Every iteration compares the two
paths' results bit for bit: the statistics table, the truthy-label keys and get_matrix of 1 Mi keys for the build, the
outputs and status words for the enrichment.  Prints one JSON line with the per-iteration times, the launches of one device
build (`b2s_launch_count`) and the card name and power limit, read in the same run.

    python tools/bench_online_device.py [--keys 16777216] [--features 32] [--batch 1048576] [--iters 3]
"""

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

from tools.bench_training_set import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=16 << 20)
    ap.add_argument("--features", type=int, default=32)
    ap.add_argument("--batch", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()

    import torch
    from sklearn.linear_model import LinearRegression

    from mlrun_b200 import _native as nat
    from mlrun_b200 import api
    from mlrun_b200.feature_store import online as bo

    nat.init(0)
    name, limit = card()
    n, F = args.keys, args.features
    rng = np.random.default_rng(0)
    feats = [f"f{j}" for j in range(F)]
    cols = {"id": rng.permutation(n).astype(np.int64) * 7 + 3}
    vals = rng.normal(size=(n, F)).astype(np.float32)
    vals[rng.random(size=(n, F)) < 0.02] = np.nan
    for j, f in enumerate(feats):
        cols[f] = np.ascontiguousarray(vals[:, j])
    del vals
    cols["label"] = rng.integers(0, 2, size=n).astype(np.int32)
    frame = pd.DataFrame(cols, copy=False).set_index("id")
    dev = {k: torch.from_numpy(v).cuda() for k, v in cols.items()}
    policy = {"*": "$mean"}
    ask = cols["id"][rng.integers(0, n, size=args.batch)]
    ask[::97] = -1  # not an entity
    d_ask = torch.from_numpy(ask).cuda()
    torch.cuda.synchronize()

    def build(source):
        t = time.perf_counter()
        svc = bo.FeatureVector("v", feats + ["label"], ["id"], source, label_column="label").get_online_feature_service(
            impute_policy=policy)
        torch.cuda.synchronize()
        return svc, time.perf_counter() - t

    def server_over(svc):
        api.register_feature_vector("store://bench", svc.vector)
        fn = api.new_function("enrich", kind="serving")
        graph = fn.set_topology("router", api.EnrichmentVotingEnsemble(feature_vector_uri="store://bench", impute_policy=policy,
                                                                       vote_type="regression", executor_type="array"))
        mrng = np.random.default_rng(1)
        for i in range(4):
            m = LinearRegression()
            m.coef_, m.intercept_, m.n_features_in_ = mrng.normal(size=F), 0.1 * i, F
            graph.add_route(f"m{i}", class_name="SKLearnModelServer", model=m, model_path="")
        return fn.to_mock_server(namespace={"SKLearnModelServer": api.SKLearnModelServer})

    build_host, build_dev, enr_host, enr_dev, equal = [], [], [], [], True
    launches = None
    server = None
    for it in range(args.iters + 1):  # iteration 0 warms both paths up and is not reported
        hs, th = build(frame)
        before = nat.launch_count()
        ds, td = build(dev)
        launches = nat.launch_count() - before
        X, found = hs.get_matrix(ask)
        rows, dfound = ds.get_matrix(d_ask)
        same = (hs.vector.get_stats_table().equals(ds.vector.get_stats_table())
                and np.array_equal(hs._label_alive, ds._label_alive)
                and np.array_equal(rows.numpy().view(np.uint32), X.view(np.uint32))
                and np.array_equal(dfound.numpy().astype(bool), found))
        del rows, dfound
        hs.close()
        if server is not None:
            server.graph._object._feature_service.close()
        server = server_over(ds)
        ds.close()
        t = time.perf_counter()
        out, st = server.run_enriched(ask, with_status=True)
        torch.cuda.synchronize()
        te_h = time.perf_counter() - t
        t = time.perf_counter()
        d_out, d_st = server.run_enriched(d_ask, with_status=True)
        torch.cuda.synchronize()
        te_d = time.perf_counter() - t
        same = same and np.array_equal(d_out.numpy().view(np.uint32), out.view(np.uint32)) and np.array_equal(d_st.numpy(), st)
        equal = equal and same
        if it:
            build_host.append(round(th, 4))
            build_dev.append(round(td, 4))
            enr_host.append(round(te_h, 5))
            enr_dev.append(round(te_d, 5))
    rec = {"bench": "online_device", "keys": n, "features": F, "batch": args.batch, "iters": args.iters,
           "build_host_s": build_host, "build_device_s": build_dev, "enrich_host_keys_s": enr_host, "enrich_cuda_keys_s": enr_dev,
           "build_speedup_best": round(min(build_host) / min(build_dev), 2),
           "enrich_speedup_best": round(min(enr_host) / min(enr_dev), 2),
           "device_build_launches": launches, "equal": equal, "gpu": name, "power_limit": limit}
    print(json.dumps(rec))
    out_dir = os.environ.get("BENCH_OUT")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_online_device.json"), "w") as f:
            f.write(json.dumps(rec) + "\n")
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
