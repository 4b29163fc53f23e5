"""Scoring rows that are in HBM with `GraphServer.run_batch`, against the host path that copies them off the device first, on
tools/bench_device_chain.py's workload:

- matrix: the training matrix of get_offline_tensors (transactions 16 Mi rows over 1 Mi cards, 8 float32 columns and 24
  float64 aggregations; events 4 Mi x 8 float32; labels 2 Mi with 30 % NaN; 7 301 472 x 40 float32 at the defaults), scored
  by a 4-model linear ensemble.  Device: run_batch(t.features, names=t.columns), in place.  Host:
  run_batch(torch.from_dlpack(t.features).cpu().numpy(), names).
- columns: the transactions DeviceColumnBatch of FeatureSet.ingest on torch CUDA columns, scored by an Imputer -> 4-model
  linear ensemble flow over its 32 feature columns.  Device: run_batch(batch, names), packed on the device.  Host: each
  column's .cpu().numpy(), astype(float32), stacked, then run_batch.

The two paths alternate; each stage is the host clock from its start to a torch.cuda.synchronize() after it, and every
iteration compares the outputs and status words bit for bit.  A separate profiled call per workload gives the kernel times
(torch.profiler, CUDA activities): the pack (rows_pack_kernel) and the scoring launches, and the pack's bytes/s (source
bytes read plus 4 * F written per row) against the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line with the card's
name and power limit, read in the same run.

    python tools/bench_device_scoring.py [--rows 16777216] [--keys 1048576] [--iters 3]
"""

import argparse
import contextlib
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from tools.bench_training_set import card  # noqa: E402

HBM_TBS = 3.35  # H100 SXM5 80GB HBM3, data sheet


def linear_server(names, impute=None, n_models=4, seed=0):
    """a 4-model mean-vote linear ensemble over `names`, behind an optional Imputer"""
    from sklearn.linear_model import LinearRegression

    from mlrun_b200 import api

    rng = np.random.default_rng(seed)
    fn = api.new_function("scoring", kind="serving")
    step = fn.set_topology("flow", engine="sync")
    if impute is not None:
        step = step.to(api.Imputer(mapping=impute), name="imputer")
    step = step.to("*FeatureRowVotingEnsemble", name="ensemble", vote_type="regression", executor_type="array")
    for i in range(n_models):
        m = LinearRegression()
        m.coef_, m.intercept_, m.n_features_in_ = rng.normal(size=len(names)), float(rng.normal()), len(names)
        step.add_route(f"m{i + 1}", class_name="FeatureRowModelServer", model=m, model_path="")
    server = fn.to_mock_server(namespace={"FeatureRowVotingEnsemble": api.FeatureRowVotingEnsemble,
                                          "FeatureRowModelServer": api.FeatureRowModelServer})
    server.compile(list(names))
    return server


def kernel_ms(fn):
    """(pack ms, scoring ms) of the CUDA kernels one call of fn launches, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    pack = score = 0.0
    for e in prof.events():
        if getattr(e, "device_type", None) is None or "CUDA" not in str(e.device_type):
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "rows_pack_kernel" in e.name:
            pack += us / 1e3
        elif "kernel" in e.name and "Memcpy" not in e.name and "Memset" not in e.name:
            score += us / 1e3
    return pack, score


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16 << 20)
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()

    import torch

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bingest
    from mlrun_b200.feature_store import offline as boff

    nat.init(0)
    rng = np.random.default_rng(0)
    n, m, nl = args.rows, args.rows // 4, args.rows // 8
    base = 1_600_000_000 * 10**9
    tx = {"card": rng.integers(0, args.keys, size=n).astype(np.int64),
          "when": (np.arange(n, dtype=np.int64) * 10**8 + base)}
    for j in range(8):
        tx[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    ev = {"card": rng.integers(0, args.keys, size=m).astype(np.int64),
          "when": (rng.permutation(m).astype(np.int64) * 4 * 10**8 + base + 5 * 10**7)}
    for j in range(8):
        ev[f"e{j}"] = rng.standard_normal(m, dtype=np.float32)
    pick = np.sort(rng.choice(n, size=nl, replace=False))
    lab = rng.standard_normal(nl)
    lab[rng.random(nl) < 0.3] = np.nan
    labels = {"card": tx["card"][pick], "when": tx["when"][pick], "label": lab}
    tx["t3"][np.random.default_rng(1).random(n) < 0.01] = np.nan  # the Imputer's input (drawn last: the same data as before)
    cuda = {k: {c: torch.from_numpy(a).cuda() for c, a in v.items()} for k, v in (("transactions", tx), ("events", ev),
                                                                                  ("labels", labels))}
    torch.cuda.synchronize()
    txn = bingest.FeatureSet("transactions", entities=["card"], timestamp_key="when")
    for j in range(2):  # 2 columns x 6 operations x 2 windows = 24 float64 columns
        txn.add_aggregation(f"t{j}", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "1d"], "10m")
    with contextlib.redirect_stdout(io.StringIO()):
        batch = txn.ingest(cuda["transactions"])
        boff.register_offline_frame(txn, batch)
        boff.register_offline_frame(bingest.FeatureSet("events", entities=["card"], timestamp_key="when"), cuda["events"])
        boff.register_offline_frame(bingest.FeatureSet("labels", entities=["card"], timestamp_key="when"), cuda["labels"])
        t = boff.get_offline_tensors(boff.FeatureVector("v", ["transactions.*", "events.*"], label_feature="labels.label"),
                                     dtype="float32")
    torch.cuda.synchronize()
    del cuda

    feat = [k for k in batch.names if np.dtype(batch.columns[k].dtype).kind != "M"]
    servers = {"matrix": linear_server(t.columns, seed=1), "columns": linear_server(feat, impute={"t3": 0.0}, seed=2)}
    sources = {"matrix": (t.features, t.columns), "columns": (batch, feat)}

    def device(kind):
        src, names = sources[kind]
        return servers[kind].run_batch(src, names=names, with_status=True)

    def host(kind):
        src, names = sources[kind]
        if kind == "matrix":
            X = torch.from_dlpack(src).cpu().numpy()
        else:
            X = np.stack([torch.from_dlpack(src.columns[k]).cpu().numpy().astype(np.float32) for k in names], axis=1)
        return servers[kind].run_batch(X, names=names, with_status=True)

    def timed(fn, times):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        return out

    res, equal = {}, True
    for kind in ("matrix", "columns"):
        device(kind)  # warm-up: module loads, the plan's first launch
        dev_s, host_s, launches = [], [], None
        for _ in range(args.iters):
            before = nat.launch_count()
            d_out, d_st = timed(lambda: device(kind), dev_s)
            launches = nat.launch_count() - before
            h_out, h_st = timed(lambda: host(kind), host_s)
            same = d_out.numpy().tobytes() == h_out.tobytes() and d_st.numpy().tobytes() == h_st.tobytes()
            equal = equal and same
            rows, flagged = int(h_st.shape[0]), int(np.count_nonzero(h_st))
            del d_out, d_st, h_out, h_st
        try:
            pack_ms, score_ms = kernel_ms(lambda: device(kind))
        except Exception as exc:  # noqa: BLE001 -- a profiler that cannot trace leaves the kernel times unmeasured
            pack_ms = score_ms = None
            res.setdefault("profiler_error", repr(exc))
        src, names = sources[kind]
        entry = {"rows": rows, "features": len(names), "flagged_rows": flagged, "device_s": [round(x, 4) for x in dev_s],
                 "host_s": [round(x, 4) for x in host_s], "speedup_best": round(min(host_s) / min(dev_s), 1),
                 "device_launches": launches,
                 "score_kernels_ms": None if score_ms is None else round(score_ms, 3)}
        if kind == "columns":
            src_bytes = sum(np.dtype(src.columns[k].dtype).itemsize for k in names)
            pack_bytes = rows * (src_bytes + 4 * len(names))
            entry.update({"pack_kernel_ms": None if pack_ms is None else round(pack_ms, 3), "pack_bytes": pack_bytes,
                          "pack_TBps": round(pack_bytes / (pack_ms * 1e-3) / 1e12, 3) if pack_ms else None,
                          "pack_share_of_3.35TBps": round(pack_bytes / (pack_ms * 1e-3) / 1e12 / HBM_TBS, 3) if pack_ms else None})
        res[kind] = entry
    for name in list(boff._OFFLINE):
        boff._OFFLINE.pop(name).close()
    name, limit = card()
    print(json.dumps({"workload": f"transactions {n} rows over {args.keys} cards; events {m}; labels {nl}", **res,
                      "equal": equal, "gpu": name, "power_limit": limit}))
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
