"""Training-set benchmark: a fraud-shaped entity-less vector with a label.

transactions: 16 Mi rows over 1 Mi cards, 8 float32 columns plus 24 float64 aggregation columns made by add_aggregation at
ingest (the spine); events: 4 Mi rows x 8 float32 columns; labels: 2 Mi rows, 30 % of their labels NaN.  The query is
get_offline_features(FeatureVector(["transactions.*", "events.*"], label_feature="labels.label")).

Prints one JSON line: the device time split into the entity sort, the join and the label compaction (CUDA events), the
bytes copied back with the filter and without it, the end-to-end rate, the oracle's pandas time on the same frames, and
the card and power limit the numbers were taken on.

    python tools/bench_training_set.py [--rows 16777216] [--keys 1048576] [--iters 3] [--oracle 1]
"""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402


def card():
    """name and power limit of GPU 0, read now (nvidia-smi's query only reads)"""
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [s.strip() for s in out.split(",")]
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16 << 20)
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--oracle", type=int, default=1)
    args = ap.parse_args()

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bingest
    from mlrun_b200.feature_store import offline as boff

    nat.init(0)
    rng = np.random.default_rng(0)
    n, m, nl = args.rows, args.rows // 4, args.rows // 8
    base = 1_600_000_000 * 10**9
    raw = {"card": rng.integers(0, args.keys, size=n).astype(np.int64),
           "when": pd.to_datetime(np.arange(n, dtype=np.int64) * 10**8 + base)}  # distinct: pandas' unstable sort is exact
    for j in range(8):
        raw[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    txn = bingest.FeatureSet("transactions", entities=["card"], timestamp_key="when")
    for j in range(2):  # 2 columns x 6 operations x 2 windows = 24 float64 columns
        txn.add_aggregation(f"t{j}", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "1d"], "10m")
    t0 = time.perf_counter()
    ingested = txn.ingest(pd.DataFrame(raw))
    ingest_s = time.perf_counter() - t0
    ingested = ingested.reset_index() if ingested.index.names[0] else ingested
    events = {"card": rng.integers(0, args.keys, size=m).astype(np.int64),
              "when": pd.to_datetime(rng.permutation(m).astype(np.int64) * 4 * 10**8 + base + 5 * 10**7)}
    for j in range(8):
        events[f"e{j}"] = rng.standard_normal(m, dtype=np.float32)
    events = pd.DataFrame(events)
    pick = np.sort(rng.choice(n, size=nl, replace=False))
    lab = rng.standard_normal(nl)
    lab[rng.random(nl) < 0.3] = np.nan
    labels = pd.DataFrame({"card": raw["card"][pick], "when": raw["when"][pick], "label": lab})
    ev = bingest.FeatureSet("events", entities=["card"], timestamp_key="when")
    ls = bingest.FeatureSet("labels", entities=["card"], timestamp_key="when")
    t0 = time.perf_counter()
    for fs, fr in ((txn, ingested), (ev, events), (ls, labels)):
        boff.register_offline_frame(fs, fr)
    register_s = time.perf_counter() - t0

    calls = []
    real = boff.pit_train

    def recorded(*a, **k):
        res = real(*a, with_stats=True)
        calls.append(res[-1])
        return res[:-1]

    boff.pit_train = recorded
    vector = boff.FeatureVector("v", ["transactions.*", "events.*"], label_feature="labels.label")
    boff.get_offline_features(vector).to_dataframe()  # warm-up
    times = []
    for _ in range(args.iters):
        calls.clear()
        t0 = time.perf_counter()
        got = boff.get_offline_features(vector).to_dataframe()
        times.append(time.perf_counter() - t0)
    st = calls[-1]
    # bytes per row the device copies back: every output, found flag and ts_out of the joined sets, the spine's device
    # columns and order
    spine_cols = [c for c in ingested.columns if ingested[c].dtype.kind in "iufMb"]
    row_bytes = sum(ingested[c].dtype.itemsize for c in spine_cols) + 8 * 4 + 9 + 8 + 9 + 8
    name, limit = card()
    res = {
        "workload": f"transactions {n} rows x (8 f32 + 24 f64 aggregations) over {args.keys} cards; events {m} x 8 f32; labels {nl}, 30% NaN",
        "rows": n, "kept_rows": st["kept"], "result_columns": got.shape[1],
        "sort_ms": round(st["sort_ms"], 2), "join_ms": round(st["join_ms"], 2), "compact_ms": round(st["compact_ms"], 2),
        "h2d_ms": round(st["h2d_ms"], 2), "d2h_ms": round(st["d2h_ms"], 2), "kernels": st["kernels"],
        "copy_back_bytes_filtered": st["kept"] * row_bytes, "copy_back_bytes_unfiltered": n * row_bytes,
        "end_to_end_s": [round(t, 3) for t in times], "rows_per_s": round(n / min(times)),
        "ingest_s": round(ingest_s, 3), "register_s": round(register_s, 3),
        "gpu": name, "power_limit": limit,
    }
    if args.oracle:
        from tests import training_oracle

        frames = {"transactions": (["card"], "when", ingested), "events": (["card"], "when", events), "labels": (["card"], "when", labels)}
        t0 = time.perf_counter()
        want = training_oracle.get_offline_features(frames, ["transactions.*", "events.*"], None, label_feature="labels.label")
        res["oracle_pandas_s"] = round(time.perf_counter() - t0, 3)
        pd.testing.assert_frame_equal(got, want, check_exact=True)
        res["equal_to_oracle"] = True
    print(json.dumps(res))


if __name__ == "__main__":
    main()
