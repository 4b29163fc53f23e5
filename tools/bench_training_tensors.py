"""Training-set tensors benchmark: tools/bench_training_set.py's workload handed over as device tensors.

transactions: 16 Mi rows over 1 Mi cards, 8 float32 columns plus 24 float64 aggregation columns made by add_aggregation at
ingest (the spine); events: 4 Mi rows x 8 float32 columns; labels: 2 Mi rows, 30 % of their labels NaN; no entity rows,
label_feature="labels.label", a float32 matrix.

Prints one JSON line: the device time per phase (CUDA events), the pack kernel alone (CUDA events around its launch,
over 10 calls), its algorithmic bytes/s against the H100's 3.35 TB/s HBM3, end to end from registered
frames to a CUDA torch tensor, the baseline (get_offline_features -> to_dataframe -> to_numpy(float32) ->
torch.from_numpy().cuda()) alternated with it, whether both give the same matrix, and the card and power limit.

    python tools/bench_training_tensors.py [--rows 16777216] [--keys 1048576] [--iters 3]
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

HBM_TBS = 3.35  # H100 SXM5 80GB HBM3 peak


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
    args = ap.parse_args()

    import torch

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bingest
    from mlrun_b200.feature_store import offline as boff

    nat.init(0)
    rng = np.random.default_rng(0)
    n, m, nl = args.rows, args.rows // 4, args.rows // 8
    base = 1_600_000_000 * 10**9
    raw = {"card": rng.integers(0, args.keys, size=n).astype(np.int64),
           "when": pd.to_datetime(np.arange(n, dtype=np.int64) * 10**8 + base)}
    for j in range(8):
        raw[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    txn = bingest.FeatureSet("transactions", entities=["card"], timestamp_key="when")
    for j in range(2):  # 2 columns x 6 operations x 2 windows = 24 float64 columns
        txn.add_aggregation(f"t{j}", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "1d"], "10m")
    ingested = txn.ingest(pd.DataFrame(raw))
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
    for fs, fr in ((txn, ingested), (ev, events), (ls, labels)):
        boff.register_offline_frame(fs, fr)
    vector = boff.FeatureVector("v", ["transactions.*", "events.*"], label_feature="labels.label")

    def new_path():
        t = boff.get_offline_tensors(vector, dtype="float32")
        x = torch.from_dlpack(t.features)
        torch.cuda.synchronize()
        return t, x

    def baseline():
        resp = boff.get_offline_features(vector)
        frame = resp.to_dataframe()
        cols = [c for c in frame.columns if c != "label"]
        x = torch.from_numpy(frame[cols].to_numpy(np.float32)).cuda()
        torch.cuda.synchronize()
        return cols, x

    t, x_new = new_path()  # warm-up of both
    cols, x_old = baseline()
    same = cols == t.columns and torch.equal(torch.isnan(x_new), torch.isnan(x_old)) and bool(
        (x_new.nan_to_num(0.0).view(torch.int32) == x_old.nan_to_num(0.0).view(torch.int32)).all())
    del x_old
    new_s, old_s, stats = [], [], []
    for _ in range(args.iters):  # alternated, so that drift hits both
        del t, x_new
        t0 = time.perf_counter()
        t, x_new = new_path()
        new_s.append(time.perf_counter() - t0)
        stats.append(t.stats)
        t0 = time.perf_counter()
        _cols, x_old = baseline()
        old_s.append(time.perf_counter() - t0)
        del x_old

    # the pack kernel alone: CUDA events around its launch, over repeated calls of the whole entry point
    pack = []
    for _ in range(10):
        tt = boff.get_offline_tensors(vector, dtype="float32")
        pack.append(tt.stats["pack_ms"])
        del tt
    st = stats[-1]
    kept, f = t.rows, len(t.columns)
    width = {c: ingested[c].dtype.itemsize for c in ingested.columns}
    width.update({c: events[c].dtype.itemsize for c in events.columns})
    # algorithmic bytes: every selected output read once per entity row, with the keep flag and the events' found flag;
    # the kept rows' order and label read and written; the matrix written once
    read = n * (sum(width[c] for c in t.columns) + 1 + 1) + kept * (8 + 8)
    write = kept * f * 4 + kept * (8 + 8)
    pack_ms = float(np.median(pack))
    name, limit = card()
    res = {
        "workload": f"transactions {n} rows x (8 f32 + 24 f64 aggregations) over {args.keys} cards; events {m} x 8 f32; labels {nl}, 30% NaN; float32 matrix",
        "rows": n, "kept_rows": kept, "features": f,
        "sort_ms": round(st["sort_ms"], 2), "join_ms": round(st["join_ms"], 2), "compact_ms": round(st["compact_ms"], 2),
        "keep_scan_ms": round(st["compact_ms"] - st["pack_ms"], 2), "pack_ms_median_of_10": round(pack_ms, 2),
        "pack_ms_all": [round(p, 2) for p in pack],
        "h2d_ms": round(st["h2d_ms"], 2), "kernel_ms": round(st["kernel_ms"], 2), "kernels": st["kernels"],
        "pack_bytes": read + write, "pack_tb_per_s": round((read + write) / pack_ms / 1e9, 3),
        "pack_share_of_hbm_peak": round((read + write) / pack_ms / 1e9 / HBM_TBS, 3),
        "tensors_end_to_end_s": [round(s, 3) for s in new_s], "baseline_end_to_end_s": [round(s, 3) for s in old_s],
        "speedup": round(min(old_s) / min(new_s), 2), "same_matrix": bool(same),
        "gpu": name, "power_limit": limit,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
