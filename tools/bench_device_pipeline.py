"""Feature-set ingest from CUDA columns against the same ingest from a pandas frame, on the fraud workload's transactions set
(tools/bench_training_set.py): 16 Mi rows over 1 Mi cards, 8 float32 columns, 24 float64 aggregation columns made by
add_aggregation.  The two paths alternate; each iteration checks that the device batch equals the frame bit for bit.

Prints one JSON line: each path's ingest times (the frame path from a pandas frame to a result frame; the device path from
torch CUDA columns to a DeviceColumnBatch in HBM, synchronised), the device path's launches, staged and converted bytes, and
the card and power limit the numbers were taken on.  Registration and training tensors from device sets are measured by
tools/bench_device_chain.py, which times the whole chain from CUDA columns to a training matrix.

    python tools/bench_device_pipeline.py [--rows 16777216] [--keys 1048576] [--iters 3]
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
    ap.add_argument("--rows", type=int, default=16 << 20)
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()

    import torch

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bingest

    nat.init(0)
    rng = np.random.default_rng(0)
    n = args.rows
    base = 1_600_000_000 * 10**9
    raw = {"card": rng.integers(0, args.keys, size=n).astype(np.int64),
           "when": pd.to_datetime(np.arange(n, dtype=np.int64) * 10**8 + base)}
    for j in range(8):
        raw[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    frame = pd.DataFrame(raw)
    cuda = {k: torch.from_numpy(np.array(v.to_numpy().view(np.int64) if k == "when" else v)).cuda()
            for k, v in frame.items()}
    torch.cuda.synchronize()

    def txn():
        fs = bingest.FeatureSet("transactions", entities=["card"], timestamp_key="when")
        for j in range(2):  # 2 columns x 6 operations x 2 windows = 24 float64 columns
            fs.add_aggregation(f"t{j}", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "1d"], "10m")
        return fs

    fs_host, fs_dev = txn(), txn()
    fs_host.ingest(frame.iloc[:4096])  # warm-up: lowering, first launches
    fs_dev.ingest({k: v[:4096] for k, v in cuda.items()})
    host_s, dev_s = [], []
    for _ in range(args.iters):
        t0 = time.perf_counter()
        want = fs_host.ingest(frame)
        host_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        got = fs_dev.ingest(cuda)
        dev_s.append(time.perf_counter() - t0)  # results are ready when ingest returns
        for name in got.names:
            a, b = got[name].numpy(), want[name].to_numpy()
            assert a.dtype == b.dtype and a.tobytes() == b.tobytes(), name
        del got, want
    st = fs_dev.plan.stats
    name, limit = card()
    print(json.dumps({
        "workload": f"transactions {n} rows x (8 f32 + 24 f64 aggregations) over {args.keys} cards",
        "frame_ingest_s": [round(t, 3) for t in host_s], "device_ingest_s": [round(t, 3) for t in dev_s],
        "speedup": round(min(host_s) / min(dev_s), 1), "device_kernels": st["kernels"],
        "staged_bytes": st["staged_bytes"], "converted_bytes": st["converted_bytes"], "equal": True,
        "gpu": name, "power_limit": limit,
    }))


if __name__ == "__main__":
    main()
