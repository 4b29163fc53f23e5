"""Windowed-aggregation benchmark: 16 Mi rows over 1 Mi int64 keys, timestamps over 7 days (each key's rows in time order),
two float32 columns; count / sum / avg / min / max / stddev over 1 h, 6 h and 24 h sliding every 10 min on one column, and
the same operations over a fixed 1 h window on the other.

Prints one JSON line: the device-resident run (b2s_agg_time_device, CUDA events on the library stream; every input far larger
than L2) split into the key sort and the aggregation, the launches of one run, the algorithmic bytes per row and their share of
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), FeatureSet.ingest rows/s end to end from a pandas frame, the oracle's rate
on the same host over a bounded sample, and the card and power limit the numbers were taken on.

    python tools/bench_aggregate.py [--rows 16777216] [--keys 1048576] [--iters 5] [--oracle-rows 2000]
"""

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

HBM_DATASHEET = 3.35e12
MIN, HOUR, DAY = 60 * 10**9, 3600 * 10**9, 86400 * 10**9
OPS = ["count", "sum", "avg", "min", "max", "stddev"]


def card():
    """name and power limit of GPU 0, read now (nvidia-smi's query only reads)"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:  # noqa: BLE001 -- reported as unknown rather than guessed
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16 << 20)
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--oracle-rows", type=int, default=2000)
    args = ap.parse_args()

    import torch

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bi
    from oracle import aggregate as oa

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the H100")
    lib = nat.init(0)
    n = args.rows
    rng = np.random.default_rng(0)
    keys = rng.integers(0, args.keys, n).astype(np.int64)
    ts = np.sort(rng.integers(0, 7 * DAY, n)).astype(np.int64) + 1_700_000_000 * 10**9  # arrival order = time order
    x = rng.standard_normal(n, dtype=np.float32) * 50 + 100
    y = rng.standard_normal(n, dtype=np.float32)
    sliding = [("1h", HOUR), ("6h", 6 * HOUR), ("24h", DAY)]
    aggs = [dict(name="x", column="x", operations=OPS, windows=sliding, period=10 * MIN),
            dict(name="y", column="y", operations=OPS, windows=[("1h", HOUR)], period=None)]
    n_out = sum(len(a["operations"]) * len(a["windows"]) for a in aggs)

    # device-resident run
    dev = torch.device("cuda", 0)
    d_keys, d_ts = torch.from_numpy(keys).to(dev), torch.from_numpy(ts).to(dev)
    d_src = {"x": torch.from_numpy(x).to(dev), "y": torch.from_numpy(y).to(dev)}
    d_cnt = torch.zeros(3, dtype=torch.int64, device=dev)
    d_outs, specs, keep = [], [], []
    for a in aggs:
        ptrs = []
        for _op in sorted(a["operations"], key=nat.AGG_OPS.get):  # the C-ABI's output order: op bits ascending
            for _w in a["windows"]:
                t = torch.empty(n, dtype=torch.float64, device=dev)
                d_outs.append(t)
                ptrs.append(t.data_ptr())
        win = np.array([w for _l, w in a["windows"]], np.int64)
        parr = (C.c_void_p * len(ptrs))(*ptrs)
        keep += [win, parr]
        specs.append(nat.AggSpec(d_src[a["column"]].data_ptr(), nat.COL_F32, sum(nat.AGG_OPS[o] for o in a["operations"]),
                                 a["period"] or 0, len(win), win.ctypes.data_as(C.POINTER(C.c_int64)), parr))
    c_specs = (nat.AggSpec * len(specs))(*specs)
    torch.cuda.synchronize()
    sort_ms, total_ms = C.c_float(), C.c_float()
    nat.check(lib.b2s_agg_time_device(d_keys.data_ptr(), d_ts.data_ptr(), n, c_specs, len(specs), d_cnt.data_ptr(), 1,
                                      C.byref(sort_ms), C.byref(total_ms)))  # warm-up: the stream's memory pool grows here
    before = nat.launch_count()
    nat.check(lib.b2s_agg_time_device(d_keys.data_ptr(), d_ts.data_ptr(), n, c_specs, len(specs), d_cnt.data_ptr(), args.iters,
                                      C.byref(sort_ms), C.byref(total_ms)))
    launches = (nat.launch_count() - before) // args.iters
    sort = sort_ms.value / args.iters
    total = total_ms.value / args.iters
    # algorithmic bytes per row: key and timestamp in, each source column in, each float64 output out
    bytes_row = 8 + 8 + 4 * len(d_src) + 8 * n_out
    dev_rate = n / (total * 1e-3)
    del d_outs, d_keys, d_ts, d_src
    torch.cuda.empty_cache()

    # end to end from a pandas frame
    df = pd.DataFrame({"card": keys, "ts": pd.to_datetime(ts), "x": x, "y": y})
    fset = bi.FeatureSet("quotes", entities=["card"], timestamp_key="ts")
    fset.add_aggregation("x", OPS, [w for w, _ in sliding], "10m")
    fset.add_aggregation("y", OPS, "1h")
    fset.ingest(df)  # lowering, pinned blocks
    t0 = time.perf_counter()
    reps = 2
    for _ in range(reps):
        out = fset.ingest(df)
    e2e = (time.perf_counter() - t0) / reps
    assert out.shape == (n, 3 + n_out), out.shape
    agg_stats = fset.plan.agg.stats

    # the oracle on the same host, over a bounded sample: the last rows of the frame's first 64 x oracle-rows rows (about 1.3 h
    # of the 7 days, so a key has few earlier rows there: an upper bound on its rate over the whole frame)
    m = args.oracle_rows * 64
    sub = slice(0, m)
    t0 = time.perf_counter()
    oa.aggregate(keys[sub], ts[sub], {"x": x[sub], "y": y[sub]}, aggs, rows=np.arange(m - args.oracle_rows, m))
    oracle_rate = args.oracle_rows / (time.perf_counter() - t0)

    name, limit = card()
    print(json.dumps({
        "workload": {"rows": n, "keys": args.keys, "span": "7d", "columns": 2, "outputs": n_out,
                     "aggregations": "count/sum/avg/min/max/stddev x 1h/6h/24h every 10m on x; the same x fixed 1h on y"},
        "device_ms": {"sort": round(sort, 3), "aggregate": round(total - sort, 3), "total": round(total, 3)},
        "launches": launches,
        "device_rows_per_s": round(dev_rate),
        "bytes_per_row_algorithmic": bytes_row,
        "hbm_share_of_datasheet_3.35TBps": round(dev_rate * bytes_row / HBM_DATASHEET, 4),
        "ingest_e2e_s": round(e2e, 3), "ingest_rows_per_s": round(n / e2e),
        "ingest_agg_call": {"h2d_ms": round(agg_stats["h2d_ms"], 3), "kernel_ms": round(agg_stats["kernel_ms"], 3),
                            "kernels": agg_stats["kernels"]},
        "oracle_rows_per_s": round(oracle_rate, 1), "oracle_sample_rows": args.oracle_rows,
        "gpu": name, "power_limit": limit,
    }))


if __name__ == "__main__":
    main()
