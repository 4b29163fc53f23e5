"""The feature pipeline end to end, from raw columns to a training matrix in a torch CUDA tensor, two ways, alternated in one
run on tools/bench_training_tensors.py's workload: transactions 16 Mi rows over 1 Mi cards (8 float32 columns, 24 float64
aggregations made by add_aggregation at ingest), events 4 Mi x 8 float32, labels 2 Mi with 30 % NaN,
label_feature="labels.label", a float32 matrix.

- host chain: pandas frames -> ingest -> register_offline_frame(frame) -> get_offline_tensors -> torch.from_dlpack
- device chain: torch CUDA columns -> ingest -> register_offline_frame(DeviceColumnBatch / mapping) -> get_offline_tensors ->
  torch.from_dlpack

Each stage's time is the host clock from its start to a torch.cuda.synchronize() after it.  Prints one JSON line: the
per-iteration stage times of both chains, the launches of each device stage (`b2s_launch_count`), whether both chains gave
the same matrix (bit for bit where finite, NaN where NaN) and the card name and power limit, read in the same run.

    python tools/bench_device_chain.py [--rows 16777216] [--keys 1048576] [--iters 3]
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
    from mlrun_b200.feature_store import offline as boff

    nat.init(0)
    rng = np.random.default_rng(0)
    n, m, nl = args.rows, args.rows // 4, args.rows // 8
    base = 1_600_000_000 * 10**9
    tx = {"card": rng.integers(0, args.keys, size=n).astype(np.int64),
          "when": (np.arange(n, dtype=np.int64) * 10**8 + base).view("datetime64[ns]")}
    for j in range(8):
        tx[f"t{j}"] = rng.standard_normal(n, dtype=np.float32)
    ev = {"card": rng.integers(0, args.keys, size=m).astype(np.int64),
          "when": (rng.permutation(m).astype(np.int64) * 4 * 10**8 + base + 5 * 10**7).view("datetime64[ns]")}
    for j in range(8):
        ev[f"e{j}"] = rng.standard_normal(m, dtype=np.float32)
    pick = np.sort(rng.choice(n, size=nl, replace=False))
    lab = rng.standard_normal(nl)
    lab[rng.random(nl) < 0.3] = np.nan
    labels = {"card": tx["card"][pick], "when": tx["when"][pick], "label": lab}
    frames = {k: pd.DataFrame(v) for k, v in (("transactions", tx), ("events", ev), ("labels", labels))}
    cuda = {k: {c: torch.from_numpy(np.array(a.view(np.int64) if a.dtype.kind == "M" else a)).cuda() for c, a in v.items()}
            for k, v in (("transactions", tx), ("events", ev), ("labels", labels))}
    torch.cuda.synchronize()

    def sets():
        txn = bingest.FeatureSet("transactions", entities=["card"], timestamp_key="when")
        for j in range(2):  # 2 columns x 6 operations x 2 windows = 24 float64 columns
            txn.add_aggregation(f"t{j}", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "1d"], "10m")
        return (txn, bingest.FeatureSet("events", entities=["card"], timestamp_key="when"),
                bingest.FeatureSet("labels", entities=["card"], timestamp_key="when"))

    vector = boff.FeatureVector("v", ["transactions.*", "events.*"], label_feature="labels.label")

    def timed(fn, times, launches=None):
        before = nat.launch_count()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        if launches is not None:
            launches.append(nat.launch_count() - before)
        return out

    def chain(device, stage_s, stage_k):
        txn, evs, lbs = sets()
        src = cuda if device else frames
        batch = timed(lambda: txn.ingest(src["transactions"]), stage_s["ingest"], stage_k["ingest"])

        def register():
            boff.register_offline_frame(txn, batch)
            boff.register_offline_frame(evs, src["events"])
            boff.register_offline_frame(lbs, src["labels"])

        timed(register, stage_s["register"], stage_k["register"])
        t = timed(lambda: boff.get_offline_tensors(vector, dtype="float32"), stage_s["tensors"], stage_k["tensors"])
        x = timed(lambda: torch.from_dlpack(t.features), stage_s["from_dlpack"])
        if not device:
            assert t.stats["h2d_ms"] > 0
        else:
            assert t.stats["h2d_ms"] == 0
        return x, t

    stages = ("ingest", "register", "tensors", "from_dlpack")
    host_s, dev_s = ({k: [] for k in stages} for _ in range(2))
    host_k, dev_k = ({k: [] for k in stages} for _ in range(2))
    equal = True
    for _ in range(args.iters):
        xh, th = chain(False, host_s, host_k)
        xd, td = chain(True, dev_s, dev_k)
        a, b = xh.cpu().numpy(), xd.cpu().numpy()
        same = a.shape == b.shape and th.columns == td.columns and np.array_equal(np.isnan(a), np.isnan(b)) and \
            a[~np.isnan(a)].tobytes() == b[~np.isnan(b)].tobytes() and th.label.numpy().tobytes() == td.label.numpy().tobytes() \
            and th.order.numpy().tobytes() == td.order.numpy().tobytes()
        equal = equal and bool(same)
        shape = list(a.shape)
        del xh, xd, th, td, a, b
    for name in list(boff._OFFLINE):
        boff._OFFLINE.pop(name).close()
    name, limit = card()

    def total(s):
        return [round(sum(s[k][i] for k in stages), 3) for i in range(args.iters)]

    print(json.dumps({
        "workload": f"transactions {n} rows x (8 f32 + 24 f64 aggregations) over {args.keys} cards; events {m} x 8 f32; "
                    f"labels {nl}, 30% NaN; float32 matrix",
        "matrix": shape,
        "host_chain_s": {k: [round(t, 3) for t in v] for k, v in host_s.items()}, "host_chain_total_s": total(host_s),
        "device_chain_s": {k: [round(t, 3) for t in v] for k, v in dev_s.items()}, "device_chain_total_s": total(dev_s),
        "device_launches": {k: v[-1] for k, v in dev_k.items() if v}, "host_launches": {k: v[-1] for k, v in host_k.items() if v},
        "speedup_best": round(min(total(host_s)) / min(total(dev_s)), 2), "equal": equal, "gpu": name, "power_limit": limit,
    }))
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
