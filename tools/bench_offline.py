"""Point-in-time retrieval benchmark: 4 feature sets of 8 Mi rows x 32 float32 features over 1 Mi keys, 4 Mi entity rows.

Prints one JSON line: index-build ms per set, the device-resident join (CUDA events on torch's stream, every input far
larger than L2) split into the entity sort and the join, all sets in one call against one call per set, algorithmic bytes per entity row and their share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), the
end-to-end rate from a pandas entity frame, and pandas merge_asof (the local engine's merge) on the same frames.

    python tools/bench_offline.py [--rows 8388608] [--keys 1048576] [--entity 4194304] [--sets 4] [--feats 32] [--iters 10]
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

HBM_DATASHEET = 3.35e12


def frames(args, rng):
    out = {}
    for s in range(args.sets):
        cols = {"id": rng.integers(0, args.keys, size=args.rows).astype(np.int64),
                "when": pd.to_datetime(rng.permutation(args.rows).astype(np.int64) * 1000 + 10**18)}
        for j in range(args.feats):
            cols[f"s{s}f{j}"] = rng.standard_normal(args.rows, dtype=np.float32)
        out[f"fs{s}"] = pd.DataFrame(cols)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=8 << 20)
    ap.add_argument("--keys", type=int, default=1 << 20)
    ap.add_argument("--entity", type=int, default=4 << 20)
    ap.add_argument("--sets", type=int, default=4)
    ap.add_argument("--feats", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--no-pandas", action="store_true")
    args = ap.parse_args()

    import torch

    from mlrun_b200 import _native as nat
    from mlrun_b200.feature_store import ingest as bingest
    from mlrun_b200.feature_store import offline as boff
    from oracle import offline as oo

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the H100")
    nat.init(0)
    rng = np.random.default_rng(0)
    fr = frames(args, rng)
    entity = pd.DataFrame({"id": rng.integers(0, args.keys, size=args.entity).astype(np.int64),
                           "t": pd.to_datetime(rng.permutation(args.entity).astype(np.int64) * 2000 + 10**18 + 7)})

    build_ms = []
    for name, frame in fr.items():
        t0 = time.perf_counter()
        boff.register_offline_frame(bingest.FeatureSet(name, entities=["id"], timestamp_key="when"), frame)
        build_ms.append((time.perf_counter() - t0) * 1e3)
    srcs = [boff._OFFLINE[n] for n in fr]

    # device-resident join on torch's stream, timed with CUDA events
    n, F = args.entity, args.feats
    dev = torch.device("cuda:0")
    d_ts = torch.from_numpy(entity["t"].to_numpy().view(np.int64).copy()).to(dev)
    d_keys = torch.from_numpy(entity["id"].to_numpy().copy()).to(dev)
    d_out = [torch.empty((F, n), dtype=torch.float32, device=dev) for _ in srcs]
    d_tsout = [torch.empty(n, dtype=torch.int64, device=dev) for _ in srcs]
    d_found = [torch.empty(n, dtype=torch.uint8, device=dev) for _ in srcs]
    d_order = torch.empty(n, dtype=torch.int64, device=dev)
    d_miss = torch.zeros(len(srcs), dtype=torch.int64, device=dev)
    keep = []

    def c_sets(which):
        arr = (nat.PitSet * max(len(which), 1))()
        for i, s in enumerate(which):
            src = srcs[s]
            descs = (nat.PitOut * F)(*[nat.PitOut(src.features[f"s{s}f{j}"][0], 4, boff._NAN32, d_out[s][j].data_ptr()) for j in range(F)])
            keep.append(descs)
            arr[i] = nat.PitSet(src.index._h, d_keys.data_ptr(), 1, F, descs, d_tsout[s].data_ptr(), d_found[s].data_ptr())
        return arr, len(which)

    lib = nat.load()
    side = torch.cuda.Stream()  # a stream of its own: handle 0 would mean the library's stream, not torch's
    torch.cuda.synchronize()
    stream = side.cuda_stream

    def run(sets):
        nat.check(lib.b2s_pit_join_device(d_ts.data_ptr(), n, sets[0], sets[1], None, 0, d_order.data_ptr(), d_miss.data_ptr(), stream))

    def timed(sets):
        for _ in range(2):
            run(sets)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(side)
        for _ in range(args.iters):
            run(sets)
        b.record(side)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.iters

    all_sets = c_sets(list(range(len(srcs))))
    one_each = [c_sets([s]) for s in range(len(srcs))]
    sort_only = c_sets([])
    t_sort = timed(sort_only)
    t_all = timed(all_sets)
    t_each = [timed(s) for s in one_each]
    join_ms = t_all - t_sort
    per_set_launches_ms = sum(t - t_sort for t in t_each)
    # algorithmic bytes per entity row: timestamp in, order out; per set: key, slot (16), a run timestamp, the feature row
    # read, the feature columns written, the matched timestamp and the found flag
    per_set = 8 + 16 + 8 + 4 * F + 4 * F + 8 + 1
    bytes_row = 8 + 8 + len(srcs) * per_set
    found = float(torch.stack([f.double().mean() for f in d_found]).mean())

    # end to end from a pandas entity frame
    vec = boff.FeatureVector("bench", [f"{n_}.*" for n_ in fr])
    boff.get_offline_features(vec, entity.iloc[:1024], "t")
    t0 = time.perf_counter()
    res = boff.get_offline_features(vec, entity, "t")
    e2e_s = time.perf_counter() - t0

    pandas_s = None
    if not args.no_pandas:
        t0 = time.perf_counter()
        want = oo.get_offline_features({k: (["id"], "when", v) for k, v in fr.items()}, vec.features, entity, "t")
        pandas_s = time.perf_counter() - t0
        pd.testing.assert_frame_equal(res.to_dataframe(), want, check_exact=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    line = {
        "workload": f"{args.sets} sets x {args.rows} rows x {F} float32 over {args.keys} keys, {n} entity rows",
        "gpu": smi, "index_build_ms": [round(x, 1) for x in build_ms],
        "entity_sort_ms": round(t_sort, 3), "join_ms_all_sets_one_call": round(join_ms, 3),
        "join_ms_one_call_per_set": round(per_set_launches_ms, 3), "sort_plus_join_ms": round(t_all, 3),
        "algorithmic_bytes_per_entity_row": bytes_row,
        "join_fraction_of_datasheet_hbm_3.35TBps": round(bytes_row * n / (join_ms * 1e-3) / HBM_DATASHEET, 3),
        "hit_rate": round(found, 4),
        "end_to_end_rows_per_s": round(n / e2e_s), "end_to_end_s": round(e2e_s, 3),
        "pandas_merge_asof_s": None if pandas_s is None else round(pandas_s, 3),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
