"""The checker of the enrichment path -- oracle/enrichment.py's OnlineVectorService restatement -- against the REAL
OnlineVectorService (feature_store/feature_vector.py:903-1067; build container only; the online-store read is the same dict
stub under both, as in the `online_service_logic` scenario): random tables (floats, ints, nan, +-inf, None, missing features,
all-zero rows), random impute policies ("*" and per-feature constants and $mean / $min / $max / $std / $count statistics, unknown
and label features), with and without label column / index columns, single and composite keys; lookups as lists, dicts, a
single dict, unknown keys, extra columns, malformed asks.  Results, impute tables and exceptions compared.

    python -m tests.golden.diff_online             # live, needs the reference sources importable (tests/golden/_refshim.py)
    python -m tests.golden.diff_online --record    # live, and store the reference's answers in ref_online.json.xz
    python -m tests.golden.diff_online --golden    # against the stored answers: runs anywhere
"""
import json
import lzma
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import pandas as pd  # noqa: E402

from tests import api_oracle as ora  # noqa: E402
from tests.scenarios import _first_line  # noqa: E402


def norm(v):
    if isinstance(v, float) and v != v:
        return "nan"
    if isinstance(v, float) and v in (float("inf"), float("-inf")):
        return repr(v)
    if isinstance(v, dict):
        return {k: norm(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [norm(x) for x in v]
    return v.item() if hasattr(v, "item") else v


def attempt(fn):
    try:
        return norm(fn())
    except Exception as exc:  # noqa: BLE001
        return {"raised": type(exc).__name__, "message": _first_line(str(exc))}


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_online.json.xz")


def cases():
    """the 500 seeded services and lookups, in order"""
    rnd = random.Random(23)
    for case in range(500):
        nf = rnd.randint(1, 6)
        feats = [f"f{i}" for i in range(nf)]
        label = rnd.choice([None, feats[-1]]) if nf > 1 else None
        composite = rnd.random() < 0.2
        index = ["a", "b"] if composite else ["k"]
        val = lambda: rnd.choice([rnd.uniform(-5, 5), rnd.randint(-3, 3), float("nan"), float("inf"), float("-inf"), None, 0.0, 0])  # noqa: E731
        table = {}
        for i in range(rnd.randint(1, 6)):
            key = (f"k{i}", i) if composite else (f"k{i}",)
            row = {f: val() for f in feats if rnd.random() < 0.85}
            if rnd.random() < 0.1:
                row = {f: 0.0 for f in feats}
            table[key] = row
        stats = pd.DataFrame({c: [rnd.uniform(-3, 3) for _ in feats] for c in ("mean", "min", "max", "std", "count")}, index=feats)
        policy = None
        if rnd.random() < 0.75:
            policy = {}
            if rnd.random() < 0.6:
                policy["*"] = rnd.choice(["$mean", "$min", "$max", "$std", "$count", 0, 0.5, -1])
            for f in feats:
                if rnd.random() < 0.3:
                    policy[f] = rnd.choice(["$mean", "$max", 7, -2.5, 0])
            if rnd.random() < 0.08:
                policy["ghost"] = 1
        with_idx = rnd.random() < 0.3
        keys = list(table) + [("nobody", 9) if composite else ("nobody",)]
        asks = [list(rnd.choice(keys)) for _ in range(rnd.randint(1, 4))]
        yield case, (feats, label, index, table, stats, policy, with_idx, asks, composite)


def run(api, feats, label, index, table, stats, policy, with_idx, asks, composite):
    """repr of everything one service answers (results, impute table, exceptions)"""
    def go():
        svc = api.online_service(feats, index, table, stats, label, with_idx, policy)
        res = {"impute": norm(dict(svc._impute_values)),
               "lists": attempt(lambda: svc.get(asks, as_list=True)),
               "dicts": attempt(lambda: svc.get([dict(zip(index, a)) for a in asks])),
               "one": attempt(lambda: svc.get(dict(zip(index, asks[0])))),
               "extra": attempt(lambda: svc.get([{**dict(zip(index, asks[0])), "note": 1}])),
               "short": attempt(lambda: svc.get([asks[0][:1]])) if composite else None,
               "empty": attempt(lambda: svc.get([])), "string": attempt(lambda: svc.get("k0"))}
        return res
    return repr(attempt(go))


def reference_outputs():
    from tests.golden import api_reference as ref

    return [run(ref, *args) for _case, args in cases()]


def check(want_all):
    n = 0
    for (case, args), want in zip(cases(), want_all, strict=True):
        mine = run(ora, *args)
        n += 1
        if want != mine:
            print("DIFF", case, *args[:4], *args[5:])
            print("  ref :", want[:1200])
            print("  mine:", mine[:1200])
            return None
    return n


def main():
    if "--golden" in sys.argv:  # the reference's answers as recorded by --record: no reference tree needed
        with lzma.open(GOLDEN, "rt") as f:
            n = check(json.load(f))
        if n is None:
            return 1
        print("identical on", n, "random online services (recorded reference answers)")
        return 0
    want = reference_outputs()
    if "--record" in sys.argv:
        with lzma.open(GOLDEN, "wt") as f:
            json.dump(want, f)
    n = check(want)
    if n is None:
        return 1
    print("identical on", n, "random online services")
    return 0


if __name__ == "__main__":
    sys.exit(main())
