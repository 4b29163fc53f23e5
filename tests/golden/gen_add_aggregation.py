"""Records what the REAL reference's FeatureSet.add_aggregation / _add_aggregation_to_existing do (feature_set.py:689-851) on
a fixed list of call sequences: the graph's steps (name, class, class_args, after), the registered features and the errors.
`python -m tests.golden.gen_add_aggregation --record` writes tests/golden/ref_add_aggregation.json where the reference sources
are importable; tests/test_aggregate_cpu.py compares the mirror with it on every machine.  Operations merged into an existing
aggregation come from the reference's list(set(...)), whose order varies between processes: they are recorded sorted."""

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "ref_add_aggregation.json")

# each scenario: feature-set keyword arguments, then add_aggregation calls (keyword arguments)
SCENARIOS = [
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum", "max"], windows="1h", period="10m", name="bids")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum", "max"], windows="1h", period="10m", name="bids"),
                                                  dict(column="bid", operations=["min", "sum"], windows="1h", period="10m", name="bids")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows=["1h", "2h"], period="1h"),
                                                  dict(column="bid", operations=["max"], windows=["1h"], period="1h")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows="1h", period="10m", name="b"),
                                                  dict(column="bid", operations=["max"], windows="1h", period="20m", name="b")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows="1h", period="10m", name="b"),
                                                  dict(column="ask", operations=["max"], windows="1h", period="10m", name="b")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows="1h")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows="1h"),
                                                  dict(column="bid", operations=["max"], windows="1h")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations="sum", windows="1h")]),
    ({"entities": ["k"], "timestamp_key": "ts"}, [dict(column="bid", operations=["sum"], windows=["1h"], period="1h", step_name="A1"),
                                                  dict(column="ask", operations=["avg", "count"], windows=["1d", "2d"], step_name="A2")]),
    ({"entities": ["first_name"]}, [dict(name="bids", column="bid", operations=["sum", "max"], windows="1h", period="10m")]),
]


def observe(fs_cls, entity_cls, kwargs, calls):
    kw = dict(kwargs)
    kw["entities"] = [entity_cls(e) for e in kw["entities"]]
    fset = fs_cls("s", **kw)
    out = []
    for call in calls:
        try:
            fset.add_aggregation(**call)
            out.append(None)
        except Exception as err:  # noqa: BLE001 -- the outcome is what is recorded
            out.append([type(err).__name__, str(err)])
    graph = fset.graph if hasattr(fset, "graph") else fset.spec.graph
    steps = []
    for name, step in graph.steps.items():
        args = json.loads(json.dumps(step.class_args, default=str))
        for agg in args.get("aggregates", []):
            agg["operations"] = sorted(agg["operations"])
        steps.append([name, step.class_name, args, list(step.after or [])])
    feats = fset.features if not hasattr(fset, "spec") or not hasattr(fset.spec, "features") else fset.spec.features
    features = {k: [f.name, bool(getattr(f, "aggregate", False)), str(getattr(f.value_type, "value", f.value_type))]
                for k, f in feats.items()}
    return {"errors": out, "steps": steps, "features": features}


def main():
    if "--record" not in sys.argv:
        print(__doc__)
        return
    sys.path.insert(0, HERE)
    import _refshim

    _refshim.install()
    import mlrun.feature_store as fs
    from mlrun.features import Entity

    got = [observe(fs.FeatureSet, Entity, kw, calls) for kw, calls in SCENARIOS]
    with open(GOLDEN, "w") as f:
        json.dump(got, f, indent=1, sort_keys=True)
    print("recorded", len(got), "scenarios of the real reference's add_aggregation")


if __name__ == "__main__":
    main()
