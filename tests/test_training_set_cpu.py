"""Training sets on CPU: the oracle against the goldens of the REAL BaseMerger.start (tests/golden/gen_training_set.py);
the product's host layer -- the spine, the label append, `*` exclusion and dropna, float64 columns, dtypes, row labels --
over a numpy emulation of b2s_pit_train_host (tests/emulated_train.py) against the same goldens; and every refusal.  The
CUDA kernels are tests/test_gpu_training_set.py."""

import lzma
import pickle

import numpy as np
import pandas as pd
import pytest

from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from mlrun_b200.lowering import LoweringError
from mlrun_b200.serving.resolve import MLRunInvalidArgumentError
from tests import emulated_train
from tests import offline_fixtures as fx
from tests.golden import diff_training_set
from tests.golden import gen_training_set as gen

GOLDEN = pickle.load(lzma.open(gen.GOLDEN))


@pytest.mark.parametrize("seed", range(gen.N_GOLDEN))
def test_oracle_equals_the_real_reference(seed):
    got = gen.run(diff_training_set.oracle_training_set, seed)
    assert diff_training_set.same(got, GOLDEN[seed])


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    emulated_train.install(monkeypatch)
    monkeypatch.setattr(boff, "_OFFLINE", {})


def product_training_set(frames, features, label_feature, entity_rows, entity_timestamp_column, with_indexes):
    for name, (entities, ts, frame) in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)
    vector = boff.FeatureVector("v", features, label_feature=label_feature)
    return boff.get_offline_features(vector, entity_rows, entity_timestamp_column, with_indexes=with_indexes).to_dataframe()


@pytest.mark.parametrize("seed", range(gen.N_GOLDEN))
def test_host_layer_equals_the_real_reference(seed):
    want = GOLDEN[seed]
    got = gen.run(product_training_set, seed)
    if isinstance(want, dict):
        assert got == want
    else:
        pd.testing.assert_frame_equal(got, want, check_exact=True)


def _fraud(seed=3, label_dtype="float32", nan_share=0.3, label_in="labels", n=300):
    """transactions (the spine, float64 aggregation columns), events and labels keyed alike"""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 40, size=n)
    when = pd.to_datetime(rng.choice(10**6, size=n, replace=False) * 10**9)
    txn = pd.DataFrame({"card": keys, "when": when, "amount": rng.normal(size=n).astype(np.float32),
                        "amount_sum_1h": rng.normal(size=n), "amount_max_1h": rng.normal(size=n)})
    m = n // 2
    events = pd.DataFrame({"card": rng.integers(0, 40, size=m), "when": pd.to_datetime(rng.choice(10**6, size=m, replace=False) * 10**9),
                           "clicks": rng.normal(size=m).astype(np.float32)})
    lab = rng.normal(size=n).astype(label_dtype) if label_dtype.startswith("float") else rng.integers(0, 2, size=n).astype(label_dtype)
    if label_dtype.startswith("float"):
        lab[rng.random(n) < nan_share] = np.nan
    labels = pd.DataFrame({"card": keys, "when": when, "label": lab})
    frames = {"txn": (["card"], "when", txn), "events": (["card"], "when", events), "labels": (["card"], "when", labels)}
    if label_in == "txn":
        txn["label"] = lab
        del frames["labels"]
    return frames


@pytest.mark.parametrize("label_dtype", ["float32", "float64", "int32", "bool"])
@pytest.mark.parametrize("label_in", ["labels", "txn"])
def test_entity_less_fraud_vector_equals_the_oracle(label_dtype, label_in):
    from tests.golden.diff_training_set import oracle_training_set

    frames = _fraud(label_dtype=label_dtype, label_in=label_in)
    args = dict(frames=frames, features=["txn.*", "events.clicks"], label_feature=f"{label_in}.label", entity_rows=None,
                entity_timestamp_column=None, with_indexes=False)
    got = product_training_set(**args)
    pd.testing.assert_frame_equal(got, oracle_training_set(**args), check_exact=True)
    assert "label" in got.columns and "amount_sum_1h" in got.columns and got["amount_sum_1h"].dtype == np.float64


@pytest.mark.parametrize("share", [0.0, 1.0])
def test_labels_that_drop_no_row_and_every_row(share):
    from tests.golden.diff_training_set import oracle_training_set

    args = dict(frames=_fraud(nan_share=share), features=["txn.amount"], label_feature="labels.label", entity_rows=None,
                entity_timestamp_column=None, with_indexes=True)
    got = product_training_set(**args)
    pd.testing.assert_frame_equal(got, oracle_training_set(**args), check_exact=True)
    assert len(got) == (300 if share == 0.0 else 0)


def test_float64_features_pass_through_bit_for_bit():
    fsets, frames, feats, entity, ts = fx.workload(4, n_sets=1)
    special = np.array([np.nan, -0.0, np.inf, -np.inf, 5e-324, 1.5, np.float64(np.uint64(0x7FF8000000000123).view(np.float64))])
    frame = frames["fs0"][2]
    frame["agg"] = special[np.arange(len(frame)) % len(special)]
    boff.register_offline_frame(fsets[0], frame)
    got = boff.get_offline_features(boff.FeatureVector("v", ["fs0.agg"]), entity, ts).to_dataframe()
    order = np.argsort(entity["t"].to_numpy(), kind="stable")
    keys = frame["id"].to_numpy()
    want = []
    for r in order:  # the last row of the key at or before the entity time, NaN bits where there is none
        hit = np.flatnonzero((keys == entity["id"].iloc[r]) & (frame["when"].to_numpy() <= entity["t"].iloc[r]))
        hit = hit[np.argsort(frame["when"].to_numpy()[hit], kind="stable")]
        want.append(frame["agg"].to_numpy()[hit[-1]] if len(hit) else np.uint64(0x7FF8000000000000).view(np.float64))
    assert got["agg"].dtype == np.float64
    np.testing.assert_array_equal(got["agg"].to_numpy().view(np.uint64), np.array(want, np.float64).view(np.uint64))


def test_entity_timestamp_column_without_entity_rows_raises_the_reference_error():
    frames = _fraud()
    for name, (entities, ts, frame) in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)
    with pytest.raises(MLRunInvalidArgumentError, match="^entity_timestamp_column param can not be specified without entity_rows param$"):
        boff.get_offline_features(boff.FeatureVector("v", ["txn.amount"]), None, "when")


def _registered():
    frames = _fraud()
    for name, (entities, ts, frame) in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)
    txn = frames["txn"][2]
    boff.register_offline_frame(bingest.FeatureSet("big", entities=["card"], timestamp_key="when"), txn.assign(n=np.arange(len(txn))))
    boff.register_offline_frame(bingest.FeatureSet("other", entities=["user"], timestamp_key="when"), txn.rename(columns={"card": "user"}))
    return frames


@pytest.mark.parametrize("vector, kwargs, match", [
    (dict(features=["big.n"]), {}, "int64"),
    (dict(features=["txn.amount"], label_feature="big.n"), {}, "int64"),
    (dict(features=["txn.amount", "other.amount"]), {}, "relations"),
    (dict(features=["txn.amount"], relations={"x": "y"}), {}, "relations"),
    (dict(features=["txn.amount"], join_graph=object()), {}, "join graphs"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(start_time="2020-01-01"), "start_time"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(timestamp_for_filtering="when"), "start_time"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(query="amount > 0"), "query"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(order_by="amount"), "query"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(additional_filters=[]), "query"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(target=object()), "targets"),
    (dict(features=["txn.amount"], label_feature="labels.label"), dict(drop_columns=["amount"]), "drop_columns"),
])
def test_refusals(vector, kwargs, match):
    _registered()
    with pytest.raises(LoweringError, match=match):
        boff.get_offline_features(boff.FeatureVector("v", **vector), None, **kwargs)


def test_int64_features_stay_refused_with_entity_rows_and_a_label():
    frames = _registered()
    entity = frames["txn"][2][["card", "when"]].rename(columns={"when": "t"})
    with pytest.raises(LoweringError, match="int64"):
        boff.get_offline_features(boff.FeatureVector("v", ["txn.amount", "big.n"], label_feature="labels.label"), entity, "t")
