"""Training sets as device tensors on CPU: `get_offline_tensors`' host layer -- the shared planner, the feature columns
and their order, the device descriptors of each column and of the label -- over a numpy emulation of b2s_pit_train_pack
(tests/emulated_tensors.py), against the frames the REAL BaseMerger.start produced (tests/golden/ref_training_set.pkl.xz):
the matrix is the frame's feature columns `.to_numpy(dtype)`, the label its label column.  And every refusal, which must
be `get_offline_features`' own.  The CUDA kernel is tests/test_gpu_training_tensors.py."""

import lzma
import pickle

import numpy as np
import pandas as pd
import pytest

from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from mlrun_b200.lowering import LoweringError
from tests import emulated_tensors
from tests.golden import gen_training_set as gen

GOLDEN = pickle.load(lzma.open(gen.GOLDEN))
NOT_FEATURES = {"label", "t", "w", "id", "a", "b"}  # the label, the entity frame's own columns and the keys


def feature_columns(frame):
    """the columns of a golden frame that are features: not the label, an entity column, a key or a timestamp"""
    return [c for c in frame.columns if c not in NOT_FEATURES and not c.startswith("when")]


def same_values(got, want):
    """equal bits where the reference is not NaN (-0.0 kept), NaN where it is"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    if want.dtype.kind == "f":
        nan = np.isnan(want)
        np.testing.assert_array_equal(np.isnan(got), nan)
        got, want = got[~nan], want[~nan]
        bits = np.uint32 if want.dtype == np.float32 else np.uint64
        np.testing.assert_array_equal(got.view(bits), want.view(bits))
    else:
        np.testing.assert_array_equal(got, want)


def label_values(column, got_dtype):
    """the frame's label column as the label vector holds it"""
    values = column.to_numpy()
    if got_dtype == np.bool_:
        return values.astype(bool)
    if got_dtype == np.int64:
        return values.astype(np.int64)
    return values


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    emulated_tensors.install(monkeypatch)
    monkeypatch.setattr(boff, "_OFFLINE", {})


def register(frames):
    for name, (entities, ts, frame) in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)


def tensors_and_frame(dtype, frames, features, label_feature, entity_rows, entity_timestamp_column, with_indexes):
    register(frames)
    vector = boff.FeatureVector("v", features, label_feature=label_feature)
    t = boff.get_offline_tensors(vector, entity_rows, entity_timestamp_column, dtype=dtype, with_indexes=with_indexes)
    return t, boff.get_offline_features(vector, entity_rows, entity_timestamp_column, with_indexes=with_indexes).to_dataframe()


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("seed", range(gen.N_GOLDEN))
def test_golden_workloads(seed, dtype):
    want = GOLDEN[seed]
    with np.errstate(over="ignore"):  # float64 aggregations past float32's range become inf, as in the frame's to_numpy
        got = gen.run(lambda **kw: tensors_and_frame(dtype, **kw), seed)
    if isinstance(want, dict):
        assert got == want
        return
    t, frame = got
    pd.testing.assert_frame_equal(frame, want, check_exact=True)
    cols = feature_columns(want)
    assert t.columns == cols
    assert t.rows == len(want)
    with np.errstate(over="ignore"):
        same_values(t.features, want[cols].to_numpy(dtype) if cols else np.zeros((len(want), 0), dtype))
    assert np.asarray(t.features).flags.c_contiguous
    if "label" in want.columns:
        # floats at their stored width; an int label is int64 even where the frame made it float64 (its NaN rows are gone)
        same_values(t.label, label_values(want["label"], np.asarray(t.label).dtype))
    else:
        assert t.label is None
    assert len(t.order) == len(want)


def _fraud(n=200, seed=5):
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 30, size=n)
    when = pd.to_datetime(rng.choice(10**6, size=n, replace=False) * 10**9)
    txn = pd.DataFrame({"card": keys, "when": when, "amount": rng.normal(size=n).astype(np.float32), "n": rng.integers(0, 9, size=n).astype(np.int16),
                        "flag": rng.random(n) < 0.5, "seen": when})
    labels = pd.DataFrame({"card": keys, "when": when, "label": rng.normal(size=n)})
    big = txn.assign(m=np.arange(n, dtype=np.int64))
    other = txn.rename(columns={"card": "user"})
    register({"txn": (["card"], "when", txn), "labels": (["card"], "when", labels), "big": (["card"], "when", big),
              "other": (["user"], "when", other)})
    return txn


REFUSALS = [
    (dict(features=["big.m"]), None, {}),
    (dict(features=["txn.amount"], label_feature="big.m"), None, {}),
    (dict(features=["txn.amount", "other.amount"]), None, {}),
    (dict(features=["txn.amount"], relations={"x": "y"}), None, {}),
    (dict(features=["txn.amount"], join_graph=object()), None, {}),
    (dict(features=["txn.amount"], label_feature="labels.label"), None, dict(start_time="2020-01-01")),
    (dict(features=["txn.amount"], label_feature="labels.label"), None, dict(timestamp_for_filtering="when")),
    (dict(features=["txn.amount"], label_feature="labels.label"), None, dict(query="amount > 0")),
    (dict(features=["txn.amount"], label_feature="labels.label"), None, dict(additional_filters=[])),
    (dict(features=["txn.amount"], label_feature="labels.label"), None, dict(engine="spark")),
    (dict(features=["txn.amount"]), None, dict(entity_timestamp_column="when")),
    (dict(features=["nope.amount"]), None, {}),
    (dict(features=["txn.nope"]), None, {}),
    (dict(features=["txn"]), None, {}),
    (dict(features=[]), None, {}),
    (dict(features=["txn.amount"], label_feature="label"), None, {}),
    (dict(features=["txn.amount"]), "string_keys", dict(entity_timestamp_column="when")),
    (dict(features=["txn.amount"]), "no_key", dict(entity_timestamp_column="when")),
    (dict(features=["txn.amount"]), "nat", dict(entity_timestamp_column="when")),
]


@pytest.mark.parametrize("i", range(len(REFUSALS)))
def test_refusals_are_get_offline_features_own(i):
    vector, entity, kwargs = REFUSALS[i]
    txn = _fraud()
    entity_rows = None
    if entity == "string_keys":
        entity_rows = pd.DataFrame({"card": [f"k{c}" for c in txn["card"]], "when": txn["when"]})
    elif entity == "no_key":
        entity_rows = pd.DataFrame({"when": txn["when"]})
    elif entity == "nat":
        entity_rows = pd.DataFrame({"card": txn["card"], "when": txn["when"].where(np.arange(len(txn)) != 3)})
    ts_col = kwargs.pop("entity_timestamp_column", None)
    outcomes = []
    for fn in (boff.get_offline_features, boff.get_offline_tensors):
        with pytest.raises(Exception) as info:
            fn(boff.FeatureVector("v", **vector), entity_rows, ts_col, **kwargs)
        outcomes.append((type(info.value), str(info.value)))
    assert outcomes[0] == outcomes[1]


@pytest.mark.parametrize("features, label, name", [
    (["txn.amount", "txn.seen"], "labels.label", "seen"),          # the spine's own column
    (["labels.label", "txn.seen as when_seen"], None, "when_seen"),  # a set's output, under its alias
    (["labels.*", "txn.seen"], None, "seen"),
])
def test_a_datetime_feature_is_refused_by_name(features, label, name):
    _fraud()
    with pytest.raises(LoweringError, match=f"feature {name!r} is a datetime64"):
        boff.get_offline_tensors(boff.FeatureVector("v", features, label_feature=label))
    boff.get_offline_features(boff.FeatureVector("v", features, label_feature=label)).to_dataframe()  # the frame has it


def test_the_label_may_not_be_a_datetime():
    _fraud()
    with pytest.raises(LoweringError, match="label 'txn.seen' is a datetime64"):
        boff.get_offline_tensors(boff.FeatureVector("v", ["labels.label"], label_feature="txn.seen"))


def test_dtype_is_float32_or_float64():
    _fraud()
    with pytest.raises(ValueError, match="float32 or float64"):
        boff.get_offline_tensors(boff.FeatureVector("v", ["txn.amount"]), dtype="int32")


def test_bool_int_and_aliases_in_vector_order():
    txn = _fraud()
    t = boff.get_offline_tensors(boff.FeatureVector("v", ["txn.flag as f", "txn.n", "txn.amount"], label_feature="labels.label"),
                                 dtype="float64")
    assert t.columns == ["f", "n", "amount"]
    order = np.asarray(t.order)
    want = np.stack([txn["flag"].to_numpy()[order], txn["n"].to_numpy()[order], txn["amount"].to_numpy()[order]], axis=1)
    same_values(t.features, want.astype(np.float64))
    assert np.asarray(t.label).dtype == np.float64


def test_the_planner_is_shared(monkeypatch):
    _fraud()
    seen = []
    real = boff._plan_query

    def planner(*a, **k):
        seen.append(a[0].name)
        return real(*a, **k)

    monkeypatch.setattr(boff, "_plan_query", planner)
    boff.get_offline_features(boff.FeatureVector("frame", ["txn.amount"]))
    boff.get_offline_tensors(boff.FeatureVector("tensors", ["txn.amount"]))
    assert seen == ["frame", "tensors"]

    def refuse(*a, **k):
        raise LoweringError("planned elsewhere")

    monkeypatch.setattr(boff, "_plan_query", refuse)
    for fn in (boff.get_offline_features, boff.get_offline_tensors):
        with pytest.raises(LoweringError, match="planned elsewhere"):
            fn(boff.FeatureVector("v", ["txn.amount"]))
