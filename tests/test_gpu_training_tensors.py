"""Training sets as device tensors on the H100 (b2s_pit_train_pack, `get_offline_tensors`) against the frame
`get_offline_features(...).to_dataframe()` builds from the same registered frames: the matrix is the frame's feature
columns `.to_numpy(dtype)`, bit for bit where finite (-0.0 kept) and NaN where NaN, the label its label column, `order`
the join's order.  Covers F from 1 to 512 over 1- to 8-byte sources, kept rows at the tile edges and warp lanes of the
keep kernel, 0 to 2 Mi + 3 kept rows, labels of every kind and place, both dtypes, the zero-copy hand-over to torch, the
arrays' lifetime, the launch count, and the 64 golden workloads of the REAL reference."""

import gc
import lzma
import pickle

import numpy as np
import pandas as pd
import pytest
import torch

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from tests import pit_reference as ref
from tests.golden import gen_training_set as gen
from tests.test_training_tensors_cpu import feature_columns, label_values, same_values

pytestmark = pytest.mark.gpu
GOLDEN = pickle.load(lzma.open(gen.GOLDEN))
BASE = 1_600_000_000 * 10**9
SPINE_DTYPES = ["int8", "uint8", "int16", "uint16", "int32", "bool", "float32", "float64"]
SET_DTYPES = ["float32", "float64", "int32", "float64", "int16", "bool"]


@pytest.fixture(autouse=True)
def _fresh():
    nat.init()
    boff._OFFLINE.clear()
    yield
    boff._OFFLINE.clear()


def column(rng, dtype, n):
    """values that stress the conversion: ints past 2^24, float64 that float32 rounds, -0.0 and NaN"""
    if dtype == "bool":
        return rng.random(n) < 0.5
    if dtype.startswith("float"):
        v = rng.normal(size=n) * 10.0 ** rng.integers(-3, 30, size=n)
        v[rng.random(n) < 0.05] = -0.0
        v[rng.random(n) < 0.05] = np.nan
        return v.astype(dtype)
    info = np.iinfo(dtype)
    return rng.integers(info.min, info.max, size=n, endpoint=True).astype(dtype)


def fraud(n, n_spine, n_set, seed=0, label=None, nan_share=0.3, keep=None):
    """an entity-less vector: the spine `txn` (n rows, increasing timestamps, so the join keeps input order) with n_spine
    features of every spine dtype, a set `ev` of n_set features of 4- and 8-byte outputs joined as-of (some rows miss),
    and optionally a label: ("set", dtype) on `lab`, ("spine", dtype) on the spine; `keep` replaces the label's NaN rows"""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, max(n // 4, 1), size=n)
    txn = {"card": keys, "when": pd.to_datetime(np.arange(n, dtype=np.int64) * 10**9 + BASE)}
    for j in range(n_spine):
        txn[f"s{j}"] = column(rng, SPINE_DTYPES[j % len(SPINE_DTYPES)], n)
    m = max(n // 2, 1)
    ev = {"card": rng.integers(0, max(n // 4, 1), size=m), "when": pd.to_datetime(rng.permutation(m).astype(np.int64) * 2 * 10**9 + BASE + 10**9)}
    for j in range(n_set):
        ev[f"e{j}"] = column(rng, SET_DTYPES[j % len(SET_DTYPES)], m)
    frames = {"txn": txn, "ev": ev}
    label_feature = None
    if label is not None:
        place, dtype = label
        lab = column(rng, dtype, n)
        if dtype.startswith("float"):
            lab = np.where(np.isnan(lab), 0.5, lab).astype(dtype)
            lab[rng.random(n) < nan_share] = np.nan
            if keep is not None:
                lab = np.where(keep, np.arange(n), np.nan).astype(dtype)
        if place == "spine":
            txn["label"] = lab
            label_feature = "txn.label"
        else:
            frames["lab"] = {"card": keys, "when": txn["when"], "label": lab}
            label_feature = "lab.label"
    for name, cols in frames.items():
        boff.register_offline_frame(bingest.FeatureSet(name, entities=["card"], timestamp_key="when"), pd.DataFrame(cols))
    features = ["txn.*"] if n_spine else []
    features += ["ev.*"] if n_set else []
    return boff.FeatureVector("v", features, label_feature=label_feature)


def check(vector, dtype, entity_rows=None, entity_ts=None):
    """the tensors against the frame; -> the tensors"""
    before = nat.launch_count()
    t = boff.get_offline_tensors(vector, entity_rows, entity_ts, dtype=dtype)
    launched = nat.launch_count() - before
    frame = boff.get_offline_features(vector, entity_rows, entity_ts).to_dataframe()
    cols = feature_columns(frame)
    assert t.columns == cols and t.rows == len(frame)
    assert t.features.shape == (len(frame), len(cols)) and t.features.dtype == np.dtype(dtype)
    with np.errstate(over="ignore"):
        same_values(t.features.numpy(), frame[cols].to_numpy(dtype) if cols else np.zeros((len(frame), 0), dtype))
    if "label" in frame.columns:
        same_values(t.label.numpy(), label_values(frame["label"], t.label.dtype))
    else:
        assert t.label is None
    assert t.order.shape == (len(frame),)
    if t.stats["rows"]:
        # without entity rows the first set is the spine: its columns are entity columns, the other sets are joined
        named = [f.split(".")[0] for f in vector.features + ([vector.label_feature] if vector.label_feature else [])]
        spine = named[0] if entity_rows is None else None
        prefix = {"txn": "s", "ev": "e"}.get(spine)
        n_cols = sum(1 for c in cols if prefix and c.startswith(prefix)) + (spine is not None and vector.label_feature == f"{spine}.label")
        n_sets = len(set(named) - {spine})
        assert t.stats["kernels"] == 24 + max(1, n_sets, -(-n_cols // 64)) + 2 + 1 == launched
    return t


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("f", [1, 31, 32, 33, 64, 65, 257, 512])
def test_feature_counts(f, dtype):
    n_spine = f // 2
    check(fraud(3000, n_spine, f - n_spine, seed=f, label=("set", "float32")), dtype)


@pytest.mark.parametrize("pattern", ref.LABEL_PATTERNS)
def test_kept_rows_at_tile_edges_and_lanes(pattern):
    n = 3 * ref.TILE + 5
    keep = ref.keep_pattern(n, pattern, np.random.default_rng(1))
    t = check(fraud(n, 9, 40, seed=2, label=("spine", "float32"), keep=keep), "float32")
    np.testing.assert_array_equal(t.order.numpy(), np.flatnonzero(keep))


@pytest.mark.parametrize("n", [1, 2, (1 << 20) - 1, (1 << 20) + 1, (1 << 21) + 3])
def test_row_counts(n):
    t = check(fraud(n, 3, 5, seed=n % 97, label=("set", "float64"), nan_share=0.0), "float32")
    assert t.rows == n


def test_no_entity_rows_gives_empty_arrays():
    vector = fraud(100, 4, 6, label=("set", "int32"))
    entity = pd.DataFrame({"card": np.zeros(0, np.int64), "when": pd.to_datetime(np.zeros(0, np.int64))})
    t = boff.get_offline_tensors(boff.FeatureVector("v", ["ev.*"], label_feature="lab.label"), entity, "when")
    assert t.features.shape == (0, 6) and t.label.shape == (0,) and t.order.shape == (0,) and t.rows == 0
    assert torch.as_tensor(t.features, device="cuda").shape == (0, 6) and torch.from_dlpack(t.label).shape == (0,)
    assert vector.label_feature == "lab.label"


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("label", [None, ("set", "float32"), ("set", "float64"), ("set", "int32"), ("set", "bool"),
                                   ("spine", "float32"), ("spine", "float64"), ("spine", "int16"), ("spine", "uint8"),
                                   ("spine", "bool")])
def test_labels(label, dtype):
    t = check(fraud(2500, 8, 12, seed=3, label=label), dtype)
    if label is not None:
        want = {"float32": np.float32, "float64": np.float64, "bool": np.bool_}.get(label[1], np.int64)
        assert t.label.dtype == want


def test_entity_rows_and_order():
    vector = fraud(4000, 0, 20, seed=4, label=("set", "float32"))
    rng = np.random.default_rng(5)
    entity = pd.DataFrame({"card": rng.integers(0, 1200, size=3000), "t": pd.to_datetime(rng.permutation(3000) * 10**9 + BASE + 7),
                           "w": rng.normal(size=3000)})
    t = check(vector, "float64", entity, "t")
    frame = boff.get_offline_features(vector, entity, "t").to_dataframe()
    np.testing.assert_array_equal(entity["w"].to_numpy()[t.order.numpy()], frame["w"].to_numpy())


def test_zero_copy_hand_over_and_lifetime():
    gc.collect()
    live = nat.darray_live()
    vector = fraud(5000, 6, 10, seed=6, label=("set", "float32"))
    t = boff.get_offline_tensors(vector)
    want = t.features.numpy()
    assert nat.darray_live() == live + 3
    a = torch.as_tensor(t.features, device="cuda")
    b = torch.from_dlpack(t.features)
    y = torch.from_dlpack(t.label)
    assert a.data_ptr() == b.data_ptr() == t.features.ptr and y.data_ptr() == t.label.ptr
    assert a.shape == b.shape == want.shape and a.is_contiguous() and b.dtype == torch.float32
    del t
    gc.collect()
    assert nat.darray_live() == live + 2  # the order had no other owner; the matrix and label are held by torch
    torch.cuda.synchronize()
    np.testing.assert_array_equal(b.cpu().numpy().view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(a.cpu().numpy().view(np.uint32), want.view(np.uint32))
    del a
    gc.collect()
    assert nat.darray_live() == live + 2  # the DLPack consumer still holds the matrix
    same_values((b * 1).cpu().numpy(), want)  # computed on: torch's own NaN bits differ, the values do not
    del b, y
    gc.collect()
    assert nat.darray_live() == live


def test_an_unconsumed_capsule_frees_its_reference():
    gc.collect()
    live = nat.darray_live()
    t = boff.get_offline_tensors(fraud(500, 2, 3, seed=7))
    capsule = t.features.__dlpack__()
    del t
    gc.collect()
    assert nat.darray_live() == live + 1
    del capsule
    gc.collect()
    assert nat.darray_live() == live


@pytest.mark.parametrize("seed", range(gen.N_GOLDEN))
def test_golden_workloads(seed):
    want = GOLDEN[seed]

    def tensors(frames, features, label_feature, entity_rows, entity_timestamp_column, with_indexes):
        for name, (entities, ts, frame) in frames.items():
            boff.register_offline_frame(bingest.FeatureSet(name, entities=entities, timestamp_key=ts), frame)
        vector = boff.FeatureVector("v", features, label_feature=label_feature)
        return [boff.get_offline_tensors(vector, entity_rows, entity_timestamp_column, dtype=d, with_indexes=with_indexes)
                for d in ("float32", "float64")]

    got = gen.run(tensors, seed)
    if isinstance(want, dict):
        assert got == want
        return
    cols = feature_columns(want)
    for t, dtype in zip(got, ("float32", "float64")):
        assert t.columns == cols and t.rows == len(want)
        with np.errstate(over="ignore"):
            same_values(t.features.numpy(), want[cols].to_numpy(dtype) if cols else np.zeros((len(want), 0), dtype))
        if "label" in want.columns:
            same_values(t.label.numpy(), label_values(want["label"], t.label.dtype))
        else:
            assert t.label is None
