"""Offline retrieval on CPU: the oracle against the goldens of the REAL LocalFeatureMerger.merge; the product's host layer
(naming, aliases, dtype rules, row order, refusals) over a numpy emulation of the b2s_pit join (tests/emulated_pit.py); and
the radix sort's digit and sign handling restated in numpy.  The CUDA kernels are tests/test_gpu_offline.py."""

import lzma
import os
import pickle

import numpy as np
import pandas as pd
import pytest

from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from mlrun_b200.lowering import LoweringError
from oracle import offline as oo
from tests import emulated_pit
from tests import offline_fixtures as fx
from tests.golden import gen_offline

GOLDEN = pickle.load(lzma.open(gen_offline.GOLDEN))


@pytest.mark.parametrize("seed", range(gen_offline.N_GOLDEN))
def test_oracle_merge_equals_the_real_reference(seed):
    want = GOLDEN[seed]
    got = gen_offline.run_merge(oo.merge, seed)
    assert isinstance(got, dict) == isinstance(want, dict)
    if isinstance(want, dict):
        assert got == want
        return
    pd.testing.assert_frame_equal(got[0], want[0], check_exact=True)
    assert got[1:] == want[1:]


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    emulated_pit.install(monkeypatch)
    monkeypatch.setattr(boff, "_OFFLINE", {})


def _check(fsets, frames, feats, entity, ts, with_indexes=False):
    fx.register(fsets, frames)
    want = oo.get_offline_features(frames, feats, entity, ts, with_indexes=with_indexes)
    got = boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts, with_indexes=with_indexes).to_dataframe()
    pd.testing.assert_frame_equal(got, want, check_exact=True)
    return got


CASES = {
    "int64": dict(), "string": dict(key_kind="str"), "pairs": dict(key_kind="pair"), "four_sets_ms": dict(n_sets=4, unit="ms"),
    "exact_last": dict(exact_sets=(1,)), "exact_then_asof": dict(n_sets=3, exact_sets=(1,)), "exact_first": dict(exact_sets=(0,)),
    "all_unknown": dict(unknown=1.0), "one_row": dict(n_entity=1, n_rows=1, n_keys=1, unknown=0.0),
}


@pytest.mark.parametrize("with_indexes", [False, True])
@pytest.mark.parametrize("case", sorted(CASES))
def test_host_layer_equals_the_oracle(case, with_indexes):
    _check(*fx.workload(13, **CASES[case]), with_indexes=with_indexes)


def test_aliases_and_star_name_the_columns_like_the_reference():
    got = _check(*fx.workload(2, n_sets=2))
    assert list(got.columns)[:3] == ["label", "weight", "first0"] and "s1x0" in got.columns and "id" not in got.columns


def test_int_columns_keep_their_dtype_when_every_row_matches():
    fsets, frames, feats, entity, ts = fx.workload(5, n_sets=1, unknown=0.0)
    _keys, _t, frame = frames["fs0"]
    first = frame.groupby("id", as_index=False).head(1).copy()
    first["when"] = pd.Timestamp("1900-01-01").as_unit("ns") - pd.to_timedelta(np.arange(len(first)), unit="s")
    frames["fs0"] = (["id"], "when", pd.concat([frame, first], ignore_index=True))
    entity["t"] = frame["when"].max() + pd.to_timedelta(np.arange(len(entity)) + 1, unit="s")
    got = _check(fsets, frames, feats, entity, ts)
    assert (str(got["s0count"].dtype), str(got["s0small"].dtype), str(got["s0flag"].dtype)) == ("int32", "int8", "bool")


def test_rows_come_back_in_entity_time_order_with_ties_in_input_order():
    fsets, frames, feats, entity, ts = fx.workload(8, ties=True, n_entity=50)
    fx.register(fsets, frames)
    got = boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts).to_dataframe()
    order = np.argsort(entity["t"].to_numpy(), kind="stable")
    np.testing.assert_array_equal(got["label"].to_numpy(), entity["label"].to_numpy()[order])


def test_nat_entity_time_raises_the_reference_error():
    fsets, frames, feats, entity, ts = fx.workload(2)
    fx.register(fsets, frames)
    entity.loc[0, "t"] = pd.NaT
    with pytest.raises(ValueError, match="^Merge keys contain null values on left side$"):
        boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts)


@pytest.mark.parametrize("kwargs", [dict(engine="dask"), dict(start_time="2020-01-01"), dict(end_time="2020-01-01"),
                                    dict(query="x > 1"), dict(order_by="x"), dict(target=object())])
def test_unlowered_arguments_are_refused(kwargs):
    fsets, frames, feats, entity, ts = fx.workload(2)
    fx.register(fsets, frames)
    with pytest.raises(LoweringError):
        boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts, **kwargs)


def test_refusals_of_keys_dtypes_and_relations():
    fsets, frames, feats, entity, ts = fx.workload(2, n_sets=1)
    frame = frames["fs0"][2]
    with pytest.raises(LoweringError, match="keys"):
        boff.register_offline_frame(bingest.FeatureSet("f", entities=["k"], timestamp_key="when"),
                                    frame.assign(k=frame["id"].astype(np.float64)))
    boff.register_offline_frame(bingest.FeatureSet("g", entities=["id"], timestamp_key="when"), frame.assign(big=np.arange(len(frame))))
    with pytest.raises(LoweringError, match="int64"):
        boff.get_offline_features(boff.FeatureVector("v", ["g.big"]), entity, ts)
    boff.register_offline_frame(bingest.FeatureSet("h", entities=["other"], timestamp_key="when"), frame.assign(other=frame["id"]))
    with pytest.raises(LoweringError, match="relations"):
        boff.get_offline_features(boff.FeatureVector("v", ["h.s0x0"]), entity, ts)
    with pytest.raises(LoweringError, match="several rows per key"):
        boff.get_offline_features(boff.FeatureVector("v", ["g.s0x0"]), entity, None)


# ---- the radix sort of b2s_pit.cu restated: 8 passes of 8-bit digits over sign-flipped keys, tiles ranked in order ----
def _radix_argsort(keys, tile=4096):
    keys = np.asarray(keys, np.int64)
    flipped = keys.view(np.uint64) ^ np.uint64(1 << 63)
    order = np.arange(len(keys))
    n_blocks = (len(keys) + tile - 1) // tile
    for shift in range(0, 64, 8):
        digit = ((flipped[order] >> np.uint64(shift)) & np.uint64(0xFF)).astype(np.int64)
        block = np.arange(len(keys)) // tile
        hist = np.zeros((256, n_blocks), np.int64)
        np.add.at(hist, (digit, block), 1)
        base = (np.cumsum(hist.ravel()) - hist.ravel()).reshape(256, n_blocks)  # digit-major exclusive scan
        out = np.empty_like(order)
        nxt = base.copy()
        for e in range(len(keys)):  # each block writes its items in input order
            d, b = digit[e], block[e]
            out[nxt[d, b]] = order[e]
            nxt[d, b] += 1
        order = out
    return order


@pytest.mark.parametrize("kind", ["all_equal", "reversed", "random", "extremes"])
def test_radix_digits_and_sign_flip_give_a_stable_argsort(kind):
    rng = np.random.default_rng(4)
    n = 9000
    keys = {"all_equal": np.full(n, -3, np.int64), "reversed": np.arange(n, 0, -1, dtype=np.int64) - n // 2,
            "random": rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=n, dtype=np.int64),
            "extremes": rng.choice(np.array([np.iinfo(np.int64).min, -1, 0, 1, np.iinfo(np.int64).max], np.int64), size=n)}[kind]
    np.testing.assert_array_equal(_radix_argsort(keys), np.argsort(keys, kind="stable"))
