"""Point-in-time training sets on the H100 (b2s_pit.cu) against the oracle's restatement of the local engine's merge:
values bit for bit, NaN / NaT positions, dtypes, column names and row order."""

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from oracle import offline as oo
from tests import offline_fixtures as fx
from tests import table_hash

pytestmark = pytest.mark.gpu


def _check(fsets, frames, feats, entity, ts, with_indexes=False):
    fx.register(fsets, frames)
    want = oo.get_offline_features(frames, feats, entity, ts, with_indexes=with_indexes)
    got = boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts, with_indexes=with_indexes).to_dataframe()
    pd.testing.assert_frame_equal(got, want, check_exact=True)
    return got


CASES = {
    "one_row": dict(n_entity=1, n_rows=1, n_keys=1, unknown=0.0),
    "int64_extremes": dict(),
    "string_keys": dict(key_kind="str"),
    "int32_pairs": dict(key_kind="pair"),
    "exact_key_set": dict(n_sets=3, exact_sets=(1,)),
    "four_sets_us": dict(n_sets=4, unit="us"),
    "one_set_s": dict(n_sets=1, unit="s"),
    "all_unknown": dict(unknown=1.0),
    "dense_keys": dict(n_keys=4, n_rows=3000, n_entity=5000, unknown=0.0),
}


@pytest.mark.parametrize("with_indexes", [False, True])
@pytest.mark.parametrize("case", sorted(CASES))
def test_offline_features_equal_the_oracle(case, with_indexes):
    _check(*fx.workload(7, **CASES[case]), with_indexes=with_indexes)


def test_offline_features_two_mi_entity_rows():
    _check(*fx.workload(11, n_sets=2, n_rows=1 << 20, n_keys=1 << 16, n_entity=2 << 20, n_float=4))


def _no_miss_workload():
    fsets, frames, feats, entity, ts = fx.workload(5, n_sets=2, unknown=0.0, before_1970=True)
    latest = max(f[2]["when"].max() for f in frames.values())
    for name, (keys, _t, frame) in frames.items():  # every key has a row at the earliest time
        first = frame.groupby("id", as_index=False).head(1).copy()
        first["when"] = pd.Timestamp("1900-01-01").as_unit("ns") - pd.to_timedelta(np.arange(len(first)), unit="s")
        frames[name] = (keys, "when", pd.concat([frame, first], ignore_index=True))
    entity["t"] = latest + pd.to_timedelta(np.arange(len(entity)) + 1, unit="s")
    return fsets, frames, feats, entity, ts


def test_int_features_stay_int_without_a_miss_and_become_float64_with_one():
    got = _check(*_no_miss_workload())
    assert str(got["s0count"].dtype) == "int32" and str(got["s0small"].dtype) == "int8" and str(got["s0flag"].dtype) == "bool"
    got = _check(*fx.workload(5, unknown=1.0))
    assert got["s0count"].isna().all() and str(got["s0count"].dtype) == "float64"


def test_probe_run_wraps_past_the_last_slot():
    rng = np.random.default_rng(3)
    keys = table_hash.keys_with_home_slots([15, 15, 15, 14], 16, rng)  # 4 keys -> 16 slots; the last two wrap to 0, 1
    n = 64
    frame = pd.DataFrame({"id": np.tile(keys, n // 4), "when": pd.to_datetime(np.arange(n) * 10**9),
                          "v": rng.normal(size=n).astype(np.float32)})
    fs = bingest.FeatureSet("wrap", entities=["id"], timestamp_key="when")
    entity = pd.DataFrame({"id": np.concatenate([keys, keys + 1]), "t": pd.to_datetime((np.arange(8) * 7 + 3) * 10**9)})
    src = boff.register_offline_frame(fs, frame)
    assert src.index.n_keys == 4 and table_hash.capacity(4) == 16
    got = _check([fs], {"wrap": (["id"], "when", frame)}, ["wrap.v"], entity, "t")
    assert got["v"].notna().sum() == 4  # the four known keys, each with rows before its time


def test_equal_entity_times_match_as_an_ordered_set():
    """pandas' unstable sort may order rows of equal timestamp differently: compare those rows as a set"""
    fsets, frames, feats, entity, ts = fx.workload(9, ties=True, n_entity=400)
    for name, (k, t, frame) in frames.items():  # keep (key, timestamp) pairs unique in the feature sets
        frames[name] = (k, t, frame.drop_duplicates(subset=["id", "when"], keep="first").reset_index(drop=True))
    fx.register(fsets, frames)
    want = oo.get_offline_features(frames, feats, entity, ts, with_indexes=True).reset_index()
    got = boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts, with_indexes=True).to_dataframe().reset_index()
    assert list(got.columns) == list(want.columns) and (got.dtypes == want.dtypes).all()
    assert (got["t"].to_numpy() == np.sort(entity["t"].to_numpy(), kind="stable")).all()
    key = list(got.columns)
    pd.testing.assert_frame_equal(got.sort_values(key, ignore_index=True), want.sort_values(key, ignore_index=True), check_exact=True)


def test_nat_entity_time_raises_like_pandas():
    fsets, frames, feats, entity, ts = fx.workload(2)
    fx.register(fsets, frames)
    entity.loc[3, "t"] = pd.NaT
    with pytest.raises(ValueError, match="Merge keys contain null values on left side"):
        oo.get_offline_features(frames, feats, entity, ts)
    with pytest.raises(ValueError, match="Merge keys contain null values on left side"):
        boff.get_offline_features(boff.FeatureVector("v", feats), entity, ts)


@pytest.mark.parametrize("kind", ["all_equal", "reversed", "random", "extremes"])
def test_radix_sort_is_a_stable_argsort(kind):
    rng = np.random.default_rng(1)
    n = 300_001
    ts = {"all_equal": np.full(n, -5, np.int64), "reversed": np.arange(n, 0, -1, dtype=np.int64) * -(10**9),
          "random": rng.integers(-(2**62), 2**62, size=n, dtype=np.int64),
          "extremes": rng.choice(np.array([np.iinfo(np.int64).min, -1, 0, 1, np.iinfo(np.int64).max], np.int64), size=n)}[kind]
    order, _sets, _cols, _miss = boff.pit_join(ts, [], [])
    np.testing.assert_array_equal(order, np.argsort(ts, kind="stable"))


def test_device_resident_join_equals_the_host_run():
    fsets, frames, _feats, entity, _ts = fx.workload(4, n_sets=2, n_entity=5000)
    fx.register(fsets, frames)
    ts = entity["t"].to_numpy().view(np.int64)
    keys = entity["id"].to_numpy().astype(np.int64)
    srcs = [boff._OFFLINE[f.name] for f in fsets]
    outs = [[(src.features[c][0], np.float32, boff._NAN32) for c in ("s%dx0" % i, "s%dx1" % i)] for i, src in enumerate(srcs)]
    weight = entity["weight"].to_numpy()
    h_order, h_sets, h_cols, h_miss = boff.pit_join(ts, [(s.index, keys, 1, o) for s, o in zip(srcs, outs)], [weight])
    n = len(ts)
    bufs = []

    def dev(arr=None, nbytes=None):
        b = nat.DeviceBuffer(nbytes if nbytes is not None else arr.nbytes)
        if arr is not None:
            b.upload(arr)
        bufs.append(b)
        return b

    d_ts, d_keys = dev(ts), dev(keys)
    d_outs = [[dev(nbytes=4 * n) for _ in o] for o in outs]
    d_tsout = [dev(nbytes=8 * n) for _ in srcs]
    d_found = [dev(nbytes=n) for _ in srcs]
    d_w, d_wo, d_order = dev(weight), dev(nbytes=weight.nbytes), dev(nbytes=8 * n)
    d_miss = dev(np.zeros(2, np.uint64))
    keep, c_sets = [], (nat.PitSet * 2)()
    for i, (s, o) in enumerate(zip(srcs, outs)):
        descs = (nat.PitOut * len(o))(*[nat.PitOut(w, 4, m, b.ptr) for (w, _dt, m), b in zip(o, d_outs[i])])
        keep.append(descs)
        c_sets[i] = nat.PitSet(s.index._h, d_keys.ptr, 1, len(o), descs, d_tsout[i].ptr, d_found[i].ptr)
    cols = (nat.PitCol * 1)(nat.PitCol(d_w.ptr, d_wo.ptr, weight.dtype.itemsize))
    nat.check(nat.load().b2s_pit_join_device(d_ts.ptr, n, c_sets, 2, cols, 1, d_order.ptr, d_miss.ptr, None))
    nat.check(nat.load().b2s_device_sync())
    np.testing.assert_array_equal(d_order.download(np.int64, n), h_order)
    np.testing.assert_array_equal(d_wo.download(weight.dtype, n), h_cols[0])
    np.testing.assert_array_equal(d_miss.download(np.uint64, 2), h_miss)
    for i in range(2):
        for b, h in zip(d_outs[i], h_sets[i][0]):
            np.testing.assert_array_equal(b.download(np.uint32, n), h.view(np.uint32))
        np.testing.assert_array_equal(d_tsout[i].download(np.int64, n), h_sets[i][1])
        np.testing.assert_array_equal(d_found[i].download(np.uint8, n).astype(bool), h_sets[i][2])


def test_exact_join_on_a_set_with_repeated_keys_is_refused_before_launch():
    fsets, frames, _f, entity, _ts = fx.workload(6, n_sets=1)
    fx.register(fsets, frames)
    src = boff._OFFLINE["fs0"]
    assert src.index.longest_run > 1
    with pytest.raises(nat.NativeError, match="exact-key join"):
        boff.pit_join(None, [(src.index, entity["id"].to_numpy(), 0, [])], [])
