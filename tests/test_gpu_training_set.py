"""Training sets on the H100 (b2s_pit_train_*, b2s_pit.cu) against the oracle and the goldens of the REAL merger: values
bit for bit, dtypes, column names, row order and row labels; the label filter's compaction across tiles and copy-back
ranges; the device entry point on the library stream and a caller's; launches; refusals."""

import ctypes as C

import numpy as np
import pandas as pd
import pytest

from mlrun_b200 import _native as nat
from mlrun_b200.feature_store import ingest as bingest
from mlrun_b200.feature_store import offline as boff
from tests.golden import diff_training_set
from tests.golden import gen_training_set as gen
from tests.test_training_set_cpu import GOLDEN, _fraud, product_training_set

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh(monkeypatch):
    nat.init(0)
    monkeypatch.setattr(boff, "_OFFLINE", {})


def _same_as_oracle(**args):
    got = product_training_set(**args)
    pd.testing.assert_frame_equal(got, diff_training_set.oracle_training_set(**args), check_exact=True)
    return got


@pytest.mark.parametrize("seed", range(gen.N_GOLDEN))
def test_device_equals_the_real_reference(seed):
    want, got = GOLDEN[seed], gen.run(product_training_set, seed)
    if isinstance(want, dict):
        assert got == want
    else:
        pd.testing.assert_frame_equal(got, want, check_exact=True)


SPECIAL = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 5e-324, -2.2250738585072014e-308, 1.7976931348623157e308,
                    np.uint64(0x7FF8000000000123).view(np.float64), np.uint64(0xFFF0000000000001).view(np.float64)])


@pytest.mark.parametrize("entity_less", [True, False])
def test_float64_special_values_pass_bit_for_bit(entity_less):
    frames = _fraud(n=400)
    for _e, _t, f in frames.values():
        for name in [c for c in f.columns if c.startswith("amount_")] + (["clicks"] if "clicks" in f.columns else []):
            f[name] = SPECIAL[np.arange(len(f)) % len(SPECIAL)]
    entity = None if entity_less else frames["txn"][2][["card", "when"]].rename(columns={"when": "t"}).iloc[::3].reset_index(drop=True)
    got = _same_as_oracle(frames=frames, features=["txn.*", "events.clicks"], label_feature=None if not entity_less else "labels.label",
                          entity_rows=entity, entity_timestamp_column=None if entity_less else "t", with_indexes=False)
    assert got["amount_sum_1h"].dtype == np.float64 and got["clicks"].dtype == np.float64
    assert (got["clicks"].to_numpy().view(np.uint64) == np.uint64(0x7FF8000000000000)).any() or entity_less


# a present int or bool label is never NaN: only float labels drop rows by value
@pytest.mark.parametrize("label_dtype, drop", [(d, p) for d in ("float32", "float64") for p in ("none", "all_but_one", "all")]
                         + [(d, "none") for d in ("int32", "int8", "bool")])
@pytest.mark.parametrize("label_in", ["labels", "txn", "events_exact"])
def test_label_kinds_and_drop_shares(label_dtype, drop, label_in):
    rng = np.random.default_rng(5)
    frames = _fraud(label_dtype=label_dtype, n=500, label_in="txn" if label_in == "txn" else "labels")
    lname = {"labels": "labels", "txn": "txn", "events_exact": "cards"}[label_in]
    if label_in == "events_exact":  # an exact-key label set: one row per card, no timestamp key
        cards = np.unique(frames["txn"][2]["card"].to_numpy())
        lab = frames["labels"][2]["label"].to_numpy()[: len(cards)].copy()
        frames["cards"] = (["card"], None, pd.DataFrame({"card": cards, "label": lab}))
    frame = frames[lname][2]
    is_float = label_dtype.startswith("float")
    if is_float:
        v = frame["label"].to_numpy().copy()
        v[:] = rng.normal(size=len(v)).astype(v.dtype)
        if drop == "all":
            v[:] = np.nan
        elif drop == "all_but_one":
            v[1:] = np.nan
        frame["label"] = v
    got = _same_as_oracle(frames=frames, features=["txn.*", "events.clicks"], label_feature=f"{lname}.label", entity_rows=None,
                          entity_timestamp_column=None, with_indexes=False)
    if drop == "all":
        assert len(got) == 0
    if drop == "all_but_one" and lname == "txn":
        assert len(got) == 1


@pytest.mark.parametrize("n", [(1 << 20) - 1, 1 << 20, (1 << 20) + 1, 3 * (1 << 20) + 5])
def test_compaction_across_tiles_and_copy_back_ranges(n):
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 1 << 16, size=n)
    when = pd.to_datetime(rng.permutation(n).astype(np.int64) * 1000 + 10**15)
    txn = pd.DataFrame({"card": keys, "when": when, "amount": rng.normal(size=n).astype(np.float32), "amount_sum_1h": rng.normal(size=n)})
    m = n // 4
    events = pd.DataFrame({"card": rng.integers(0, 1 << 16, size=m), "when": pd.to_datetime(rng.permutation(m).astype(np.int64) * 4000 + 10**15),
                           "clicks": rng.normal(size=m).astype(np.float32)})
    lab = rng.normal(size=n)
    lab[rng.random(n) < 0.3] = np.nan
    labels = pd.DataFrame({"card": keys, "when": when, "label": lab})
    frames = {"txn": (["card"], "when", txn), "events": (["card"], "when", events), "labels": (["card"], "when", labels)}
    got = _same_as_oracle(frames=frames, features=["txn.*", "events.clicks"], label_feature="labels.label", entity_rows=None,
                          entity_timestamp_column=None, with_indexes=False)
    assert len(got) == int((~np.isnan(lab)).sum())


def test_spine_without_timestamp_key_and_with_tied_timestamps():
    rng = np.random.default_rng(2)
    n = 5000
    cards = rng.permutation(n)
    spine = pd.DataFrame({"card": cards, "risk": rng.normal(size=n), "label": rng.normal(size=n).astype(np.float32)})
    spine.loc[rng.random(n) < 0.4, "label"] = np.nan
    other = pd.DataFrame({"card": rng.permutation(n)[: n // 2], "score": rng.normal(size=n // 2).astype(np.float32)})
    frames = {"spine": (["card"], None, spine), "other": (["card"], None, other)}
    _same_as_oracle(frames=frames, features=["spine.*", "other.score"], label_feature="spine.label", entity_rows=None,
                    entity_timestamp_column=None, with_indexes=True)
    # ties: the spine keeps its input order among equal timestamps (pandas' quicksort need not: DESIGN §2)
    tied = pd.DataFrame({"card": rng.integers(0, 50, size=n), "when": pd.to_datetime(rng.integers(0, 20, size=n) * 10**9),
                         "pos": np.arange(n, dtype=np.int32)})
    feats = pd.DataFrame({"card": rng.integers(0, 50, size=300), "when": pd.to_datetime(rng.permutation(300) * 10**8),
                          "f": rng.normal(size=300).astype(np.float32)})
    frames = {"tied": (["card"], "when", tied), "feats": (["card"], "when", feats)}
    got = product_training_set(frames=frames, features=["tied.pos", "feats.f"], label_feature=None, entity_rows=None,
                               entity_timestamp_column=None, with_indexes=False)
    np.testing.assert_array_equal(got["pos"].to_numpy(), np.argsort(tied["when"].to_numpy(), kind="stable"))
    want = diff_training_set.oracle_training_set(frames=frames, features=["tied.pos", "feats.f"], label_feature=None, entity_rows=None,
                                                 entity_timestamp_column=None, with_indexes=False)
    pd.testing.assert_frame_equal(got.sort_values("pos", ignore_index=True), want.sort_values("pos", ignore_index=True), check_exact=True)


def test_string_spine_keys():
    frames = _fraud(n=2000)
    for _e, _t, f in frames.values():
        f["card"] = np.array([f"card-{k}" for k in f["card"]], dtype=object)
    for with_indexes in (False, True):
        _same_as_oracle(frames=frames, features=["txn.*", "events.clicks"], label_feature="labels.label", entity_rows=None,
                        entity_timestamp_column=None, with_indexes=with_indexes)


def test_aggregations_end_to_end():
    rng = np.random.default_rng(11)
    n = 20000
    raw = pd.DataFrame({"card": rng.integers(0, 300, size=n), "ts": pd.to_datetime(np.arange(n, dtype=np.int64) * 7 * 10**9),
                        "amount": (rng.random(n) * 500).astype(np.float32)})
    fset = bingest.FeatureSet("txn", entities=["card"], timestamp_key="ts")
    fset.add_aggregation("amount", ["count", "sum", "avg", "min", "max", "stddev"], ["1h", "6h"], "10m")
    ingested = fset.ingest(raw)
    assert ingested["amount_sum_1h"].dtype == np.float64
    labels = pd.DataFrame({"card": raw["card"], "ts": raw["ts"], "label": rng.normal(size=n)})
    labels.loc[rng.random(n) < 0.3, "label"] = np.nan
    lset = bingest.FeatureSet("labels", entities=["card"], timestamp_key="ts")
    boff.register_offline_frame(fset, ingested)
    boff.register_offline_frame(lset, labels)
    vector = boff.FeatureVector("v", ["txn.*"], label_feature="labels.label")
    got = boff.get_offline_features(vector).to_dataframe()
    frame = ingested.reset_index() if ingested.index.names[0] else ingested
    want = diff_training_set.oracle_training_set(frames={"txn": (["card"], "ts", frame), "labels": (["card"], "ts", labels)},
                                                 features=["txn.*"], label_feature="labels.label", entity_rows=None,
                                                 entity_timestamp_column=None, with_indexes=False)
    pd.testing.assert_frame_equal(got, want, check_exact=True)
    assert "amount_stddev_6h" in got.columns and len(got) == int(labels["label"].notna().sum())


# ------------------------------------------------------------------------------------------------ the C-ABI directly
def _setup(n=3000, seed=1):
    """two indexes (as-of with a float32 and a float64 column, exact-key with an int32 column) and entity columns"""
    rng = np.random.default_rng(seed)
    keys = rng.integers(0, 64, size=4 * n).astype(np.int64)
    ts = rng.permutation(4 * n).astype(np.int64) * 10
    f32, f64 = rng.normal(size=4 * n).astype(np.float32), rng.normal(size=4 * n)
    f64[rng.random(4 * n) < 0.3] = np.nan
    asof = boff.PitIndex(keys, ts, [f32, f64])
    exact = boff.PitIndex(np.arange(48, dtype=np.int64), np.zeros(48, np.int64), [np.arange(48, dtype=np.int32)])
    ekeys = rng.integers(0, 64, size=n).astype(np.int64)
    ets = rng.permutation(n).astype(np.int64) * 40
    col = rng.normal(size=n)
    return asof, exact, ekeys, ets, col


def _host_train(asof, exact, ekeys, ets, col, label):
    sets = [(asof, ekeys, True, [(0, np.float32, boff._NAN32), (1, np.float64, boff._NAN64)]), (exact, ekeys, False, [(0, np.int32, 0)])]
    before = nat.launch_count()
    res = boff.pit_train(ets, sets, [col], label, with_stats=True)
    assert nat.launch_count() - before == res[-1]["kernels"]
    return res


def train_launches(with_ts, n_sets, n_cols, arrays):
    return (24 if with_ts else 0) + max(1, n_sets, -(-n_cols // 64)) + 2 + -(-arrays // 64)


def test_host_launches_and_keep_rule():
    asof, exact, ekeys, ets, col = _setup()
    order, joined, cols, miss, stats = _host_train(asof, exact, ekeys, ets, col, (0, 1, nat.PIT_LABEL_NAN))
    assert stats["kernels"] == train_launches(True, 2, 1, 2 + 2 + 1 + 2 + 1 + 1)
    full = boff.pit_join(ets, [(asof, ekeys, True, [(0, np.float32, boff._NAN32), (1, np.float64, boff._NAN64)]),
                               (exact, ekeys, False, [(0, np.int32, 0)])], [col])
    keep = full[1][1][2] & full[1][0][2] & ~np.isnan(full[1][0][0][1])
    np.testing.assert_array_equal(order, full[0][keep])
    np.testing.assert_array_equal(joined[0][0][1].view(np.uint64), full[1][0][0][1][keep].view(np.uint64))
    np.testing.assert_array_equal(cols[0], full[2][0][keep])
    np.testing.assert_array_equal(miss, [int((~full[1][0][2]).sum()), int((~full[1][1][2]).sum())])


@pytest.mark.parametrize("stream", ["library", "caller"])
def test_device_entry_point_equals_the_host_run(stream):
    import torch

    asof, exact, ekeys, ets, col = _setup(seed=4)
    n = len(ekeys)
    label = (0, 1, nat.PIT_LABEL_NAN)
    h_order, h_joined, h_cols, h_miss, _stats = _host_train(asof, exact, ekeys, ets, col, label)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d_ts, d_keys, d_col = dev(ets), dev(ekeys), dev(col)
    out32, out64, outi = (torch.full((n,), -7, dtype=t, device="cuda") for t in (torch.float32, torch.float64, torch.int32))
    ts0, ts1 = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2))
    f0, f1 = (torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(2))
    d_dst, d_order = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda")
    d_miss, d_kept = torch.full((2,), 99, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda")
    o0 = (nat.PitOut * 2)(nat.PitOut(0, 4, boff._NAN32, out32.data_ptr()), nat.PitOut(1, 8, boff._NAN64, out64.data_ptr()))
    o1 = (nat.PitOut * 1)(nat.PitOut(0, 4, 0, outi.data_ptr()))
    c_s = (nat.PitSet * 2)(nat.PitSet(asof._h, d_keys.data_ptr(), 1, 2, o0, ts0.data_ptr(), f0.data_ptr()),
                           nat.PitSet(exact._h, d_keys.data_ptr(), 0, 1, o1, ts1.data_ptr(), f1.data_ptr()))
    cc = (nat.PitCol * 1)(nat.PitCol(d_col.data_ptr(), d_dst.data_ptr(), 8))
    strm = torch.cuda.Stream() if stream == "caller" else None
    torch.cuda.synchronize()
    before = nat.launch_count()
    nat.check(nat.load().b2s_pit_train_device(d_ts.data_ptr(), n, c_s, 2, cc, 1, C.byref(nat.PitLabel(*label)), d_order.data_ptr(),
                                              d_miss.data_ptr(), d_kept.data_ptr(), None if strm is None else strm.cuda_stream))
    assert nat.launch_count() - before == train_launches(True, 2, 1, 9)
    (strm or torch.cuda.current_stream()).synchronize()
    nat.check(nat.load().b2s_device_sync())
    k = int(d_kept.item())
    assert k == len(h_order)
    np.testing.assert_array_equal(d_order.cpu().numpy()[:k], h_order)
    np.testing.assert_array_equal(out64.cpu().numpy()[:k].view(np.uint64), h_joined[0][0][1].view(np.uint64))
    np.testing.assert_array_equal(out32.cpu().numpy()[:k].view(np.uint32), h_joined[0][0][0].view(np.uint32))
    np.testing.assert_array_equal(outi.cpu().numpy()[:k], h_joined[1][0][0])
    np.testing.assert_array_equal(d_dst.cpu().numpy()[:k], h_cols[0])
    np.testing.assert_array_equal(d_miss.cpu().numpy().astype(np.uint64), h_miss)
    assert (outi.cpu().numpy()[k:] == -7).all()  # nothing written past the kept rows


def test_refusals_launch_nothing():
    asof, exact, ekeys, ets, col = _setup(n=64)
    lib, n = nat.load(), 64
    bufs = [np.zeros(n + 1, np.int64) for _ in range(8)]
    keys, ts, out4, out8, ts_out, found, order, miss = [b.ctypes.data for b in bufs]
    kept, dst = np.zeros(1, np.int64), np.zeros(n, np.float64)

    def call(found=found, label=(0, 0, nat.PIT_LABEL_NAN), n_sets=1, miss=miss, kept=kept.ctypes.data, big=False):
        o = (nat.PitOut * 2)(nat.PitOut(0, 4, 0, out4), nat.PitOut(1, 8, 0, out8))
        c_s = (nat.PitSet * 65)(*[nat.PitSet(asof._h, keys, 1, 2, o, ts_out, found)] * 65)
        cc = (nat.PitCol * 1)(nat.PitCol(col.ctypes.data, dst.ctypes.data, 8))
        before = nat.launch_count()
        rc = lib.b2s_pit_train_host(ts, n, c_s, 65 if big else n_sets, cc, 1, None if label is None else C.byref(nat.PitLabel(*label)),
                                    order, miss, kept, None, None)
        return "launched" if nat.launch_count() != before and rc != 0 else rc

    assert call() == 0 and call(label=None) == 0 and call(label=(-1, 0, nat.PIT_LABEL_NAN)) == 0
    refused = {"no_found": call(found=None), "label_set": call(label=(1, 0, 0)), "label_out": call(label=(0, 2, 0)),
               "label_col": call(label=(-1, 1, 0)), "label_kind": call(label=(0, 0, 7)), "nat_on_4_bytes": call(label=(0, 0, nat.PIT_LABEL_NAT)),
               "null_miss": call(miss=None), "null_kept": call(kept=None), "65_sets": call(big=True),
               "misaligned_kept": call(kept=kept.ctypes.data + 4)}
    assert refused == dict.fromkeys(refused, -1), refused  # B2S_ERR_INVALID
