"""FeatureSet.ingest / IngestPlan.run end to end on CPU: column extraction, result block, output dtypes, violation and miss
counters and the DataFrame assembly of the product, with the columnar kernel's arithmetic emulated in numpy
(tests/device_emulator.py EmulatedColumns), against the per-row and the vectorised oracle -- the very assertions
tests/test_gpu_ingest.py makes on the real kernel."""

import pytest

from tests import device_emulator


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    device_emulator.install_columns(monkeypatch)


def _cases():
    from tests import test_gpu_ingest as g  # its own tests are `-m gpu`; here their bodies run on the emulation

    return [(g.test_config5_matches_the_per_row_reference_walk, dict(n_rows=1)),
            (g.test_config5_matches_the_per_row_reference_walk, dict(n_rows=5)),
            (g.test_config5_matches_the_per_row_reference_walk, dict(n_rows=4097)),
            (g.test_config5_matches_the_per_row_reference_walk, dict(n_rows=20000)),
            (g.test_edge_values_match_the_reference_semantics, {}), (g.test_nat_and_wide_date_range, {}),
            (g.test_feature_set_ingest_api_and_dropped_validated_column, {})]


@pytest.mark.parametrize("case,kwargs", _cases(), ids=lambda v: v.__name__ if callable(v) else "-".join(map(str, v.values())))
def test_gpu_ingest_cases_hold_on_the_emulated_columns_plan(case, kwargs):
    case(**kwargs)


def test_ingest_runs_the_steps_argument_checks_first():
    """FeatureSet.validate_steps (feature_set.py:508-534; tests/feature-store/test_steps.py:466-547): bad MapValues mappings
    and DropFeatures of an entity / the timestamp key are refused before anything is lowered; steps given as objects or by
    class name alike"""
    import numpy as np
    import pandas as pd

    from mlrun_b200.feature_store import ingest as bi
    from mlrun_b200.feature_store import steps as bs
    from mlrun_b200.serving.resolve import MLRunInvalidArgumentError

    df = pd.DataFrame({"id": np.arange(6, dtype=np.int32), "age": np.array([1, 20, 40, 5, 70, 33], dtype=np.float32),
                       "dep": np.array([0, 1, 2, 1, 0, 2], dtype=np.int32),
                       "when": pd.date_range("2024-01-01", periods=6, freq="h").astype("datetime64[ns]")})

    def fset(*steps):
        fs = bi.FeatureSet("t", entities=[bi.Entity("id")], timestamp_key="when")
        cur = fs.graph
        for s in steps:
            cur = cur.to(*s[0], **s[1]) if isinstance(s, tuple) else cur.to(s)
        return fs

    with pytest.raises(MLRunInvalidArgumentError, match="can not combine ranges and single replacement.*'age'"):
        fset(bs.MapValues(mapping={"age": {"ranges": {0: [0, 30], 1: [30, "inf"]}, 4: 9}})).ingest(df)
    with pytest.raises(MLRunInvalidArgumentError, match="must be in the same type.*'dep'"):
        fset((("MapValues",), {"mapping": {"dep": {0: 1, 1: "x"}}})).ingest(df)
    with pytest.raises(MLRunInvalidArgumentError, match="not entities"):
        fset(bs.DropFeatures(features=["id"])).ingest(df)
    with pytest.raises(MLRunInvalidArgumentError, match="can not drop timestamp_key: when"):
        fset((("DropFeatures",), {"features": ["when"]})).ingest(df)
    good = fset(bs.MapValues(mapping={"age": {"ranges": {0: [0, 30], 1: [30, "inf"]}}}, with_original_features=True),
                bs.DropFeatures(features=["dep"]))
    out = good.ingest(df)
    assert list(out.columns) == ["age_mapped", "age", "when"] and out.index.name == "id"  # mapped first (steps.py:206-211)
    assert out["age_mapped"].tolist() == [0, 0, 1, 0, 1, 1]


def test_columnar_sources_give_the_frame_path_results_without_pandas():
    """dict of arrays / Arrow table in, ColumnBatch (-> Arrow) out: the same columns, dtypes and counters as FeatureSet.ingest(df)
    (SURVEY 8(f) #1); entity columns are carried through; int64 / float64 columns are refused like in frames"""
    import contextlib
    import io

    import numpy as np
    import pandas as pd
    import pyarrow as pa

    from mlrun_b200.feature_store import columnar
    from mlrun_b200.feature_store import ingest as bi
    from mlrun_b200.feature_store import steps as bs
    from mlrun_b200.lowering import LoweringError
    from mlrun_b200.synthetic import ingest_workload

    iw = ingest_workload(n_rows=3000, seed=11)

    def fset():
        fs = bi.FeatureSet("cols", timestamp_key="timestamp")
        cur = fs.graph
        for st in iw.build_steps(bs):
            cur = cur.to(st)
        return fs

    with contextlib.redirect_stdout(io.StringIO()):
        want = fset().ingest(iw.df)
        cols = {name: iw.df[name].to_numpy() for name in iw.df.columns}
        batch = fset().ingest(cols)
        from_arrow = fset().ingest(pa.table(cols))
    assert isinstance(batch, columnar.ColumnBatch) and len(batch) == 3000 and batch.names == list(want.columns)
    for got in (batch, from_arrow):
        for name in want.columns:
            a, b = got[name], want[name].to_numpy()
            assert a.dtype == b.dtype, (name, a.dtype, b.dtype)
            assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), name
    table = batch.to_arrow()
    assert table.num_rows == 3000 and table.column_names == list(want.columns)
    pd.testing.assert_frame_equal(batch.to_pandas(), want.reset_index(drop=True), check_exact=True)

    # entities ride along, untouched
    fs = bi.FeatureSet("e", entities=[bi.Entity("id")])
    fs.graph.to(bs.Imputer(mapping={"x": 1.5}))
    got = fs.ingest({"id": np.arange(5, dtype=np.int32), "x": np.array([1, np.nan, 3, np.nan, 5], dtype=np.float32)})
    assert got.names == ["x"] and got["x"].tolist() == [1.0, 1.5, 3.0, 1.5, 5.0] and got.index["id"].tolist() == [0, 1, 2, 3, 4]
    assert got.to_pandas().index.name == "id"
    with pytest.raises(LoweringError, match="int64"):
        fs.ingest({"id": np.arange(5, dtype=np.int32), "x": np.arange(5, dtype=np.int64)})
    with pytest.raises(LoweringError, match="float64"):
        fs.ingest({"id": np.arange(5, dtype=np.int32), "x": np.arange(5, dtype=np.float64)})
    with pytest.raises(ValueError, match="Arrow nulls"):
        fs.ingest(pa.table({"id": pa.array([1, 2], type=pa.int32()), "x": pa.array([1.0, None], type=pa.float32())}))



@pytest.mark.parametrize("kind", ["value", "range"])
def test_int32_values_beyond_float32_pass_through_maps_exactly(kind):
    """a MapValues of an int32 column to int32 integers writes int32 words: values that match nothing keep every digit
    (float32 would round 16 777 217 to 16 777 216 and INT32_MAX to 2^31).  A map to other values writes float32, and a
    frame whose int32 source holds a value float32 cannot represent is refused instead of rounded"""
    import contextlib
    import io

    import numpy as np
    import pandas as pd

    from mlrun_b200.feature_store import ingest as bi
    from mlrun_b200.feature_store import steps as bs
    from mlrun_b200.lowering import LoweringError
    from oracle import ingest as oi
    from oracle import transforms as ot

    big = [16_777_217, -16_777_219, 2**31 - 1, -2**31, 16_777_216, 1, 2, 0]
    df = pd.DataFrame({"k": np.array(big, dtype=np.int32), "x": np.arange(len(big), dtype=np.float32)})

    def steps(api, labels=(10, 20)):
        fmap = {"ranges": {labels[0]: [1, 2], labels[1]: [2, 3]}} if kind == "range" else {1: labels[0], 2: labels[1]}
        return [api.MapValues(mapping={"k": fmap}, with_original_features=True),
                api.FeaturesetValidator(validators={"k_mapped": api.MinMaxValidator(severity="info", min=-2**31, max=2**24)})]

    plan = bi.lower_steps(steps(bs), df)
    with contextlib.redirect_stdout(io.StringIO()):
        got = plan.run(df)
        want, n_viol = oi.ingest_rows(steps(ot), df)
    assert got["k_mapped"].dtype == np.int32
    assert got["k_mapped"].tolist() == want["k_mapped"].tolist() == [16_777_217, -16_777_219, 2**31 - 1, -2**31, 16_777_216, 10, 20, 0]
    assert plan.unmatched == {"k_mapped": 6} and plan.violations == {"k_mapped": 2} and n_viol == 2
    pd.testing.assert_frame_equal(got, want, check_dtype=False, check_exact=True)

    halves = bi.lower_steps(steps(bs, (0.5, 20)), df)  # float32 output: the frame above would be rounded
    with pytest.raises(LoweringError, match="float32 cannot represent"):
        halves.run(df)
    small = df[df["k"].abs() <= 2**24].reset_index(drop=True)  # every value float32-exact: served
    with contextlib.redirect_stdout(io.StringIO()):
        got = halves.run(small)
        want, _ = oi.ingest_rows(steps(ot, (0.5, 20)), small)
    assert got["k_mapped"].dtype == np.float32
    pd.testing.assert_frame_equal(got, want, check_dtype=False, check_exact=True)
