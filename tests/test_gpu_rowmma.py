"""rowmma_kernel (fp64 tensor-core dot products, b2s_rowmma.cuh) against the oracle and against the DFMA row kernel it
replaces: every (columns, scores) instantiation, ragged and tiny batches, NaN / out-of-vocabulary inputs, the generic
epilogue (classifier links + majority vote), row status.  Needs an H100: `-m gpu`.

Tolerance: rtol 1e-5 + atol 1e-5 against the float64 oracle (both kernels compute exact-product fp64 FMAs; they differ in the
order of the additions only, which the second half of each test bounds at a few float32 ulps of the result)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from mlrun_b200.synthetic import flow3_workload  # noqa: E402
from oracle import batch as obatch  # noqa: E402
from tests.test_gpu_parity import flow3_plan  # noqa: E402

RTOL, ATOL = 1e-5, 1e-5


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


@pytest.fixture(autouse=True)
def _opt_in(monkeypatch):
    """the DMMA variant is opt-in (the DFMA row kernel is the default)"""
    monkeypatch.setenv("B2S_RT_MMA", "1")
    yield


@pytest.mark.parametrize("n_num,n_cat", [(56, 8), (24, 8), (32, 0), (64, 0), (49, 15)])
@pytest.mark.parametrize("n_models", [1, 2, 3, 4, 7, 8])
def test_shapes_against_oracle_and_dfma_kernel(monkeypatch, n_num, n_cat, n_models):
    for n_rows in (1, 31, 32, 33, 4739, 150_001):
        wl = flow3_workload(n_rows=n_rows, n_num=n_num, n_cat=max(n_cat, 1), seed=n_num + 3 * n_models + n_rows % 7, n_models=n_models)
        if n_cat == 0:
            wl = flow3_workload(n_rows=n_rows, n_num=n_num - 1, n_cat=1, seed=n_num + n_models, n_models=n_models)
        plan = flow3_plan(wl, vote=False)
        assert plan.kernel.startswith("rowmma_kernel<NCH=%d" % ((n_num + n_cat) // 4)), plan.kernel
        out, status = plan.run(wl.X, with_status=True)
        ref = obatch.flow3(wl)["per_model"]
        np.testing.assert_allclose(out, ref, rtol=RTOL, atol=ATOL)
        assert (status == 0).all()
        monkeypatch.setenv("B2S_RT_MMA", "0")
        old = flow3_plan(wl, vote=False)
        monkeypatch.setenv("B2S_RT_MMA", "1")
        assert old.kernel.startswith("rowthread_kernel"), old.kernel
        out_old = old.run(wl.X)
        np.testing.assert_allclose(out, out_old, rtol=3e-7, atol=1e-6)


def test_mean_vote_and_status_words():
    wl = flow3_workload(n_rows=70_000, n_num=56, n_cat=8, seed=91, n_models=4)
    X = wl.X.copy()
    X[5, 60] = np.inf       # categorical column: encodes to zeros, row stays finite
    plan = flow3_plan(wl)
    out, status = plan.run(X, with_status=True)
    wl.X = X
    np.testing.assert_allclose(out[:, 0], obatch.flow3(wl)["out"], rtol=RTOL, atol=ATOL)
    assert (status == 0).all()
    # without the Imputer a NaN / Inf in a model input reaches the scores: the row is flagged, its neighbours are not
    prog = ColumnProgram(wl.names)
    from mlrun_b200.feature_store.steps import OneHotEncoder
    prog.apply(OneHotEncoder(mapping={k: list(v) for k, v in wl.onehot_mapping.items()}))
    raw = prog.build_plan([packing.pack_model(m) for m in wl.sklearn_models()])
    assert raw.kernel.startswith("rowmma_kernel"), raw.kernel
    Y = np.nan_to_num(X, nan=0.25, posinf=1.0, neginf=-1.0)
    bad = np.array([0, 31, 32, 4097, 69_999])
    Y[bad, [3, 17, 40, 55, 0]] = [np.nan, np.inf, -np.inf, np.nan, np.inf]
    out, status = raw.run(Y, with_status=True)
    want = np.zeros(len(Y), dtype=np.int32)
    want[bad] = 1
    np.testing.assert_array_equal(status & 1, want)
    assert np.isfinite(out[want == 0]).all()


def test_classifier_links_and_majority_vote_are_exact():
    from sklearn.linear_model import LogisticRegression

    rng = np.random.default_rng(5)
    X = rng.normal(size=(20_000, 32)).astype(np.float32)
    y3 = np.digitize(X[:, 0] + X[:, 1] * X[:, 2], [-0.5, 0.5])
    models = [LogisticRegression(max_iter=200).fit(X[:1500] + 0.1 * i, y3[:1500]) for i in range(2)]
    models.append(LogisticRegression(max_iter=200).fit(X[:1500], (y3[:1500] > 0).astype(int)))
    prog = ColumnProgram([f"f{i}" for i in range(32)])
    packed = [packing.pack_model(m) for m in models]
    plan = prog.build_plan(packed)
    assert plan.kernel.startswith("rowmma_kernel<NCH=8,NS=8>"), plan.kernel
    per_model = plan.run(X)
    want = np.stack([m.predict(X.astype(np.float64)) for m in models], axis=1)
    np.testing.assert_array_equal(per_model, want)
    w = [0.4, 0.3, 0.3]
    out = prog.build_plan(packed, vote=(nat.VOTE_MAJORITY, w)).run(X)
    np.testing.assert_array_equal(out[:, 0], obatch.majority_vote(want, w))


def test_cancellation_keeps_fp64_accuracy():
    """scores that cancel to ~1e-6 of the summed magnitudes: fp64 accumulation keeps them (a float32 accumulator would not)"""
    rng = np.random.default_rng(11)
    n, F = 8192, 64
    X = rng.normal(size=(n, F)).astype(np.float32)
    X[:, 32:] = X[:, :32]                      # pairs of equal inputs ...
    w = rng.normal(size=F)
    w[32:] = -w[:32] * (1 + 1e-6)              # ... with almost opposite weights

    class Lin:  # duck-typed LinearRegression for the packer
        pass
    from sklearn.linear_model import LinearRegression
    m = LinearRegression()
    m.coef_ = w
    m.intercept_ = 0.0
    m.n_features_in_ = F
    prog = ColumnProgram([f"f{i}" for i in range(F)])
    plan = prog.build_plan([packing.pack_model(m)])
    assert plan.kernel.startswith("rowmma_kernel<NCH=16,NS=1>"), plan.kernel
    out = plan.run(X)[:, 0]
    ref = X.astype(np.float64) @ w
    np.testing.assert_allclose(out, ref, rtol=1e-5, atol=1e-12)
