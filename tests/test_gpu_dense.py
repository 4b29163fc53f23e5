"""Dense linear head on the tensor cores (csrc/b2s_dense.cu: wgmma tf32 over split operands, register accumulator
groups) vs scikit-learn's own predict().  Needs an H100: `-m gpu`.  Scores rtol 1e-5 (+ atol 1e-5); labels exact (see the tie
note in the test)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing  # noqa: E402
from mlrun_b200.feature_store.steps import Imputer  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from oracle import batch as obatch  # noqa: E402

RTOL, ATOL = 1e-5, 1e-5


@pytest.fixture(scope="module", autouse=True)
def _device():
    nat.init(0)
    yield


def names(n):
    return [f"f{i}" for i in range(n)]


def linear_models(n_models, n_feat, seed, scale=1.0):
    from sklearn.linear_model import LinearRegression

    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_models):
        m = LinearRegression()
        m.coef_, m.intercept_, m.n_features_in_ = rng.normal(size=n_feat) * scale, float(rng.normal()), n_feat
        out.append(m)
    return out


@pytest.mark.parametrize("n_rows", [1, 127, 128, 129, 5000])
def test_twelve_regressors_scores(n_rows):
    """12 linear scorers over 64 columns: N = 16 on the tensor core for the 5000-row batch, the fp64 rows kernel for the
    small ones; every model's prediction against X @ coef + intercept"""
    models = linear_models(12, 64, seed=1)
    X = np.random.default_rng(2).normal(size=(n_rows, 64)).astype(np.float32)
    plan = ColumnProgram(names(64)).build_plan([packing.pack_model(m) for m in models])
    assert plan.kernel.startswith("dense_head_kernel<N=16> (wgmma"), plan.kernel
    out, status = plan.run(X, with_status=True)
    # up to 64 KB (256 rows) the kernels read the batch from pinned host memory: no TMA, so the fp64 rows kernel serves it
    assert plan.last_kernel == ("rows" if n_rows <= 256 else "dense"), plan.last_kernel
    want = np.stack([m.predict(X.astype(np.float64)) for m in models], axis=1)
    np.testing.assert_allclose(out, want, rtol=RTOL, atol=ATOL)
    assert not status.any()
    vplan = ColumnProgram(names(64)).build_plan([packing.pack_model(m) for m in models], vote=(nat.VOTE_MEAN, [1 / 12] * 12))
    voted = vplan.run(X)
    assert vplan.last_kernel == plan.last_kernel
    np.testing.assert_allclose(voted[:, 0], obatch.mean_vote(want, [1 / 12] * 12), rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("exact", [0, 1])
def test_error_against_float64_at_unit_scale(exact, monkeypatch):
    """what the splits buy: inputs as xh + xm (second term rounded to nearest: 2^-23 |x| is dropped) or, B2S_DENSE_EXACT=1,
    as three exact terms; weights always as three terms of the float64 coefficient; one accumulator group per 32-column box.
    Unit-scale data, 128 columns, 16 scores of magnitude ~10: the error stays a few float32 ulp of the partial sums"""
    monkeypatch.setenv("B2S_DENSE_EXACT", str(exact))
    models = linear_models(16, 128, seed=21)
    X = np.random.default_rng(22).normal(size=(40000, 128)).astype(np.float32)
    plan = ColumnProgram(names(128)).build_plan([packing.pack_model(m) for m in models])
    assert "dense_head_kernel<N=16>" in plan.kernel and ("exact 3-term" in plan.kernel) == bool(exact), plan.kernel
    out = plan.run(X).astype(np.float64)
    assert plan.last_kernel == "dense", plan.last_kernel
    want = np.stack([m.predict(X.astype(np.float64)) for m in models], axis=1)
    err = np.abs(out - want)
    print("dense head, exact=%d: max |err| %.3e, mean %.3e (max |score| %.1f)" % (exact, err.max(), err.mean(), np.abs(want).max()))
    np.testing.assert_allclose(out, want, rtol=RTOL, atol=ATOL)
    # what is left is the fp32 arithmetic on the accumulators (float32 output rounding alone is ~2e-6 at scores of ~60), not the
    # input split
    assert err.max() < 2.5e-7 * np.abs(want).max() and err.mean() < 1.5e-6


def test_sixteen_class_logistic_regression_labels():
    """the case the north_star names: a multi-class linear classifier, argmax fused into the epilogue"""
    from sklearn.linear_model import LogisticRegression

    rng = np.random.default_rng(3)
    centres = rng.normal(size=(16, 64)) * 1.5
    y = rng.integers(0, 16, size=6000)
    Xf = (centres[y] + rng.normal(size=(6000, 64))).astype(np.float32)
    model = LogisticRegression(max_iter=300).fit(Xf, y * 3 + 5)  # labels 5, 8, ... (classes_ mapping is exercised)
    X = (centres[rng.integers(0, 16, size=20000)] + rng.normal(size=(20000, 64))).astype(np.float32)
    plan = ColumnProgram(names(64)).build_plan([packing.pack_model(model)])
    assert "dense_head_kernel<N=16>" in plan.kernel, plan.kernel
    out = plan.run(X)[:, 0]
    assert plan.last_kernel == "dense", plan.last_kernel
    want = model.predict(X.astype(np.float64))
    # 3xTF32 scores sit within ~1e-6 of the float64 ones: a label can differ only where the two best classes are closer
    # than that, which no row of this workload is
    scores = model.decision_function(X.astype(np.float64))
    top2 = np.sort(scores, axis=1)[:, -2:]
    assert (top2[:, 1] - top2[:, 0] > 1e-4).all()
    assert np.array_equal(out, want)


def test_ensemble_of_classifiers_with_majority_vote_and_wide_rows():
    """3 x 10-class classifiers over 128 columns (30 scores -> N = 32), VotingEnsemble majority vote"""
    from sklearn.linear_model import LogisticRegression, RidgeClassifier

    rng = np.random.default_rng(4)
    centres = rng.normal(size=(10, 128))
    y = rng.integers(0, 10, size=4000)
    Xf = (centres[y] * 0.8 + rng.normal(size=(4000, 128))).astype(np.float32)
    models = [LogisticRegression(max_iter=200, C=c).fit(Xf, y) for c in (0.1, 1.0)] + [RidgeClassifier().fit(Xf, y)]
    X = (centres[rng.integers(0, 10, size=9000)] * 0.8 + rng.normal(size=(9000, 128))).astype(np.float32)
    packed = [packing.pack_model(m) for m in models]
    plan = ColumnProgram(names(128)).build_plan(packed, vote=(nat.VOTE_MAJORITY, [0.5, 0.3, 0.2]))
    assert "dense_head_kernel<N=32>" in plan.kernel, plan.kernel
    per = np.stack([m.predict(X.astype(np.float64)) for m in models], axis=1)
    assert np.array_equal(ColumnProgram(names(128)).build_plan(packed).run(X), per)
    assert np.array_equal(plan.run(X)[:, 0], obatch.majority_vote(per, [0.5, 0.3, 0.2]))
    assert plan.last_kernel == "dense", plan.last_kernel


def test_cancellation_and_large_magnitudes():
    """adversarial for a split-precision product: weights +-1e3 that cancel to O(1), inputs spanning 1e-3 .. 1e3"""
    rng = np.random.default_rng(5)
    models = linear_models(10, 32, seed=6, scale=1e3)
    for m in models:  # pair the weights so that sums cancel: w[2j+1] = -w[2j] * (1 + 1e-4)
        m.coef_[1::2] = -m.coef_[0::2] * (1 + 1e-4)
    X = (rng.normal(size=(4096, 32)) * 10.0 ** rng.integers(-3, 4, size=(4096, 32))).astype(np.float32)
    X[:, 1::2] = X[:, 0::2]  # x[2j+1] = x[2j]: every pair contributes w x 1e-4, the large parts cancel
    plan = ColumnProgram(names(32)).build_plan([packing.pack_model(m) for m in models])
    assert "dense_head_kernel" in plan.kernel
    out = plan.run(X)
    assert plan.last_kernel == "dense", plan.last_kernel
    want = np.stack([m.predict(X.astype(np.float64)) for m in models], axis=1)
    # relative to the size of the terms that were summed (what any finite-precision dot product is bounded by)
    scale = np.abs(X.astype(np.float64)) @ np.abs(np.stack([m.coef_ for m in models], axis=1))
    assert (np.abs(out - want) <= 2e-6 * scale + ATOL).all(), float((np.abs(out - want) / (scale + 1e-30)).max())


def test_imputer_and_flagged_rows():
    models = linear_models(9, 64, seed=7)
    rng = np.random.default_rng(8)
    X = rng.normal(size=(3000, 64)).astype(np.float32)
    X[rng.random(X.shape) < 0.02] = np.nan
    X[5, 60] = np.inf
    prog = ColumnProgram(names(64))
    mapping = {f"f{i}": 0.25 * i for i in range(0, 64, 2)}  # odd columns are not imputed: their NaN rows are errors
    prog.apply(Imputer(mapping=mapping))
    plan = prog.build_plan([packing.pack_model(m) for m in models])
    assert "dense_head_kernel" in plan.kernel
    out, status = plan.run(X, with_status=True)
    assert plan.last_kernel == "dense", plan.last_kernel
    Xi = obatch.impute(X, names(64), mapping)
    ok = np.isfinite(Xi).all(axis=1)
    assert np.array_equal(status != 0, ~ok) and ok.sum() > 100 and (~ok).sum() > 100
    want = np.stack([m.predict(Xi[ok]) for m in models], axis=1)
    np.testing.assert_allclose(out[ok], want, rtol=RTOL, atol=ATOL)


def test_dense_head_beats_the_fp64_path_at_sixteen_scores(monkeypatch):
    """the reason it exists: at K = 16 scores the DFMA kernels are FP64-pipe bound"""
    import os

    models = linear_models(16, 64, seed=9)
    packed = [packing.pack_model(m) for m in models]
    X = np.random.default_rng(10).normal(size=(1 << 20, 64)).astype(np.float32)
    d_in = nat.DeviceBuffer(X.nbytes).upload(X)
    d_out = nat.DeviceBuffer(X.shape[0] * 16 * 4)
    times = {}
    for label, env in (("dense", "1"), ("fp64", "0")):
        os.environ["B2S_DENSE"] = env
        plan = ColumnProgram(names(64)).build_plan(packed)
        assert ("dense_head_kernel" in plan.kernel) == (label == "dense"), plan.kernel
        plan.time_device([d_in.ptr], X.shape[0], 256, d_out.ptr, 5)
        times[label] = plan.time_device([d_in.ptr], X.shape[0], 256, d_out.ptr, 20) / 20
        assert plan.last_kernel == ("dense" if label == "dense" else "rows"), plan.last_kernel
    os.environ.pop("B2S_DENSE", None)
    print("dense head %.4f ms vs fp64 rows kernel %.4f ms per 1 Mi events" % (times["dense"], times["fp64"]))
    assert times["dense"] < times["fp64"]
