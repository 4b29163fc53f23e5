"""The dense linear head (csrc/b2s_dense.cu) at every template instantiation, epilogue and fallback, against plain
float64 numpy.  Needs an H100: `-m gpu`.

Rows go through `run_device` on device buffers, so which kernel serves a launch is decided by the plan and the
buffers alone; every case asserts `last_kernel`, the kernel family that actually ran.  Scores are checked against
`X64 @ W64.T + b` with the per-element bound of `score_bound` (derived there from the kernel's error model), labels and
votes exactly against `oracle.batch`, status words exactly.
"""

import contextlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.plan import DevicePlan  # noqa: E402
from oracle import batch as obatch  # noqa: E402

U = 2.0 ** -24  # float32 unit roundoff
SENT_F = np.float32(-7.77e30)  # output words no launch may touch keep this
SENT_I = np.int32(-777)


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def row_counts(sms):
    """a single CTA; warpgroup 1 of the only tile empty / partial / full; exactly one tile per CTA; several tiles per CTA
    with a ragged tail"""
    return [1, 63, 64, 65, 127, 128, 129, 128 * sms, 128 * sms + 1, 3 * 128 * sms + 77]


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def build(n_in, models, vote=None, fills=None, exact=False, dense=True):
    """models: [(W (scores, n_in) float64, b, link, classes)]"""
    plan = DevicePlan(n_in)
    plan.set_impute(fills or {})
    for W, b, link, classes in models:
        plan.add_linear(W, b, link, classes)
    if vote is not None:
        plan.set_vote(*vote)
    with env(B2S_DENSE_EXACT=int(exact), B2S_DENSE=int(dense)):
        return plan.finalize()


def regressors(W, b):
    return [(W[i:i + 1], b[i:i + 1], nat.LINK_IDENTITY, None) for i in range(len(b))]


def groups(n_pad, boxes):
    """accumulator groups G and boxes per group BPG of dense_head_kernel<NP, BOXES>"""
    g = boxes if n_pad == 16 else min(boxes, 2)
    return g, -(-boxes // g)


def score_bound(Xi, W, b, n_pad, boxes, exact):
    """|kernel score - float64 score| <= score_bound, per element, for rows Xi (float64, after the Imputer).

    With u = 2^-24 and S = sum_k |x_k| |w_k| + |b| (per row and score):
      * weights: w = wh + wm + wl, each term the leading 11 significant bits of what the previous ones left, so
        |w - wh - wm - wl| < 2^-30 |w|;
      * inputs: exact as xh + xm + xl (11 + 11 + 2 bits) in 3-term mode; in 2-term mode xm is r1 = x - xh (13 bits)
        rounded to 11 bits, |x - xh - xm| <= 2^-22 |x|;
      * dropped products xm.wl, xl.wm, xl.wl: < 2^-29 |x w|;
      together < (2^-28 + [2-term] 2^-22) S.  Every kept product of two tf32 numbers is exact in float32.
      * accumulation: each accumulator group (BPG boxes of 32 columns) runs 4 BPG wgmma k8 steps; a step adds eight exact
        products to the float32 accumulator and truncates, 2 ulp = 4u of the magnitude reached, which is at most the
        group's share S_g of S.  Over all groups: 16 BPG u S.  The small-term accumulators hold < 2^-9 S: negligible.
      * the epilogue: G - 1 group sums and main + small (float32, G u S), the intercept in float32 or float64 and the
        rounding of the stored float32 (3u S).
      * float32 weights below 2^-126 may be flushed by the tensor core: 2^-126 sum_k |x_k| at most.
    The float64 row kernels are far inside the same bound.  A plain one-term tf32 product (|x - xh| < 2^-10 |x|, the same
    for w) is not: `test_dense_matrix` checks that on every case."""
    g, bpg = groups(n_pad, boxes)
    S = np.abs(Xi) @ np.abs(W).T + np.abs(b)
    rel = (16 * bpg + g + 3) * U + 2.0 ** -28 + (0.0 if exact else 2.0 ** -22)
    return rel * S + 2.0 ** -126 * np.abs(Xi).sum(axis=1, keepdims=True)


def tf32(a):
    """the leading 11 significant bits of float32 values (what the kernel keeps as the large term)"""
    return (np.ascontiguousarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def full_split(e):
    """a coefficient whose three tf32 terms are all full: bits 0..32 below 2^e set, except bit 24 (so that the float32
    conversion does not round up into the next binade)"""
    return sum(2.0 ** (e - i) for i in range(33) if i != 24)


def make_weights(rng, n_scores, n_in):
    """normal coefficients plus split edges: exact powers of two, full 33-bit splits, float32-subnormal values"""
    W = rng.normal(size=(n_scores, n_in))
    W[:, 0] = rng.choice([-1.0, 1.0], n_scores) * 2.0 ** rng.integers(-6, 6, n_scores)
    W[:, 1] = rng.choice([-1.0, 1.0], n_scores) * np.array([full_split(int(e)) for e in rng.integers(-4, 4, n_scores)])
    W[:, 2] = rng.choice([-1.0, 1.0], n_scores) * 3e-40
    W[:, -1] = rng.choice([-1.0, 1.0], n_scores) * 2.0 ** -127
    return W


def make_rows(rng, n, n_in):
    """first half unit scale; second half every value scaled by 10^-3 .. 10^3"""
    X = rng.normal(size=(n, n_in))
    h = n // 2
    X[h:] *= 10.0 ** rng.integers(-3, 4, size=(n - h, n_in))
    return X.astype(np.float32)


class Rows:
    """one device copy of a batch, served at any prefix length"""

    def __init__(self, X, pad_bytes=0, stride_words=None):
        self.X = X
        n, k = X.shape
        self.stride = 4 * (stride_words or k)
        host = np.zeros((n, self.stride // 4), dtype=np.float32)
        host[:, :k] = X
        self.buf = nat.DeviceBuffer(host.nbytes + pad_bytes + 16)
        nat.check(nat.load().b2s_memcpy_h2d(self.buf.ptr + pad_bytes, host.ctypes.data, host.nbytes))
        self.ptr = self.buf.ptr + pad_bytes


def run(plan, rows, n):
    """run_device over the first n rows; the output and status buffers hold n + 1 rows of sentinels, and the one past the
    end must keep them"""
    is_int = plan.out_is_int
    sent = SENT_I if is_int else SENT_F
    out0 = np.full((n + 1, plan.out_cols), sent, dtype=plan.out_dtype)
    d_out = nat.DeviceBuffer(out0.nbytes).upload(out0)
    d_st = nat.DeviceBuffer(4 * (n + 1)).upload(np.full(n + 1, -1, dtype=np.int32))
    plan.run_device(rows.ptr, n, rows.stride, d_out.ptr, d_st.ptr)
    out = d_out.download(plan.out_dtype, out0.shape)
    st = d_st.download(np.int32, (n + 1,))
    assert (out[n] == sent).all() and st[n] == -1, "a row past the end was written"
    return out[:n], st[:n]


def check_scores(out, want, bound, tag):
    err = np.abs(out.astype(np.float64) - want)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{tag}: {int(bad.sum())} of {bad.size} scores outside the bound, worst err/bound "
                           f"{float(np.max(err / bound)):.3g}", np.argwhere(bad)[:5])
    return float(np.max(err / bound))


# ------------------------------------------------------------------------------------------ instantiation matrix
MATRIX = [(n_pad, boxes, fill, xt) for n_pad in (16, 32) for boxes in (1, 2, 3, 4) for fill in (False, True) for xt in (2, 3)]


def n_scores_of(n_pad, boxes, fill, xt):
    """9, 12, 13, 16 scores for N = 16, 17, 30, 32 for N = 32: padded and full, out_cols aligned to 4 and not"""
    pool = [9, 12, 13, 16] if n_pad == 16 else [17, 30, 32]
    return pool[(4 * boxes + 2 * fill + xt) % len(pool)]


@pytest.mark.parametrize("n_pad,boxes,fill,xt", MATRIX, ids=[f"N{a}-B{b}-{'fill' if c else 'nofill'}-XT{d}" for a, b, c, d in MATRIX])
def test_dense_matrix(n_pad, boxes, fill, xt, sms):
    """dense_head_kernel<NP, BOXES, FILL, XT> at every row count.  N = 16: 9-16 regressors, every score emitted (scores
    epilogue).  N = 32: a plan holds at most 16 models and never mixes classifiers with regressors, so more than 16
    scores come from one classifier with 17-32 classes (argmax epilogue): its labels are checked on every row whose best
    two scores are further apart than their bounds"""
    n_in, n_scores = 32 * boxes, n_scores_of(n_pad, boxes, fill, xt)
    rng = np.random.default_rng(1000 + 16 * boxes + n_pad + 2 * fill + xt)
    counts = row_counts(sms)
    n_max = counts[-1]
    W, b = make_weights(rng, n_scores, n_in), rng.normal(size=n_scores) * 4
    X = make_rows(rng, n_max, n_in)
    names = [f"f{i}" for i in range(n_in)]
    fills = None
    if fill:  # an Imputer over the even columns; NaN there is filled, NaN in an odd column or +-Inf flags the row
        fills = {c: float(rng.normal()) for c in range(0, n_in, 2)}
        X[rng.random(X.shape) < 0.02] = np.nan
        X[:, 1::2] = np.where(np.isnan(X[:, 1::2]), np.float32(0.5), X[:, 1::2])
        for r in rng.choice(n_max, 40, replace=False):
            X[r, rng.integers(0, n_in)] = rng.choice([np.nan, np.inf, -np.inf])
    classes = np.sort(rng.choice(np.arange(-50, 500), n_scores, replace=False)).astype(np.int32)
    models = regressors(W, b) if n_pad == 16 else [(W, b, nat.LINK_ARGMAX, classes)]
    plan = build(n_in, models, fills=fills, exact=(xt == 3))
    assert plan.kernel.startswith(f"dense_head_kernel<N={n_pad}>"), plan.kernel
    Xi = obatch.impute(X, names, {f"f{c}": v for c, v in (fills or {}).items()})
    ok = np.isfinite(Xi).all(axis=1)
    Xc = np.where(ok[:, None], Xi, 0.0)
    want = Xc @ W.T + b
    bound = score_bound(Xc, W, b, n_pad, boxes, xt == 3)
    # the bound rejects a one-term tf32 product (both the inputs and the weights truncated to 11 bits)
    one = tf32(Xc).astype(np.float64) @ tf32(W).astype(np.float64).T + b
    assert (np.abs(one - want) > bound)[ok].any(), "the bound does not tell a one-term tf32 product from the kernel"
    if n_pad == 32:
        keep = ok & clear_margin(want, bound, list(range(n_scores)))
        assert keep[ok].mean() >= 0.99, keep[ok].mean()
        labels = classes[np.argmax(want, axis=1)]
    rows = Rows(X)
    worst = 0.0
    for n in counts:
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense", (n, plan.last_kernel)
        assert np.array_equal(st, np.where(ok[:n], 0, nat.ROW_NONFINITE_INPUT)), n
        if n_pad == 16:
            worst = max(worst, check_scores(out[ok[:n]], want[:n][ok[:n]], bound[:n][ok[:n]], f"{n} rows"))
        else:
            k = keep[:n]
            assert np.array_equal(out[k, 0], labels[:n][k]), (n, np.argwhere(out[k, 0] != labels[:n][k])[:5])
    print(f"N={n_pad} boxes={boxes} fill={fill} XT={xt} scores={n_scores}: last_kernel={plan.last_kernel}, "
          + (f"worst err/bound {worst:.3f}" if n_pad == 16 else f"labels exact on {keep.mean():.4f} of the rows"))


@pytest.mark.parametrize("boxes", [3, 4])
def test_box_groups_follow_column_order(boxes, sms):
    """N = 32 keeps two accumulator groups, boxes [0, BPG) and [BPG, BOXES): here the first group's terms (+-2^20 x 1.0)
    are exact in float32 and cancel inside it, so the scores carry only the second group's rounding and a 20-class
    argmax over them is exact wherever their bound says so.  Another assignment of boxes to groups would add 2^25-sized
    partial sums to the small ones."""
    n_in, n_scores = 32 * boxes, 20
    rng = np.random.default_rng(40 + boxes)
    n = 3 * 128 * sms + 77
    X = rng.normal(size=(n, n_in)).astype(np.float32)
    X[:, :64] = 1.0
    W = rng.normal(size=(n_scores, n_in))
    W[:, :32], W[:, 32:64] = 2.0 ** 20, -(2.0 ** 20)
    b = rng.normal(size=n_scores)
    plan = build(n_in, [(W, b, nat.LINK_ARGMAX, None)])
    out, st = run(plan, Rows(X), n)
    assert plan.last_kernel == "dense" and not st.any()
    small = X[:, 64:].astype(np.float64)
    want = small @ W[:, 64:].T + b
    keep = clear_margin(want, score_bound(small, W[:, 64:], b, 32, boxes, False), list(range(n_scores)))
    assert keep.mean() >= 0.99
    assert np.array_equal(out[keep, 0], np.argmax(want, axis=1)[keep]), np.argwhere(out[keep, 0] != np.argmax(want, axis=1)[keep])[:5]


@pytest.mark.parametrize("boxes", [1, 3])
def test_cancellation_and_spanning_magnitudes(boxes, sms):
    """weights +-1e3 that cancel in pairs to 1e-4 of their size, inputs spanning 1e-3 .. 1e3 (pairs equal)"""
    n_pad, n_in, n_scores = 16, 32 * boxes, 10 + boxes
    rng = np.random.default_rng(50 + boxes)
    W = rng.normal(size=(n_scores, n_in)) * 1e3
    W[:, 1::2] = -W[:, 0::2] * (1 + 1e-4)
    X = (rng.normal(size=(4096, n_in)) * 10.0 ** rng.integers(-3, 4, size=(4096, n_in))).astype(np.float32)
    X[:, 1::2] = X[:, 0::2]
    b = rng.normal(size=n_scores)
    for exact in (False, True):
        plan = build(n_in, regressors(W, b), exact=exact)
        out, _ = run(plan, Rows(X), len(X))
        assert plan.last_kernel == "dense"
        X64 = X.astype(np.float64)
        check_scores(out, X64 @ W.T + b, score_bound(X64, W, b, n_pad, boxes, exact), f"exact={exact}")


def test_three_term_split_is_tighter_at_unit_scale():
    """what the exact input split buys: at unit scale the 2^-22 |x| input residual of the 2-term split is a visible part
    of the error"""
    rng = np.random.default_rng(60)
    W, b = rng.normal(size=(16, 128)), rng.normal(size=16)
    X = rng.normal(size=(40000, 128)).astype(np.float32)
    rows = Rows(X)
    want = X.astype(np.float64) @ W.T + b
    mean = {}
    for exact in (False, True):
        plan = build(128, regressors(W, b), exact=exact)
        out, _ = run(plan, rows, len(X))
        assert plan.last_kernel == "dense"
        mean[exact] = float(np.abs(out - want).mean())
    print(f"mean |err|: 2-term {mean[False]:.3e}, 3-term {mean[True]:.3e}")
    assert mean[True] < 0.95 * mean[False], mean  # measured on an H100: 9.8e-7 against 1.06e-6


# ------------------------------------------------------------------------------------------ epilogues
@pytest.mark.parametrize("n_models,n_in", [(13, 64), (16, 96)])
def test_mean_vote_epilogue(n_models, n_in, sms):
    """DENSE_EPI_MEAN (N = 16 only: at most 16 models): uneven weights, some zero, large intercepts"""
    rng = np.random.default_rng(70 + n_models)
    W, b = rng.normal(size=(n_models, n_in)), rng.normal(size=n_models) * 1e3
    w = rng.uniform(0.0, 1.0, n_models)
    w[[0, 3, n_models - 1]] = 0.0
    n_pad, boxes = (16 if n_models <= 16 else 32), n_in // 32
    X = make_rows(rng, 3 * 128 * sms + 77, n_in)
    plan = build(n_in, regressors(W, b), vote=(nat.VOTE_MEAN, w))
    X64 = X.astype(np.float64)
    scores = X64 @ W.T + b
    sb = score_bound(X64, W, b, n_pad, boxes, False)
    want = obatch.mean_vote(scores, w)
    # float32 vote weights (u |w|), an fmaf chain of n_pad terms (n_pad u sum |w| |score|) on top of the scores' own bounds
    vb = sb @ w + (n_pad + 2) * U * (np.abs(scores) + sb) @ w
    rows = Rows(X)
    for n in (1, 129, len(X)):
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense" and not st.any()
        check_scores(out[:, 0], want[:n], vb[:n], f"{n} rows")


def argmax_case(rng, n_classes, n_in, n):
    W, b = rng.normal(size=(n_classes, n_in)), rng.normal(size=n_classes)
    W[n_classes - 2], b[n_classes - 2] = W[1], b[1]  # two identical classes: an exact tie, the first one wins
    classes = np.sort(rng.choice(np.arange(3, 400), n_classes, replace=False)).astype(np.int32)
    X = rng.normal(size=(n, n_in)).astype(np.float32)
    return W, b, classes, X


def clear_margin(scores, bound, distinct):
    """rows whose best and second-best distinct scores are further apart than their bounds"""
    s, bd = scores[:, distinct], bound[:, distinct]
    order = np.argsort(-s, axis=1)
    r = np.arange(len(s))
    return s[r, order[:, 0]] - s[r, order[:, 1]] > bd[r, order[:, 0]] + bd[r, order[:, 1]]


@pytest.mark.parametrize("n_classes", [10, 16, 24, 32])
def test_argmax_epilogue(n_classes, sms):
    """DENSE_EPI_ARGMAX: one multi-class linear classifier, non-contiguous classes_, padded (10, 24) and full (16, 32)"""
    rng = np.random.default_rng(80 + n_classes)
    n_in = 96
    W, b, classes, X = argmax_case(rng, n_classes, n_in, 3 * 128 * sms + 77)
    plan = build(n_in, [(W, b, nat.LINK_ARGMAX, classes)])
    assert plan.out_is_int
    X64 = X.astype(np.float64)
    scores = X64 @ W.T + b
    scores[:, n_classes - 2] = scores[:, 1]  # the same column twice, whatever order the matrix product summed them in
    keep = clear_margin(scores, score_bound(X64, W, b, 16 if n_classes <= 16 else 32, 3, False),
                        [k for k in range(n_classes) if k != n_classes - 2])
    assert keep.mean() >= 0.99, keep.mean()
    want = classes[np.argmax(scores, axis=1)]
    assert (want == classes[1]).sum() > len(X) // (2 * n_classes)  # the tied pair wins often
    rows = Rows(X)
    for n in (1, 65, 128 * sms + 1, len(X)):
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense" and not st.any()
        k = keep[:n]
        assert np.array_equal(out[k, 0], want[:n][k]), (n, np.argwhere(out[k, 0] != want[:n][k])[:5])


def binary_models(rng, n_models, n_in):
    W, b = rng.normal(size=(n_models, n_in)), rng.normal(size=n_models) * 0.5
    cls = np.array([2, 5], dtype=np.int32)
    return W, b, [(W[i:i + 1], b[i:i + 1], nat.LINK_BINARY_GT, cls) for i in range(n_models)], cls


@pytest.mark.parametrize("vote", ["majority", "mean"])
def test_generic_epilogue_binary_classifiers(vote, sms):
    """DENSE_EPI_GENERIC: twelve binary logistic classifiers (classes_ [2, 5]) under a majority or a mean vote"""
    rng = np.random.default_rng(90)
    n_in = 64
    W, b, models, cls = binary_models(rng, 12, n_in)
    w = rng.uniform(0.1, 1.0, 12)
    X = rng.normal(size=(3 * 128 * sms + 77, n_in)).astype(np.float32)
    kind = nat.VOTE_MAJORITY if vote == "majority" else nat.VOTE_MEAN
    plan = build(n_in, models, vote=(kind, w))
    X64 = X.astype(np.float64)
    scores = X64 @ W.T + b
    keep = (np.abs(scores) > score_bound(X64, W, b, 16, 2, False)).all(axis=1)
    assert keep.mean() >= 0.99
    per = cls[(scores > 0).astype(int)]
    if vote == "majority":
        want = obatch.majority_vote(per, w)
    else:  # _mean_vote's float64 sum, in model order as the kernel adds it
        want = np.zeros(len(X))
        for m in range(12):
            want = want + per[:, m] * w[m]
    rows = Rows(X)
    for n in (1, 129, len(X)):
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense" and not st.any()
        k = keep[:n]
        if vote == "majority":
            assert np.array_equal(out[k, 0], want[:n][k])
        else:
            np.testing.assert_array_equal(out[k, 0], want[:n][k].astype(np.float32))


def test_generic_epilogue_mixed_links(sms):
    """DENSE_EPI_GENERIC: two 10-class argmax classifiers and four binary classifiers (24 scores, N = 32), every model's
    label emitted.  (A plan never mixes classifiers with regressors: the library refuses it.)"""
    rng = np.random.default_rng(95)
    n_in = 128
    W1, b1, c1, X = argmax_case(rng, 10, n_in, 3 * 128 * sms + 77)
    W2, b2, c2, _ = argmax_case(rng, 10, n_in, 1)
    Wb, bb, binary, cb = binary_models(rng, 4, n_in)
    models = [(W1, b1, nat.LINK_ARGMAX, c1)] + binary[:2] + [(W2, b2, nat.LINK_ARGMAX, c2)] + binary[2:]
    plan = build(n_in, models)
    assert plan.out_cols == 6 and plan.out_is_int
    X64 = X.astype(np.float64)
    keep = np.ones(len(X), dtype=bool)
    want = np.zeros((len(X), 6), dtype=np.int64)
    for col, (W, b, c) in ((0, (W1, b1, c1)), (3, (W2, b2, c2))):
        s = X64 @ W.T + b
        s[:, 8] = s[:, 1]
        keep &= clear_margin(s, score_bound(X64, W, b, 32, 4, False), [k for k in range(10) if k != 8])
        want[:, col] = c[np.argmax(s, axis=1)]
    sb = X64 @ Wb.T + bb
    keep &= (np.abs(sb) > score_bound(X64, Wb, bb, 32, 4, False)).all(axis=1)
    want[:, [1, 2, 4, 5]] = cb[(sb > 0).astype(int)]
    assert keep.mean() >= 0.99
    rows = Rows(X)
    for n in (1, 129, len(X)):
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense" and not st.any()
        k = keep[:n]
        assert np.array_equal(out[k], want[:n][k]), np.argwhere(out[k] != want[:n][k])[:5]


def test_merge_targets_on_one_device(sms):
    """the merge-target branch (every output row stored into each target at row_offset + row), with two buffers of the
    same device: both hold the same votes at the offset rows and nothing outside them"""
    rng = np.random.default_rng(99)
    n_in, n_models, off = 64, 13, 1000
    W, b = rng.normal(size=(n_models, n_in)), rng.normal(size=n_models)
    w = rng.uniform(0.0, 1.0, n_models)
    X = rng.normal(size=(3 * 128 * sms + 77, n_in)).astype(np.float32)
    n = len(X)
    plan = build(n_in, regressors(W, b), vote=(nat.VOTE_MEAN, w))
    total = off + n + 500
    init = np.full(total, SENT_F, dtype=np.float32)
    targets = [nat.DeviceBuffer(init.nbytes).upload(init) for _ in range(2)]
    plan.set_merge_targets([t.ptr for t in targets], off)
    out, st = run(plan, Rows(X), n)
    assert plan.last_kernel == "dense" and not st.any()
    assert (out == SENT_F).all(), "with merge targets the local output is not written"
    got = [t.download(np.float32, (total,)) for t in targets]
    assert np.array_equal(got[0], got[1])
    assert (got[0][:off] == SENT_F).all() and (got[0][off + n:] == SENT_F).all()
    X64 = X.astype(np.float64)
    scores = X64 @ W.T + b
    sb = score_bound(X64, W, b, 16, 2, False)
    check_scores(got[0][off:off + n], obatch.mean_vote(scores, w), sb @ w + U * (np.abs(scores) + sb) @ w, "merged")


# ------------------------------------------------------------------------------------------ row status across tiles
def test_row_status_across_tiles(sms):
    """non-finite values in tile c of CTA c (and in tile c + grid of others), in imputed and plain columns and in the
    column chunks of every warp: status words exact, the same in-tile rows of the CTA's other tiles clean and correct,
    every clean row's scores within the bound"""
    rng = np.random.default_rng(110)
    n_in, n_scores = 64, 13
    n = 3 * 128 * sms + 77  # grid = sms CTAs, each serving tiles c, c + grid, c + 2 grid
    W, b = rng.normal(size=(n_scores, n_in)), rng.normal(size=n_scores)
    X = rng.normal(size=(n, n_in)).astype(np.float32)
    fills = {c: 0.25 * c for c in range(0, n_in, 2)}
    plans = {"scores": build(n_in, regressors(W, b), fills=fills),
             "argmax": build(n_in, [(W, b, nat.LINK_ARGMAX, np.arange(n_scores, dtype=np.int32) * 7)], fills=fills)}
    ctas = sorted({0, 1, sms // 2, sms - 1})
    in_tile = [0, 5, 31, 63, 64, 100, 127]
    # (value, column): columns 8-15 and 24-31 of every 32-column box are split by warps 2 and 3, the others by warps 0, 1
    values = [(np.nan, 9), (np.nan, 8), (np.inf, 10), (-np.inf, 27), (np.nan, 43), (np.inf, 60), (np.nan, 1), (-np.inf, 20)]
    marked, clean = [], []
    for i, c in enumerate(ctas):
        for j, r in enumerate(in_tile):
            tile = 1 if (i + j) % 3 == 0 else 0  # mostly tile c, sometimes the CTA's second tile c + grid
            rows3 = [(c + t * sms) * 128 + r for t in range(3)]
            v, col = values[(i + j) % len(values)]
            X[rows3[tile], col] = v
            marked.append(rows3[tile])
            clean += [x for t, x in enumerate(rows3) if t != tile]
    X[7, 2] = np.nan  # imputed
    names = [f"f{i}" for i in range(n_in)]
    Xi = obatch.impute(X, names, {f"f{c}": v for c, v in fills.items()})
    ok = np.isfinite(Xi).all(axis=1)
    assert ok[7] and ok[clean].all() and (~ok[marked]).sum() >= len(marked) // 2
    Xc = np.where(ok[:, None], Xi, 0.0)
    scores = Xc @ W.T + b
    bound = score_bound(Xc, W, b, 16, 2, False)
    rows = Rows(X)
    for kind, plan in plans.items():
        out, st = run(plan, rows, n)
        assert plan.last_kernel == "dense", kind
        assert np.array_equal(st, np.where(ok, 0, nat.ROW_NONFINITE_INPUT)), (kind, np.argwhere(st != np.where(ok, 0, 1))[:8])
        if kind == "scores":
            check_scores(out[ok], scores[ok], bound[ok], "clean rows")
        else:
            keep = ok & clear_margin(scores, bound, list(range(n_scores)))
            assert keep[clean].mean() > 0.9
            assert np.array_equal(out[keep, 0], (np.argmax(scores, axis=1) * 7)[keep])


def test_row_status_alternating_tiles(sms):
    """every CTA alternates between a tile whose rows are all non-finite and a clean one, eight tiles each: a flag of one
    tile must neither reach the next tile's rows nor be lost to the reset of the previous tile's flags.  The NaN sits in
    a column split by warp 2, which starts on the next tile while warps 0 and 1 still store this one."""
    rng = np.random.default_rng(115)
    n_in, n_scores = 32, 13
    n = 8 * 128 * sms
    W, b = rng.normal(size=(n_scores, n_in)), rng.normal(size=n_scores)
    X = rng.normal(size=(n, n_in)).astype(np.float32)
    bad_tile = (np.arange(n) // 128 // sms) % 2 == 1
    X[bad_tile, 9] = np.nan
    plan = build(n_in, regressors(W, b))
    out, st = run(plan, Rows(X), n)
    assert plan.last_kernel == "dense"
    assert np.array_equal(st, bad_tile.astype(np.int32) * nat.ROW_NONFINITE_INPUT), np.argwhere(st != bad_tile)[:8]
    X64 = X[~bad_tile].astype(np.float64)
    check_scores(out[~bad_tile], X64 @ W.T + b, score_bound(X64, W, b, 16, 1, False), "clean tiles")


# ------------------------------------------------------------------------------------------ fallbacks
def test_fallback_paths_match_the_dense_head(sms):
    """one dense-eligible plan served by each path a launch can take, all held to the same bound"""
    rng = np.random.default_rng(120)
    n_in, n_scores = 64, 16
    W, b = make_weights(rng, n_scores, n_in), rng.normal(size=n_scores)
    plan = build(n_in, regressors(W, b))
    big = 2 * 65536 + 3000  # more than two pipelined chunks of b2s_run_host
    X = make_rows(rng, big, n_in)
    X64 = X.astype(np.float64)
    want, bound = X64 @ W.T + b, score_bound(X64, W, b, 16, 2, False)
    seen = {}

    def check(tag, out, n, expect):
        seen[tag] = plan.last_kernel
        assert plan.last_kernel == expect, (tag, plan.last_kernel)
        check_scores(out, want[:n], bound[:n], tag)

    n = 200  # 50 KB: read by the kernel from pinned host memory
    check("small host batch", plan.run(X[:n]), n, "rows")
    n = 128 * sms + 1
    check("device rows", run(plan, Rows(X[:n]), n)[0], n, "dense")
    check("pointer + 4 bytes", run(plan, Rows(X[:n], pad_bytes=4), n)[0], n, "rows")
    check("stride n_in*4 + 4", run(plan, Rows(X[:n], stride_words=n_in + 1), n)[0], n, "rows")
    check("stride n_in*4 + 16", run(plan, Rows(X[:n], stride_words=n_in + 4), n)[0], n, "dense")
    pinned = nat.pinned_empty(X.shape)
    pinned[:] = X
    check("pipelined pinned batch", plan.run(pinned), big, "dense")
    fp64 = build(n_in, regressors(W, b), dense=False)
    assert "dense" not in fp64.kernel
    out, _ = run(fp64, Rows(X[:n]), n)
    seen["B2S_DENSE=0"] = fp64.last_kernel
    assert fp64.last_kernel == "rows"
    check_scores(out, want[:n], bound[:n], "B2S_DENSE=0")
    print("last_kernel per path:", seen)


def onehot_plan(W, b, n_num, cats):
    plan = DevicePlan(n_num + 1)
    plan.set_output_schema([(c, nat.OUT_COPY, 0.0) for c in range(n_num)] + [(n_num, nat.OUT_ONEHOT, float(v)) for v in cats])
    for i in range(len(b)):
        plan.add_linear(W[i:i + 1], b[i:i + 1])
    return plan.finalize()


def test_near_eligible_plans_stay_off_the_dense_head(sms):
    """plans just outside what the dense head takes run the float64 kernels, correctly"""
    rng = np.random.default_rng(130)
    n = 128 * sms + 1

    def check(plan, X, Xm, W, b, expect):
        out, st = run(plan, Rows(X), n)
        assert plan.last_kernel == expect, (plan.kernel, plan.last_kernel)
        assert "dense" not in plan.kernel and not st.any()
        check_scores(out, Xm @ W.T + b, score_bound(Xm, W, b, 32, 4, False), plan.kernel)

    # 8 scores: below the dense head's range (the 8-score row kernels)
    W, b = rng.normal(size=(8, 64)), rng.normal(size=8)
    X = rng.normal(size=(n, 64)).astype(np.float32)
    plan = build(64, regressors(W, b))
    out, _ = run(plan, Rows(X), n)
    assert plan.last_kernel not in (None, "dense"), plan.last_kernel
    check_scores(out, X.astype(np.float64) @ W.T + b, score_bound(X.astype(np.float64), W, b, 16, 2, False), "8 scores")
    # 33 scores: more than any kernel takes, a clean error
    with pytest.raises(nat.NativeError, match="total scores 33"):
        build(64, [(rng.normal(size=(k, 64)), rng.normal(size=k), nat.LINK_ARGMAX, None) for k in (20, 13)])
    # 100 and 160 columns
    for k in (100, 160):
        W, b = rng.normal(size=(16, k)), rng.normal(size=16)
        X = rng.normal(size=(n, k)).astype(np.float32)
        check(build(k, regressors(W, b)), X, X.astype(np.float64), W, b, "rows")
    # 30 classes (32 score slots) over 100 columns
    W, b = rng.normal(size=(30, 100)), rng.normal(size=30)
    X = rng.normal(size=(n, 100)).astype(np.float32)
    plan = build(100, [(W, b, nat.LINK_ARGMAX, None)])
    out, st = run(plan, Rows(X), n)
    assert plan.last_kernel == "rows" and not st.any(), plan.last_kernel
    s = X.astype(np.float64) @ W.T + b
    keep = clear_margin(s, score_bound(X.astype(np.float64), W, b, 32, 4, False), list(range(30)))
    assert keep.mean() >= 0.99 and np.array_equal(out[keep, 0], np.argmax(s, axis=1)[keep])
    # 64 numeric columns and a one-hot column (3 categories)
    W, b = rng.normal(size=(12, 67)), rng.normal(size=12)
    X = rng.normal(size=(n, 65)).astype(np.float32)
    X[:, 64] = rng.integers(0, 4, n)
    Xm = np.concatenate([X[:, :64], (X[:, 64:65] == np.array([1.0, 2.0, 3.0])).astype(np.float32)], axis=1).astype(np.float64)
    check(onehot_plan(W, b, 64, [1, 2, 3]), X, Xm, W, b, "rows")
    # a mapped column
    W, b = rng.normal(size=(12, 64)), rng.normal(size=12)
    X = rng.normal(size=(n, 64)).astype(np.float32)
    X[:, 3] = rng.integers(0, 4, n)
    plan = DevicePlan(64).add_value_map(3, {1.0: 10.0, 2.0: -20.0})
    for i in range(12):
        plan.add_linear(W[i:i + 1], b[i:i + 1])
    plan.finalize()
    Xm = X.astype(np.float64)
    Xm[:, 3] = np.select([X[:, 3] == 1.0, X[:, 3] == 2.0], [10.0, -20.0], X[:, 3])
    check(plan, X, Xm, W, b, "rows")
