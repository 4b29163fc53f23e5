"""Running a plan on device rows and holding its output to a float64 reference (shared by the kernel-path test files).

Scores: every scoring kernel accumulates in fp64 and rounds once to float32 on output.  Per element
    |out - ref| <= 2^-24 |ref| + (n_terms + 2) 2^-52 S
with, for a linear scorer, n_terms = the columns plus the intercept and S = sum |x w| + |b|; for a tree model, the trees
of the score plus the init and S = |init| + sum |scale * leaf| along the row's paths.  A mean vote adds one fp64 rounding
per model.  Labels, votes and status words are compared exactly; classifier labels on the rows whose two best scores are
further apart than twice the bound (at least 99 % of the rows).
"""

import numpy as np

from mlrun_b200 import _native as nat
from oracle import batch as obatch
from tests import device_emulator as emu

U32, U64 = 2.0 ** -24, 2.0 ** -52
SENT_F = np.float32(-7.77e30)  # output words no launch may touch keep this
SENT_I = np.int32(-777)
ROW_NONFINITE, ROW_BAD_LABEL = 1, 2


def names(n):
    return [f"f{i}" for i in range(n)]


# ------------------------------------------------------------------------------------------ running a plan
class Rows:
    """one device copy of a batch, served at any prefix length.  stride: bytes between rows (default 4 * n_in; the
    words past n_in hold garbage no launch may read); offset: bytes between the allocation and row 0 (4 makes the rows
    unaligned for 16-byte copies)"""

    def __init__(self, X, stride=None, offset=0):
        self.X = np.ascontiguousarray(X, dtype=np.float32)
        n, n_in = self.X.shape
        self.stride = 4 * n_in if stride is None else int(stride)
        assert self.stride % 4 == 0 and self.stride >= 4 * n_in
        padded = np.full((n, self.stride // 4), np.float32(-1e38), dtype=np.float32)
        padded[:, :n_in] = self.X
        self.buf = nat.DeviceBuffer(padded.nbytes + offset + 16)
        nat.check(nat.load().b2s_memcpy_h2d(self.buf.ptr + offset, padded.ctypes.data, padded.nbytes))
        self.ptr = self.buf.ptr + offset


def run_device(plan, X, n=None):
    """run_device over the first n rows; the buffers hold one row of sentinels past the end, which must survive"""
    rows = X if isinstance(X, Rows) else Rows(X)
    n = rows.X.shape[0] if n is None else n
    sent = SENT_I if plan.out_is_int else SENT_F
    out0 = np.full((n + 1, plan.out_cols), sent, dtype=plan.out_dtype)
    d_out = nat.DeviceBuffer(out0.nbytes).upload(out0)
    d_st = nat.DeviceBuffer(4 * (n + 1)).upload(np.full(n + 1, -1, dtype=np.int32))
    plan.run_device(rows.ptr, n, rows.stride, d_out.ptr, d_st.ptr)
    out = d_out.download(plan.out_dtype, out0.shape)
    st = d_st.download(np.int32, (n + 1,))
    assert (out[n] == sent).all() and st[n] == -1, "a row past the end was written"
    return out[:n], st[:n]


def run_host(plan, X):
    return plan.run(np.ascontiguousarray(X, dtype=np.float32), with_status=True)


def assert_kernel(plan, *parts):
    for p in parts:
        assert p in plan.kernel, plan.kernel


# ------------------------------------------------------------------------------------------ float64 references
def tree_scores(t, E, acc=np.float64):
    """raw scores of a packed tree model (B, K), their magnitude S and term counts (K,), in fp64 (or `acc`), tree order.
    The same walk as the kernels: float32 x against the stored float32 threshold (xgboost's `<` already converted), NaN to
    the default child where the model routes missing values."""
    B = E.shape[0]
    K = t.n_scores
    sc = np.tile(np.asarray(t.init, dtype=acc), (B, 1))
    S = np.tile(np.abs(t.init), (B, 1))
    thr_all = emu.device_thresholds(t)
    dleft = t.default_left if t.nan_ok else None
    rows = np.arange(B)
    for ti in range(t.n_trees):
        base = t.tree_offset[ti]
        node = np.zeros(B, dtype=np.int64)
        active = t.feature[base + node] >= 0
        while active.any():
            f = t.feature[base + node]
            x = E[rows, np.where(f >= 0, f, 0)]
            with np.errstate(invalid="ignore"):
                left = x <= thr_all[base + node]
            if dleft is not None:
                left = np.where(np.isnan(x), dleft[base + node] != 0, left)
            node = np.where(active, np.where(left, t.left[base + node], t.right[base + node]), node)
            active = t.feature[base + node] >= 0
        v = t.tree_scale[ti] * t.leaf_value[base + node]
        k = t.tree_slot[ti]
        sc[:, k] = (sc[:, k] + v.astype(acc)).astype(acc)
        S[:, k] += np.abs(v)
    n_terms = np.bincount(t.tree_slot, minlength=K) + 1
    return sc.astype(np.float64), S, n_terms


def linear_scores(m, E):
    E64 = E.astype(np.float64)
    W, b = np.atleast_2d(m["W"]), np.atleast_1d(m["b"])
    return E64 @ W.T + b, np.abs(E64) @ np.abs(W).T + np.abs(b), np.full(len(b), E.shape[1] + 1)


def link_of(kind, m):
    return (m["link"], m["classes"]) if kind == "linear" else (m.link, m.classes)


class Ref:
    """per-model float64 reference of a plan's models: prediction, error bound of an identity prediction, and which rows
    give a label that no rounding within the bound can change"""

    def __init__(self, models, E):
        self.pred, self.bound, self.sure = [], [], []
        self.identity = np.array([link_of(kind, m)[0] == nat.LINK_IDENTITY for kind, m in models])
        for kind, m in models:
            sc, S, n_terms = linear_scores(m, E) if kind == "linear" else tree_scores(m, E)
            eps = (n_terms + 2) * U64 * S
            link, classes = link_of(kind, m)
            with np.errstate(invalid="ignore"):
                if link == nat.LINK_IDENTITY:
                    self.pred.append(sc[:, 0])
                    self.bound.append(eps[:, 0])
                    self.sure.append(np.ones(len(E), dtype=bool))
                    continue
                if link == nat.LINK_ARGMAX:
                    idx = np.argmax(sc, axis=1)
                    srt = np.sort(sc, axis=1)
                    sure = (srt[:, -1] - srt[:, -2]) > 2 * eps.max(axis=1)
                else:
                    idx = (sc[:, 0] > 0) if link == nat.LINK_BINARY_GT else (sc[:, 0] >= 0)
                    sure = np.abs(sc[:, 0]) > eps[:, 0]
            self.pred.append(np.asarray(idx, dtype=np.int64) if classes is None else np.asarray(classes)[np.asarray(idx, dtype=np.int64)])
            self.bound.append(np.zeros(len(E)))
            self.sure.append(sure)
        self.pred = np.stack(self.pred, axis=1)
        self.bound = np.stack(self.bound, axis=1)
        self.sure = np.stack(self.sure, axis=1)


def check_close(out, want, bound, tag=""):
    out = np.asarray(out, dtype=np.float64)
    tol = U32 * np.abs(want) + bound
    err = np.abs(out - want)
    bad = ~(err <= tol)
    assert not bad.any(), (f"{tag}: {int(bad.sum())} of {bad.size} outside the bound, worst err/bound "
                           f"{float(np.nanmax(err / np.maximum(tol, 1e-300))):.3g}", np.argwhere(bad)[:5])


def check_plan_output(out, st, models, E, vote=None, ok=None, routes_nan=False):
    """out / st of a plan over expanded rows E vs the float64 reference.  ok: rows expected unflagged (default: rows whose
    values are finite, or free of Inf when every model routes NaN)"""
    if ok is None:
        ok = ~np.isinf(E).any(axis=1) if routes_nan else np.isfinite(E).all(axis=1)
    ref = Ref(models, E)
    classify = any(link_of(k, m)[0] != nat.LINK_IDENTITY for k, m in models)
    if vote is None or vote[0] == nat.VOTE_NONE:
        if classify:
            sure = ref.sure.all(axis=1) & ok
            assert sure.sum() >= 0.99 * ok.sum(), f"only {int(sure.sum())} of {int(ok.sum())} rows have a certain label"
            np.testing.assert_array_equal(out[sure], ref.pred[sure])
        else:
            check_close(out[ok], ref.pred[ok], ref.bound[ok], "scores")
    elif vote[0] == nat.VOTE_MEAN:
        w = np.asarray(vote[1], dtype=np.float64)
        want = ref.pred.astype(np.float64) @ w
        bound = ref.bound @ np.abs(w) + (len(w) + 1) * U64 * (np.abs(ref.pred) @ np.abs(w))
        sure = ref.sure.all(axis=1) & ok
        assert sure.sum() >= 0.99 * ok.sum()
        check_close(out[sure, 0], want[sure], bound[sure], "mean vote")
    else:
        # regression outputs are voted as labels truncated to int (VotingEnsemble casts): a score closer to an integer
        # than its bound could truncate either way
        labels = np.trunc(ref.pred)
        sure = ref.sure.all(axis=1) & ok
        if ref.identity.any():
            frac = np.abs(ref.pred - np.round(ref.pred))[:, ref.identity]
            sure &= (frac > ref.bound[:, ref.identity] + U32 * np.abs(ref.pred[:, ref.identity])).all(axis=1)
        assert sure.sum() >= 0.99 * ok.sum(), f"only {int(sure.sum())} of {int(ok.sum())} rows have certain labels"
        want = obatch.majority_vote(labels, vote[1]) if labels.max() >= 0 else np.zeros(len(E), int)
        np.testing.assert_array_equal(out[sure, 0], want[sure])
        bad_label = (labels < 0).any(axis=1)
        np.testing.assert_array_equal((st[sure] & ROW_BAD_LABEL) != 0, bad_label[sure])
    np.testing.assert_array_equal((st & ROW_NONFINITE) != 0, ~ok)
    return ref
