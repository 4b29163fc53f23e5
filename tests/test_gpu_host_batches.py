"""Every host path of a plan (b2s_run_host and the coalescing ring) on every kernel family, against float64 references
and against b2s_run_device on the same rows.  Needs an H100: `-m gpu`.

b2s_run_host takes a batch one of three ways: at most 64 KiB of rows (n * row_bytes <= kZeroCopyInBytes) is read by the
kernels from pinned host memory (the caller's, or the staging copy of pageable rows); a larger batch is copied in first;
a pinned batch of at least 2 x 65 536 rows runs as a pipeline of chunks of align_up(max(65 536, ceil(n / 64)), 1024) rows.
Results and status words are written straight to pinned memory, or copied back per chunk.  Strided rows are packed into
the staging area first.  A ring batch is the same batch from its pinned slot.

Which kernel serves a batch depends on where its rows are (`plan.last_kernel`):

    plan                          device rows        zero-copy host      copied / pipelined
    row-thread, NCH >= 8, aligned rowthread/tma      rowthread/host      rowthread/tma
    row-thread, NCH 4             rowthread/bulk     rowthread/host      rowthread/bulk
    dense head                    dense              rows                dense
    trees3 (n_in % 32 == 0)       trees3[_cat]/tma   trees3[_cat]        trees3[_cat]/tma
    rows / rows_cat / store       the same on every path

Where the same family serves both, the host batch gives the votes and status words of b2s_run_device bit for bit.  The
dense head is not one of them: a zero-copy batch of a dense plan runs rows_kernel in fp64, so its scores differ from the
tensor-core ones within the dense bound, and labels agree only where the margin exceeds it.

Plans whose votes go to merge targets or an attached communicator write nothing locally: the host entry points refuse
them (B2S_ERR_UNSUPPORTED, -6), before anything is enqueued, and b2s_run_device serves them.
"""

import ctypes as C
import threading
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing  # noqa: E402
from mlrun_b200.feature_store.online import DeviceTable  # noqa: E402
from mlrun_b200.feature_store.steps import OneHotEncoder  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from mlrun_b200.sharding import MergeComm  # noqa: E402
from mlrun_b200.synthetic import flow3_workload, tree_workload  # noqa: E402
from tests import device_emulator as emu  # noqa: E402
from tests import tree_cat_fixtures as cfx  # noqa: E402
from tests import tree_fixtures as tfx  # noqa: E402
from tests.device_check import (ROW_NONFINITE, SENT_F, SENT_I, U32, U64, Ref, Rows, assert_kernel, names,  # noqa: E402
                                run_device)
from tests.test_gpu_dense_matrix import score_bound  # noqa: E402
from tests.test_gpu_linear_paths import Flow, linear, rows_case, rows_data, rowthread, scorers, store_flow  # noqa: E402
from tests.test_gpu_linear_paths import with_categories  # noqa: E402
from tests.test_gpu_tree_categorical import CARDS, inputs as cat_inputs, lgbm_model, xgb_model  # noqa: E402
from tests.test_gpu_tree_paths import xgb  # noqa: E402

ZC_BYTES = 64 << 10      # kZeroCopyInBytes: the largest batch the kernels read from pinned host memory
CHUNK = 65536            # kHostChunkRows: rows per chunk of a pipelined host batch (at least)
PIPE = 2 * CHUNK + 3000  # the smallest pinned batch that is pipelined, plus a ragged last chunk
N_MAX = PIPE             # rows of every plan's batch
REFUSED = r"error -6: .*b2s_run_device"
ERR_INVALID, ERR_STATE = r"error -1:", r"error -4:"
RING_WAIT_US = 5_000_000  # the matrix's ring batches leave on b2s_flush, not on the hold


def zc_rows(n_in):
    return ZC_BYTES // (4 * n_in)


# ------------------------------------------------------------------------------------------ float64 expectations
class Expect:
    """what a plan must give on rows [lo, hi) of its batch, computed once in float64: outputs within `tol` of `want`
    where `mask` holds (or bit for bit: `bits`), status words exactly `flagged` * B2S_ROW_NONFINITE_INPUT"""

    def __init__(self, want=None, tol=None, mask=None, flagged=None, bits=None):
        self.want, self.tol, self.mask, self.bits = want, tol, mask, bits
        self.flagged = flagged

    def check(self, out, st, sl, tag=""):
        """sl: the batch rows out / st belong to (a slice or an index array)"""
        if self.bits is not None:
            w = self.bits[sl]
            same = (out.view(np.uint32) == w) | (np.isnan(out) & np.isnan(w.view(np.float32)))
            assert same.all(), (tag, np.argwhere(~same)[:5])
        else:
            with np.errstate(invalid="ignore"):
                err = np.abs(out.astype(np.float64) - self.want[sl])
            bad = self.mask[sl] & ~(err <= self.tol[sl])
            assert not bad.any(), (tag, f"{int(bad.sum())} outputs outside the bound", np.argwhere(bad)[:5])
        np.testing.assert_array_equal(st, np.where(self.flagged[sl], ROW_NONFINITE, 0).astype(np.int32), err_msg=tag)


def expect_models(models, E, ok, vote=None):
    """identity outputs within the bound of device_check on rows `ok`; labels exact where no rounding can change them"""
    ref = Ref(models, E)
    if vote is None:
        want = ref.pred.astype(np.float64)
        tol = np.where(ref.identity[None, :], U32 * np.abs(want) + ref.bound, 0.0)
        mask = np.where(ref.identity[None, :], ok[:, None], ref.sure & ok[:, None])
    else:  # mean vote
        w = np.asarray(vote[1], dtype=np.float64)
        mean = ref.pred.astype(np.float64) @ w
        bound = ref.bound @ np.abs(w) + (len(w) + 1) * U64 * (np.abs(ref.pred) @ np.abs(w))
        want, tol = mean[:, None], (U32 * np.abs(mean) + bound)[:, None]
        mask = (ref.sure.all(axis=1) & ok)[:, None]
    assert (mask.sum(axis=0) >= 0.99 * ok.sum()).all(), "too few rows have a certain label"
    return Expect(want, tol, mask, ~ok)


def expect_walk(packed, X, ok):
    """a categorical tree model (one identity score) against the float64 walk of tree_cat_fixtures"""
    sc, S, n_terms = cfx.packed_walk(packed, X)
    return Expect(sc[:, :1], (U32 * np.abs(sc[:, :1]) + (n_terms[0] + 2) * U64 * S[:, :1]), ok[:, None], ~ok)


def expect_dense(W, b, E, argmax):
    """the dense head's bound (test_gpu_dense_matrix.score_bound); the fp64 rows kernel of a zero-copy batch is far
    inside it.  argmax: the label exact on the rows whose two best scores are further apart than twice the bound"""
    ok = np.isfinite(E).all(axis=1)
    with np.errstate(invalid="ignore"):
        sc = E @ W.T + b
        bound = score_bound(E, W, b, 16, 2, False) + U32 * np.abs(sc)
        if not argmax:
            return Expect(sc, bound, np.broadcast_to(ok[:, None], sc.shape), ~ok)
        srt = np.sort(sc, axis=1)
        sure = ok & ((srt[:, -1] - srt[:, -2]) > 2 * bound.max(axis=1))
    assert sure.sum() >= 0.99 * ok.sum()
    return Expect(np.argmax(sc, axis=1)[:, None].astype(np.float64), np.zeros((len(E), 1)), sure[:, None], ~ok)


# ------------------------------------------------------------------------------------------ plans
# kind -> (parts of the plan kernel, device last_kernel, zero-copy host last_kernel, kernels per batch)
KINDS = {
    "linear": (rowthread(16, 1), "rowthread/tma", "rowthread/host", 1),  # the flow3 workload: 64 columns, 8 one-hot
    "trees": (("t3_prep_kernel + trees3_kernel<D=", ",floats>"), "trees3/tma", "trees3", 3),  # 4 models, mean vote
    "rt4x1": (rowthread(4, 1), "rowthread/bulk", "rowthread/host", 1),
    "rt4x8-onehot": (rowthread(4, 8), "rowthread/bulk", "rowthread/host", 1),
    "rt8x2": (rowthread(8, 2), "rowthread/tma", "rowthread/host", 1),
    "rt16x4-onehot": (rowthread(16, 4), "rowthread/tma", "rowthread/host", 1),
    "rt32x1-onehot": (rowthread(32, 1), "rowthread/tma", "rowthread/host", 1),
    "rt32x8-argmax": (rowthread(32, 8), "rowthread/tma", "rowthread/host", 1),
    "rows-linear": ("rows_kernel<LINEAR,NS=4>", "rows", "rows", 1),  # 17 one-hot sources
    "rows-mapvalues": ("rows_kernel<LINEAR,NS=1>", "rows", "rows", 1),
    "store": ("rows_kernel<STORE,NS=1>", "store", "store", 1),
    "rows-trees": ("rows_kernel<TREES,NS=1>", "rows", "rows", 1),  # depth 10
    "rows-cat": ("rows_kernel<TREES,NS=1> (categorical splits)", "rows_cat", "rows_cat", 1),
    "trees3-nan": (("trees3_kernel<D=", ",NaN routing>"), "trees3/tma", "trees3", 3),
    "trees3-cat": (("trees3_kernel<D=", ",NaN routing,categorical>"), "trees3_cat/tma", "trees3_cat", 3),
    "dense": ("dense_head_kernel", "dense", "rows", 1),  # 12 scores over 64 columns
    "dense-argmax": ("dense_head_kernel", "dense", "rows", 1),  # one 16-class argmax model
}


def onehot_flow(n_in, seed):
    cats = {1: [0, 1, 2], n_in - 2: [3, 5, 9, 11, 20]}
    return Flow(n_in).imputer({f"f{n_in // 2}": 0.5}).one_hot({f"f{c}": v for c, v in cats.items()}), cats


def numeric_rows(n, n_in, seed, cats=None):
    X = np.random.default_rng(seed).normal(size=(n, n_in)).astype(np.float32)
    if cats:
        X = with_categories(X, cats, seed=seed, p_edge=0.05)
    X[::997, n_in - 1] = np.nan
    X[5, 0] = np.inf
    return X


def make_plan(kind):
    """-> (plan, X of N_MAX rows, Expect over X)"""
    if kind == "linear":
        wl = flow3_workload(n_rows=N_MAX, n_num=56, n_cat=8, seed=51, n_models=1, nan_frac=0.002)
        prog = ColumnProgram(wl.names)
        prog.apply(OneHotEncoder(mapping={k: list(v) for k, v in wl.onehot_mapping.items()}))
        models = [packing.pack_model(m) for m in wl.sklearn_models()]
        E = emu.transform(prog, wl.X).astype(np.float64)
        return prog.build_plan(models), wl.X, expect_models(models, E, np.isfinite(E).all(axis=1))
    if kind == "trees":
        tw = tree_workload(n_rows=N_MAX, n_feat=32, n_models=4, n_trees=20, depth=5, seed=52, n_fit=1500)
        tw.X[::997, 5] = np.nan
        models = [packing.pack_model(m) for m in tw.models]
        vote = (nat.VOTE_MEAN, [0.25] * 4)
        plan = ColumnProgram(names(32)).build_plan(models, vote=vote)
        return plan, tw.X, expect_models(models, tw.X, np.isfinite(tw.X).all(axis=1), vote)
    if kind.startswith("rt"):
        nch, ns = int(kind[2:].split("x")[0]), int(kind.split("x")[1].split("-")[0])
        n_in = 4 * nch
        flow, cats = onehot_flow(n_in, nch + ns) if kind.endswith("onehot") else (Flow(n_in), None)
        if kind.endswith("argmax"):
            models = [linear(flow.width, 8, seed=nch, link=nat.LINK_ARGMAX, classes=list(range(-3, 13, 2)))]
        else:
            models = scorers(flow.width, {1: 1, 2: 2, 4: 3, 8: 5}[ns], seed=nch + ns)
        X = numeric_rows(N_MAX, n_in, nch * 10 + ns, cats)
        E = flow.expand(X)
        return flow.plan(models), X, expect_models(models, E, np.isfinite(E).all(axis=1))
    if kind in ("rows-linear", "rows-mapvalues"):
        case, n_in, n_scores = ("17-cat-cols", 40, 4) if kind == "rows-linear" else ("value-map", 40, 1)
        flow, models, vote, cats = rows_case(case, n_in, n_scores)
        X = rows_data(case, N_MAX, n_in, cats, seed=n_in + n_scores)
        X[::1013, 39] = np.nan
        E = flow.expand(X)
        return flow.plan(models, vote=vote), X, expect_models(models, E, np.isfinite(E).all(axis=1))
    if kind == "store":
        flow, cats = store_flow(13)
        rng = np.random.default_rng(13)
        X = (rng.normal(size=(N_MAX, 13)) * 2).astype(np.float32)
        X[:, ::2] = np.round(X[:, ::2])
        X = with_categories(X, cats, seed=13)
        X[::5, 0] = np.nan
        X[3, 12] = -0.0
        bits = flow.expand(X).astype(np.float32).view(np.uint32)
        return flow.program().build_plan([]), X, Expect(bits=bits, flagged=np.zeros(N_MAX, dtype=bool))
    if kind == "rows-trees":
        _, model = xgb(10, 8, seed=3, n_trees=12, p_leaf=0.05)
        X = tfx.grid_inputs(N_MAX, 8, seed=4, nan_frac=0.01)
        return ColumnProgram(names(8)).build_plan([model]), X, expect_models([model], X, np.isfinite(X).all(axis=1))
    if kind == "rows-cat":
        _, m = lgbm_model(10, seed=51, n_trees=8)
        X = cat_inputs(N_MAX, seed=53, nan_frac=0.01)
        return ColumnProgram(names(8)).build_plan([("trees", m)]), X, expect_walk(m, X, np.isfinite(X).all(axis=1))
    if kind == "trees3-nan":
        _, model = xgb(5, 32, seed=32, p_leaf=0.1)
        X = tfx.grid_inputs(N_MAX, 32, seed=33, with_inf=True, nan_frac=0.05)
        X[np.isinf(X).any(axis=1) & (np.arange(N_MAX) % 50 != 0)] = 0.5  # a few Inf rows, flagged
        return ColumnProgram(names(32)).build_plan([model]), X, expect_models([model], X, ~np.isinf(X).any(axis=1))
    if kind == "trees3-cat":
        _, m = xgb_model(5, n_feat=32, seed=5, cards=CARDS)
        X = cat_inputs(N_MAX, n_feat=32, seed=6)
        X[7::4001, 2] = np.inf
        return ColumnProgram(names(32)).build_plan([("trees", m)]), X, expect_walk(m, X, ~np.isinf(X).any(axis=1))
    # the dense head
    rng = np.random.default_rng(64)
    X = numeric_rows(N_MAX, 64, 64)
    if kind == "dense":
        models = scorers(64, 12, seed=12)
        W = np.concatenate([m["W"] for _, m in models])
        b = np.concatenate([m["b"] for _, m in models])
    else:
        W, b = rng.normal(size=(16, 64)), rng.normal(size=16)
        models = [("linear", dict(W=W, b=b, link=nat.LINK_ARGMAX, classes=list(range(16))))]
    return Flow(64).plan(models), X, expect_dense(W, b, X.astype(np.float64), kind == "dense-argmax")


class Served:
    """one plan of a kind, its batch, its expectation and b2s_run_device's output over the whole batch"""

    def __init__(self, kind):
        self.kind = kind
        self.kernel, self.dev_kernel, self.zc_kernel, self.k = KINDS[kind]
        self.plan, self.X, self.expect = make_plan(kind)
        self.X = np.ascontiguousarray(self.X, dtype=np.float32)
        assert_kernel(self.plan, *([self.kernel] if isinstance(self.kernel, str) else self.kernel))
        # matrix ring batches leave on b2s_flush: two slots of up to 4 zero-copy batches' rows
        self.plan.set_ring(2, 4 * zc_rows(self.plan.n_in) + 8, RING_WAIT_US)
        self.dev_out, self.dev_st = run_device(self.plan, Rows(self.X))
        assert self.plan.last_kernel == self.dev_kernel, (kind, self.plan.last_kernel)
        self.expect.check(self.dev_out, self.dev_st, slice(0, N_MAX), f"{kind} run_device")
        self.dense = kind.startswith("dense")

    def same_family(self, zero_copy):
        return not (self.dense and zero_copy)


_SERVED = {}


def served(kind):
    if kind not in _SERVED:
        nat.init(0)
        assert nat.device_info()["cc"] == (9, 0)
        _SERVED[kind] = Served(kind)
    return _SERVED[kind]


@pytest.fixture(scope="module", autouse=True)
def release_plans():
    yield
    for s in _SERVED.values():
        s.plan.close()
    _SERVED.clear()


# ------------------------------------------------------------------------------------------ host rows
def pinned_rows(X, offset=0):
    """a pinned copy of X, `offset` bytes (a multiple of 4) past the start of its allocation"""
    n, n_in = X.shape
    flat = nat.pinned_empty((n * n_in + 4,), np.float32)
    rows = flat[offset // 4: offset // 4 + n * n_in].reshape(n, n_in)
    rows[:] = X
    return rows


def strided_rows(X):
    wide = np.zeros((len(X), X.shape[1] + 16), dtype=np.float32)
    wide[:, :X.shape[1]] = X
    return wide[:, :X.shape[1]]


def run_host_raw(plan, X):
    """b2s_run_host into caller buffers that hold one more row of sentinels, which must survive"""
    n = X.shape[0]
    sent = SENT_I if plan.out_is_int else SENT_F
    out = np.full((n + 1, plan.out_cols), sent, dtype=plan.out_dtype)
    st = np.full(n + 1, -1, dtype=np.int32)
    stats = nat.Stats()
    nat.check(nat.load().b2s_run_host(plan._h, X.ctypes.data, n, X.strides[0], out.ctypes.data, n * plan.out_cols * 4,
                                      st.ctypes.data, C.byref(stats)))
    assert (out[n] == sent).all() and st[n] == -1, "a row past the caller's output was written"
    return out[:n], st[:n], stats.as_dict()


# (how, rows as a function of the plan's zero-copy rows z, what the batch is: "zc", "copied" or "pipelined")
HOWS = [
    ("zero-copy", lambda z: z // 2 + 3, "zc"),                  # pageable: read from the staging copy
    ("zero-copy-pinned", lambda z: z // 2 + 5, "zc"),           # the caller's pinned rows
    ("zero-copy-pinned-off4", lambda z: z // 2 + 7, "zc"),      # ... 4 bytes past a 16-byte boundary
    ("strided-zero-copy", lambda z: z // 2, "zc"),              # packed into the staging area, read from there
    ("zero-copy-limit", lambda z: z, "zc"),                     # n * row_bytes == 64 KiB
    ("copied-limit", lambda z: z + 1, "copied"),                # one row more
    ("copied", lambda z: 4 * z + 1, "copied"),
    ("copied-pinned-off4", lambda z: 2 * z + 9, "copied"),
    ("strided", lambda z: 3 * z + 1, "copied"),                 # packed into the staging area, copied in from there
    ("pinned-below-pipeline", lambda z: 2 * CHUNK - 1, "copied"),
    ("pipelined-full", lambda z: 2 * CHUNK, "pipelined"),       # two chunks, the last one full
    ("pipelined", lambda z: PIPE, "pipelined"),                 # three chunks, the last one ragged
]


def host_rows(how, X):
    """the same rows as the host path `how` takes them"""
    if how.endswith("off4"):
        return pinned_rows(X, offset=4)
    if "pinned" in how or how.startswith("pipelined"):
        return pinned_rows(X)
    if how.startswith("strided"):
        return strided_rows(X)
    return np.ascontiguousarray(X)


def check_host_batch(s, out, st, stats, sl, zero_copy, batch_rows, kernels, tag):
    """out / st of batch rows `sl`: the reference, b2s_run_device bit for bit where the same family served it, stats"""
    s.expect.check(out, st, sl, tag)
    if s.same_family(zero_copy):
        np.testing.assert_array_equal(out.view(np.uint32), s.dev_out[sl].view(np.uint32), err_msg=tag)
        np.testing.assert_array_equal(st, s.dev_st[sl], err_msg=tag)
    assert stats["rows"] == batch_rows and stats["kernels"] == kernels, (tag, stats)
    assert stats["nonfinite_rows"] == int(((st & ROW_NONFINITE) != 0).sum()), (tag, stats)


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("how", [h for h, _, _ in HOWS])
def test_run_host_matches_run_device(kind, how):
    """one plan of every kernel family on every b2s_run_host path: the float64 reference, b2s_run_device bit for bit
    (except a zero-copy dense batch), status words, stats, a sentinel row past the caller's output, last_kernel"""
    s = served(kind)
    _, rows_of, batch = next(h for h in HOWS if h[0] == how)
    n = rows_of(zc_rows(s.plan.n_in))
    assert n <= N_MAX
    zero_copy = batch == "zc"
    assert zero_copy == (n * 4 * s.plan.n_in <= ZC_BYTES)
    out, st, stats = run_host_raw(s.plan, host_rows(how, s.X[:n]))
    assert s.plan.last_kernel == (s.zc_kernel if zero_copy else s.dev_kernel), (how, s.plan.last_kernel)
    chunks = -(-n // CHUNK) if batch == "pipelined" else 1
    check_host_batch(s, out, st, stats, slice(0, n), zero_copy, n, s.k * chunks, f"{kind} {how}")
    if kind != "store":
        assert (st != 0).any(), "the batch has no flagged row"


@pytest.mark.parametrize("kind", ["dense", "dense-argmax"])
def test_dense_plan_zero_copy_and_copied_agree(kind):
    """a zero-copy batch of a dense plan runs rows_kernel (fp64) and a copied one the dense head: both within the dense
    bound, labels equal on every row whose margin exceeds it"""
    s = served(kind)
    z = zc_rows(s.plan.n_in)
    out_zc, st_zc, _ = run_host_raw(s.plan, np.ascontiguousarray(s.X[:z]))
    assert s.plan.last_kernel == "rows"
    # the same z rows in a batch of more than 64 KiB: the first z rows of a 2z-row batch
    out_cp, st_cp, _ = run_host_raw(s.plan, np.ascontiguousarray(s.X[:2 * z]))
    assert s.plan.last_kernel == "dense"
    out_cp, st_cp = out_cp[:z], st_cp[:z]
    np.testing.assert_array_equal(st_zc, st_cp)
    if kind == "dense-argmax":
        sure = s.expect.mask[:z, 0]
        np.testing.assert_array_equal(out_zc[sure], out_cp[sure])
        print(f"{kind}: {int((out_zc[~sure] != out_cp[~sure]).sum())} of {int((~sure).sum())} uncertain labels differ")
    else:
        ok = s.expect.mask[:z]
        bound = 2 * s.expect.tol[:z]
        assert (np.abs(out_zc.astype(np.float64) - out_cp)[ok] <= bound[ok]).all()
        print(f"{kind}: {int((out_zc != out_cp).sum())} of {out_zc.size} scores differ in their last bits")


def test_pipeline_chunk_grows_past_64_chunks():
    """a pinned batch of 64 x 65 536 + 1 narrow rows: the chunk becomes align_up(ceil(n / 64), 1024) = 66 560 rows, 64
    chunks, the last one 1 025 rows; every chunk matches b2s_run_device and the reference"""
    s = served("rt4x1")
    n = 64 * CHUNK + 1
    chunk = -(-(-(-n // 64)) // 1024) * 1024
    n_chunks = -(-n // chunk)
    assert (chunk, n_chunks, n - (n_chunks - 1) * chunk) == (66560, 64, 1025)
    reps = -(-n // N_MAX)
    X = np.ascontiguousarray(np.tile(s.X, (reps, 1))[:n])
    flagged = np.tile(s.expect.flagged, reps)[:n]
    want, want_st = run_device(s.plan, Rows(X))
    np.testing.assert_array_equal(want_st, np.tile(s.dev_st, reps)[:n])
    out, st, stats = run_host_raw(s.plan, pinned_rows(X))
    assert s.plan.last_kernel == "rowthread/bulk"
    np.testing.assert_array_equal(out.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(out.view(np.uint32), np.tile(s.dev_out, (reps, 1))[:n].view(np.uint32))
    np.testing.assert_array_equal(st, want_st)
    assert stats["rows"] == n and stats["kernels"] == n_chunks
    assert stats["nonfinite_rows"] == int(flagged.sum())


# ------------------------------------------------------------------------------------------ ring batches of every plan
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("batch", ["zero-copy", "copied"])
def test_submit_wait_matches_run_device(kind, batch):
    """three tickets in one ring batch (sealed by b2s_flush), collected in reverse: each ticket gets its own rows, status
    words and non-finite count, the batch's rows and launches; a zero-copy batch is read from the slot's pinned memory"""
    s = served(kind)
    z = zc_rows(s.plan.n_in)
    total = z if batch == "zero-copy" else 3 * z + 2
    cuts = [0, total // 3, total // 3 + total // 4, total]
    base = 11 * CHUNK // 10
    tickets = []
    for a, b in zip(cuts, cuts[1:]):
        tickets.append((s.plan.submit(np.ascontiguousarray(s.X[base + a:base + b])), a, b))
    s.plan.flush()
    assert len({t >> 24 for (t, _), _, _ in tickets}) == 1, "the tickets went to different batches"
    assert [t & 0xFFFFFF for (t, _), _, _ in tickets] == cuts[:-1]
    for ticket, a, b in reversed(tickets):
        out, st, stats = s.plan.wait(ticket, with_status=True, with_stats=True)
        check_host_batch(s, out, st, stats, slice(base + a, base + b), batch == "zero-copy", total, s.k, f"{kind} ticket {a}")
    assert s.plan.last_kernel == (s.zc_kernel if batch == "zero-copy" else s.dev_kernel)


# ------------------------------------------------------------------------------------------ the ring's batch formation
def ring_plan(kind="rt16x4-onehot", slots=4, max_batch=0, wait_us=-1):
    """a fresh plan of a served kind, its ring configured (before the first submit), and the served one"""
    s = served(kind)
    plan = make_plan(kind)[0]
    assert plan.kernel == s.plan.kernel
    plan.set_ring(slots, max_batch, wait_us)
    return s, plan


def collect(plan, s, ticket, rows, tag, exact=True):
    """wait on a ticket of batch rows `rows` (a slice or an index array of s.X): its own outputs, status words and
    non-finite count; exact: bit-equal to b2s_run_device"""
    out, st, stats = plan.wait(ticket, with_status=True, with_stats=True)
    s.expect.check(out, st, rows, tag)
    if exact:
        np.testing.assert_array_equal(out.view(np.uint32), s.dev_out[rows].view(np.uint32), err_msg=tag)
        np.testing.assert_array_equal(st, s.dev_st[rows], err_msg=tag)
    assert stats["nonfinite_rows"] == int(((st & ROW_NONFINITE) != 0).sum()), (tag, stats)
    return stats


@pytest.mark.parametrize("order", ["reverse", "random"])
def test_ring_ticket_offsets_and_sizes(order):
    """tickets of 1 ... 300 rows packed into shared batches on both sides of the 64 KiB zero-copy limit (256 rows of
    this plan); flagged rows only in every other ticket and never at its offset 0; every ticket gets its own rows,
    status words and non-finite count, whichever order they are collected in"""
    s, plan = ring_plan(max_batch=4096, wait_us=RING_WAIT_US)
    rng = np.random.default_rng(len(order))
    flagged = np.flatnonzero(s.expect.flagged)
    clean = rng.permutation(np.flatnonzero(~s.expect.flagged))
    groups = [[1, 7, 2, 40, 3, 100, 1, 60], [300, 1, 17, 256, 5, 299, 2], [64, 64, 64, 64], [1]]
    assert sum(groups[0]) < 256 < sum(groups[1]) and sum(groups[2]) == 256
    used, tickets = 0, []
    for g in groups:
        off = 0
        for size in g:
            rows = clean[used:used + size].copy()
            used += size
            if size >= 2 and len(tickets) % 2 == 1:  # one or two flagged rows, at offsets >= 1
                at = rng.choice(np.arange(1, size), size=min(2, size - 1), replace=False)
                rows[at] = rng.choice(flagged, size=len(at), replace=False)
            tickets.append((plan.submit(np.ascontiguousarray(s.X[rows])), rows, sum(g), off))
            off += size
        plan.flush()
    assert sum(int(s.expect.flagged[t[1]].any()) for t in tickets) >= 5
    ids = np.asarray([t[0][0] >> 24 for t in tickets])
    per_group = np.split(ids, np.cumsum([len(g) for g in groups])[:-1])
    assert all(len(set(p)) == 1 for p in per_group) and len({p[0] for p in per_group}) == len(groups)
    assert [t[0][0] & 0xFFFFFF for t in tickets] == [t[3] for t in tickets]
    idx = range(len(tickets) - 1, -1, -1) if order == "reverse" else rng.permutation(len(tickets))
    for i in idx:
        ticket, rows, batch_rows, off = tickets[i]
        stats = collect(plan, s, ticket, rows, f"ticket {i} at offset {off}")
        assert stats["rows"] == batch_rows and stats["kernels"] == 1
    plan.close()


def test_ring_max_batch_seals_and_limits():
    """max_batch = 100: 60 + 60 rows go to two batches at offset 0; exactly 100 rows seal a batch at once (it runs
    although the hold is 10 s); 101 rows are refused; so are set_ring once the ring runs, and out-of-range settings"""
    s, plan = ring_plan(slots=4, max_batch=100, wait_us=10_000_000)
    X = s.X
    a = plan.submit(np.ascontiguousarray(X[1000:1060]))
    b = plan.submit(np.ascontiguousarray(X[2000:2060]))
    assert (b[0] >> 24) == (a[0] >> 24) + 1 and a[0] & 0xFFFFFF == 0 and b[0] & 0xFFFFFF == 0
    with pytest.raises(nat.NativeError, match=ERR_STATE):
        plan.set_ring(4, 200, 0)
    with pytest.raises(nat.NativeError, match=ERR_INVALID):
        plan.submit(np.ascontiguousarray(X[:101]))
    collect(plan, s, a, slice(1000, 1060), "first 60")  # sealed when the second did not fit
    full = plan.submit(np.ascontiguousarray(X[3000:3100]))
    assert full[0] & 0xFFFFFF == 0 and (full[0] >> 24) == (b[0] >> 24) + 1
    got = {}
    th = threading.Thread(target=lambda: got.update(stats=collect(plan, s, full, slice(3000, 3100), "exactly 100")), daemon=True)
    th.start()
    th.join(timeout=5.0)
    held = th.is_alive()
    plan.flush()  # lets a held batch go, so that a failure does not leave the waiter behind
    th.join(timeout=30.0)
    assert not held, "a batch of max_batch rows waited for the hold"
    assert got["stats"]["rows"] == 100
    collect(plan, s, b, slice(2000, 2060), "second 60")
    plan.close()
    fresh = ring_plan()[1]
    for bad in ((65, 0, 0), (-1, 0, 0), (0, (1 << 24) + 1, 0), (0, -1, 0), (0, 0, 10_000_001)):
        with pytest.raises(nat.NativeError, match=ERR_INVALID):
            fresh.set_ring(*bad)
    fresh.set_ring(64, 1 << 24, 10_000_000)
    fresh.close()


def test_ring_exhaustion_blocks_the_producer():
    """ring_slots = 2, max_batch = 100: a producer's third batch waits in b2s_submit until another thread collects a
    ticket of the first two (ordering, not timing: the collector marks the moment before it collects)"""
    s, plan = ring_plan(slots=2, max_batch=100, wait_us=0)
    X = s.X
    about_to_submit, collecting = threading.Event(), threading.Event()
    res = {}

    def producer():
        res["t"] = [plan.submit(np.ascontiguousarray(X[i * 100:(i + 1) * 100])) for i in range(2)]
        about_to_submit.set()
        t3 = plan.submit(np.ascontiguousarray(X[200:300]))
        res["collected_before_third"] = collecting.is_set()
        res["t3"] = t3

    def collector():
        about_to_submit.wait(timeout=30)
        time.sleep(0.2)  # the third submit has had time to return if it did not block
        collecting.set()
        res["s1"] = collect(plan, s, res["t"][0], slice(0, 100), "first")

    threads = [threading.Thread(target=producer, daemon=True), threading.Thread(target=collector, daemon=True)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=30)
    assert not any(t.is_alive() for t in threads), "the ring hung"
    assert res["collected_before_third"], "the third batch was accepted while both slots held uncollected tickets"
    collect(plan, s, res["t"][1], slice(100, 200), "second")
    collect(plan, s, res["t3"], slice(200, 300), "third")
    plan.close()


def test_ring_hold_and_uncollected_tickets():
    """max_wait_us = 200 ms: back-to-back submits share one batch, which leaves on its own after the hold although
    nobody waits on it; its tickets are collected afterwards"""
    s, plan = ring_plan(slots=4, max_batch=4096, wait_us=200_000)
    spans = [(10, 30), (500, 507), (2000, 2150)]
    tickets = [plan.submit(np.ascontiguousarray(s.X[a:b])) for a, b in spans]
    assert len({t >> 24 for t, _ in tickets}) == 1
    time.sleep(0.6)
    for (a, b), t in zip(spans, tickets):
        stats = collect(plan, s, t, slice(a, b), f"held {a}")
        assert stats["queue_us"] >= 200_000 and stats["rows"] == 177
    plan.close()


@pytest.mark.parametrize("kind", ["rt16x4-onehot", "trees", "dense"])
def test_ring_many_producers(kind):
    """32 threads emit and await tickets of 1 ... 300 rows over their own row ranges: every ticket bit-equal to
    b2s_run_device (the dense plan: within the dense bound, as zero-copy batches run rows_kernel)"""
    s, plan = ring_plan(kind, slots=4, max_batch=4096, wait_us=0)
    errors, done = [], [0] * 32

    def producer(t):
        rng = np.random.default_rng(t)
        span = N_MAX // 32
        try:
            for _ in range(12):
                size = int(rng.integers(1, 301))
                lo = t * span + int(rng.integers(0, span - size))
                collect(plan, s, plan.submit(np.ascontiguousarray(s.X[lo:lo + size])), slice(lo, lo + size), f"producer {t}",
                        exact=not s.dense)
                done[t] += 1
        except Exception as e:  # noqa: BLE001  (reported by the main thread)
            errors.append(e)

    threads = [threading.Thread(target=producer, args=(t,), daemon=True) for t in range(32)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
    assert not any(t.is_alive() for t in threads), "the ring hung"
    assert not errors, errors[:3]
    assert sum(done) == 32 * 12
    plan.close()


def test_ticket_collected_twice_is_refused():
    """ticket A collected twice while B of the same batch is outstanding: the second wait is refused and B still gets
    its own rows; tickets that were never issued (an offset inside a live batch, an unknown batch) are refused too"""
    s, plan = ring_plan(slots=2, max_batch=1000, wait_us=RING_WAIT_US)
    A = plan.submit(np.ascontiguousarray(s.X[0:50]))
    B = plan.submit(np.ascontiguousarray(s.X[990:1020]))
    plan.flush()
    batch = A[0] >> 24
    assert B[0] == (batch << 24) | 50
    with pytest.raises(nat.NativeError, match=ERR_INVALID):
        plan.wait(((batch << 24) | 7, 5))
    with pytest.raises(nat.NativeError, match=ERR_INVALID):
        plan.wait(((batch + 5) << 24, 5))
    collect(plan, s, A, slice(0, 50), "A")
    with pytest.raises(nat.NativeError, match=ERR_INVALID):
        plan.wait(A)
    # the slot must not have been recycled: a new batch takes the other slot, and B still holds its rows
    C2 = plan.submit(np.ascontiguousarray(s.X[2000:2040]))
    plan.flush()
    assert C2[0] >> 24 == batch + 1
    collect(plan, s, B, slice(990, 1020), "B")
    collect(plan, s, C2, slice(2000, 2040), "C")
    with pytest.raises(nat.NativeError, match=ERR_INVALID):
        plan.wait(B)
    plan.close()


# ------------------------------------------------------------------------------------------ the library stream
def test_trees3_host_batches_and_enrichment_share_the_library_stream():
    """one thread runs a trees3 plan's host batches while another enriches through the same plan (the three-launch
    fallback, on the library stream too): each result bit-identical to the same call made alone.  Both are warmed
    first with their batches, so the concurrent part never grows the plan's tree scratch"""
    s = served("trees")
    plan = s.plan
    X1 = np.ascontiguousarray(s.X[:3000])
    rng = np.random.default_rng(7)
    keys = rng.permutation(20000).astype(np.int64) * 31 + 5
    table = DeviceTable(keys, np.ascontiguousarray(s.X[20000:40000]))
    ask = keys[rng.integers(0, len(keys), size=4000)]
    want_run = plan.run(X1, with_status=True)
    want_enr = table.enrich(plan, ask)
    want_enr = (want_enr[0].copy(), want_enr[1].copy())
    np.testing.assert_array_equal(want_run[0].view(np.uint32), s.dev_out[:3000].view(np.uint32))
    errors = []

    def loop(call, want, tag):
        try:
            for i in range(200):
                out, st = call()
                if not (np.array_equal(out.view(np.uint32), want[0].view(np.uint32)) and np.array_equal(st, want[1])):
                    errors.append(f"{tag}: iteration {i} differs from the call made alone")
                    return
        except Exception as e:  # noqa: BLE001  (reported by the main thread)
            errors.append(f"{tag}: {e}")

    threads = [threading.Thread(target=loop, args=(lambda: plan.run(X1, with_status=True), want_run, "run_host"), daemon=True),
               threading.Thread(target=loop, args=(lambda: table.enrich(plan, ask), want_enr, "enrich"), daemon=True)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
    assert not any(t.is_alive() for t in threads), "the calls hung"
    table.close()
    assert not errors, errors


# ------------------------------------------------------------------------------------------ merging plans
@pytest.mark.parametrize("how", ["targets", "comm"])
def test_merging_plans_are_refused_on_host_entry_points(how):
    """with merge targets or an attached communicator the kernels store their votes there and not into the batch's
    results: b2s_run_host (small and pipelined) and a ring batch refuse the plan; b2s_run_device still fills the target"""
    s = served("linear")
    want = s.dev_out[:64]
    plan, X, _ = make_plan("linear")
    comm = target = None
    if how == "targets":
        target = nat.DeviceBuffer(4 * (PIPE + 1)).upload(np.full(PIPE + 1, SENT_F, dtype=np.float32))
        plan.set_merge_targets([target.ptr], 1)
    else:
        comm = MergeComm(0, 1, PIPE, plan.out_cols, exchange=None)
        comm.attach(plan)
    try:
        for rows in (np.ascontiguousarray(X[:64]), pinned_rows(X)):
            with pytest.raises(nat.NativeError, match=REFUSED):
                plan.run(rows)
        ticket = plan.submit(np.ascontiguousarray(X[:64]))
        with pytest.raises(nat.NativeError, match=REFUSED):
            plan.wait(ticket)

        local, _ = run_device(plan, Rows(X[:64]))
        assert (local == SENT_F).all(), "with merge targets the local output is not written"
        if how == "targets":
            got = target.download(np.float32, (PIPE + 1,))
            assert got[0] == SENT_F and (got[65:] == SENT_F).all()
            got = got[1:65].reshape(64, 1)
        else:
            ptr, epoch = comm.wait()
            assert epoch == 1, "a refused host batch launched a step of the communicator"
            got = np.empty((64, plan.out_cols), dtype=np.float32)
            nat.check(nat.load().b2s_memcpy_d2h(got.ctypes.data, ptr, got.nbytes))
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    finally:
        if comm is not None:
            comm.detach(plan)
            comm.close()
        plan.close()
