"""Linear and transform plans on every kernel that can serve them, against plain float64 references.  Needs an H100:
`-m gpu`.

A linear plan runs on one of two kernel families, chosen when the plan is finalized (b2s_plan_finalize):
  * rowthread_kernel<NCH,NS,TPR,LM>: no MapValues, <= 128 input columns, <= 8 score columns, <= 16 one-hot source columns
    with <= 256 categories in all.  NCH = 4 / 8 / 16 / 32 chunks of 16 bytes per row, NS = 1 / 2 / 4 / 8 score slots, and
    the loader LM is picked per launch, which `last_kernel` reports: "rowthread/tma" (tensor-map boxes, aligned rows of
    exactly 32, 64 or 128 columns), "rowthread/bulk" (one bulk copy per row, other aligned rows), "rowthread/ldgsts"
    (cp.async, rows that are not 16-byte aligned) and "rowthread/host" (cp.async from mapped host memory: a small
    b2s_run_host batch);
  * rows_kernel<LINEAR,NS>: every other linear plan (MapValues, wider rows, more one-hot columns or categories, 9-32 scores
    the dense head does not take), NS = 1 ... 32.
Transform-only plans run on rows_kernel<STORE>.  The dense head has its own file (test_gpu_dense_matrix.py).

Every case asserts `plan.kernel` and, after each run, `plan.last_kernel`.  References are float64: the expanded rows E come
from oracle/batch.py (impute, one_hot, map_values, drop) over the float32 batch and the scores are E @ W.T + b, held to the
bound of tests/device_check.py.  `test_float32_accumulation_breaks_the_bound` shows a float32 accumulator does not fit it.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from oracle import batch as obatch  # noqa: E402
from tests.device_check import (U32, Ref, Rows, assert_kernel, check_close, check_plan_output, names,  # noqa: E402
                                run_device, run_host)

BIG = 2.0 ** 100  # a float32-exact MapValues key no row holds: the column passes through unchanged
EDGES = [0.0, -0.0, 2.5, np.nan, np.inf, -np.inf, 2147483648.0, -2147483648.0, 3e9, -3e9]


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def bands(sms):
    """row counts the launch serves with tiles of 32, 32, 32 (ragged), 64 (ragged) and 128 (ragged) rows: the tile halves
    from 128 while there are fewer tiles than SMs, down to 32"""
    return [1, 33, 32 * sms - 5, 64 * (sms - 1) + 77, 128 * sms + 99]


# ------------------------------------------------------------------------------------------ steps and models
class Flow:
    """feature steps, lowered by ColumnProgram for the device and applied in float64 by oracle/batch.py for the reference"""

    def __init__(self, n_in):
        self.names = names(n_in)
        self.ops = []

    def imputer(self, mapping=None, default=None):
        self.ops.append(("imputer", mapping or {}, default))
        return self

    def one_hot(self, mapping):
        self.ops.append(("one_hot", mapping))
        return self

    def map_values(self, mapping):
        self.ops.append(("map_values", mapping))
        return self

    def drop(self, features):
        self.ops.append(("drop", features))
        return self

    def program(self):
        prog = ColumnProgram(self.names)
        for op in self.ops:
            if op[0] == "imputer":
                prog.imputer(op[1], op[2])
            else:
                getattr(prog, op[0])(op[1])
        return prog

    @property
    def width(self):
        return len(self.program().out_names)

    def expand(self, X):
        E, nm = X.astype(np.float64), list(self.names)
        for op in self.ops:
            if op[0] == "imputer":
                E = obatch.impute(E, nm, op[1], op[2])
            elif op[0] == "one_hot":
                E, nm = obatch.one_hot(E, nm, op[1])
            elif op[0] == "map_values":
                E, nm = obatch.map_values(E, nm, op[1])
            else:
                E, nm = obatch.drop(E, nm, op[1])
        assert nm == self.program().out_names
        return E

    def plan(self, models, vote=None):
        return self.program().build_plan(models, vote=vote)


def linear(width, K=1, seed=0, link=nat.LINK_IDENTITY, classes=None):
    rng = np.random.default_rng(seed)
    return ("linear", dict(W=rng.normal(size=(K, width)), b=rng.normal(size=K), link=link, classes=classes))


def scorers(width, n, seed):
    """n identity scorers of one score each"""
    return [linear(width, 1, seed * 100 + i) for i in range(n)]


def with_categories(X, cats_of, seed, p_edge=0.3):
    """X with the one-hot source columns drawn from their categories, first - 1, last + 1 and the edge values"""
    rng = np.random.default_rng(seed)
    X = X.copy()
    for col, cats in cats_of.items():
        c = np.asarray(cats, dtype=np.float64)
        vals = np.concatenate([c, [c.min() - 1, c.max() + 1], EDGES]).astype(np.float32)
        n_edge = len(vals) - len(c)
        p = np.concatenate([np.full(len(c), (1 - p_edge) / len(c)), np.full(n_edge, p_edge / n_edge)])
        X[:, col] = rng.choice(vals, size=len(X), p=p)
    return X


def numeric(n, n_in, seed):
    return np.random.default_rng(seed).normal(size=(n, n_in)).astype(np.float32)


def rowthread(nch, ns):
    return f"rowthread_kernel<NCH={nch},NS={ns},TPR={2 if nch >= 8 else 1},"


def check_runs(plan, flow, models, X, runs, vote=None):
    """runs: [(rows, n, want_last_kernel)]; rows: Rows over X, or "host" for b2s_run_host of the first n rows"""
    E = flow.expand(X)
    for rows, n, want in runs:
        out, st = run_host(plan, X[:n]) if rows == "host" else run_device(plan, rows, n)
        assert plan.last_kernel == want, (n, plan.last_kernel, want)
        check_plan_output(out, st, models, E[:n], vote=vote)
    return E


# ------------------------------------------------------------------------------------------ the bound itself
def test_float32_accumulation_breaks_the_bound():
    """the score bound is tight enough to catch a float32 accumulator: the plan of test_rowthread_instantiations at
    64 columns (an Imputer, two one-hot sources, 4 scorers), emulated in numpy with the products added in float32"""
    flow = Flow(64).imputer({"f32": 0.5}).one_hot({"f1": [0, 1, 2], "f62": [3, 5, 9, 11, 20]})
    models = scorers(flow.width, 4, seed=16)
    X = with_categories(numeric(5000, 64, seed=1), {1: [0, 1, 2], 62: [3, 5, 9, 11, 20]}, seed=2, p_edge=0.0)
    E = flow.expand(X)
    ref = Ref(models, E)
    broken = []
    for k, (_, m) in enumerate(models):
        acc = np.full(len(E), np.float32(m["b"][0]))
        for j in range(E.shape[1]):
            acc = (acc.astype(np.float64) + E[:, j] * m["W"][0, j]).astype(np.float32)
        tol = U32 * np.abs(ref.pred[:, k]) + ref.bound[:, k]
        broken.append(np.abs(acc - ref.pred[:, k]) > tol)
    assert np.mean(broken) > 0.05, np.mean(broken)


# ------------------------------------------------------------------------------------------ rowthread_kernel: instantiations
N_SCORES = {1: (1, 1), 2: (2, 2), 4: (3, 4), 8: (5, 8)}  # per NS: total score columns at NCH 4/16 and at NCH 8/32


@pytest.mark.parametrize("ns", [1, 2, 4, 8])
@pytest.mark.parametrize("nch", [4, 8, 16, 32])
def test_rowthread_instantiations(sms, nch, ns):
    """rowthread_kernel<NCH, NS, TPR, LM> under every loader.  4*NCH aligned columns take the tensor map (NCH >= 8; bulk
    copies at NCH = 4), 4*NCH - 4 aligned columns the per-row bulk copies; both again from a base 4 bytes off alignment
    (LDGSTS) and as a small host batch.  1-8 identity scorers (3 and 5 leave padded slots), an Imputer, a dense and a
    sparse (or a second dense: cats_fast) one-hot source, NaN / Inf in model inputs; every tile height"""
    n_scores = N_SCORES[ns][nch in (8, 32)]
    for n_in in (4 * nch, 4 * nch - 4):
        second = list(range(4, 9)) if ns in (1, 4) else [3, 5, 9, 11, 20]
        cats = {1: [0, 1, 2], n_in - 2: second}
        flow = Flow(n_in).imputer({f"f{n_in // 2}": 0.5}).one_hot({f"f{c}": v for c, v in cats.items()})
        models = scorers(flow.width, n_scores, seed=nch + ns + n_in)
        plan = flow.plan(models)
        tmap = nch >= 8 and n_in == 4 * nch
        assert_kernel(plan, rowthread(nch, ns), "TMA tensor-map loads" if tmap else "TMA bulk loads")
        sizes = bands(sms)
        X = with_categories(numeric(sizes[-1], n_in, seed=n_in + ns), cats, seed=ns)
        X[::7, n_in // 2] = np.nan
        X[17, 0] = np.inf
        X[40, n_in - 1] = np.nan
        X[sizes[2] - 1, n_in - 3] = -np.inf
        aligned, off4 = Rows(X), Rows(X, offset=4)
        runs = [(aligned, n, "rowthread/tma" if tmap else "rowthread/bulk") for n in sizes]
        runs += [(off4, n, "rowthread/ldgsts") for n in (33, sizes[3])]
        runs += [("host", 33, "rowthread/host")]
        check_runs(plan, flow, models, X, runs)


@pytest.mark.parametrize("nch,ns", [(4, 2), (8, 1), (16, 4)])
def test_rowthread_stage_ring_turns_over(sms, nch, ns):
    """at least four tiles per CTA at any grid the launch can have (2048 threads per SM): the stage ring wraps, the
    mbarrier parities flip, and with the tensor map and NS >= 4 the single-barrier loop double-buffers its partial sums"""
    n_in = 4 * nch
    tpr = 2 if nch >= 8 else 1
    n = 4 * (2048 // (128 * tpr)) * sms * 128 + 77
    flow = Flow(n_in).one_hot({"f2": [0, 1, 2, 3]})
    models = scorers(flow.width, {1: 1, 2: 2, 4: 4}[ns], seed=nch)
    plan = flow.plan(models)
    tmap = nch >= 8
    assert_kernel(plan, rowthread(nch, ns))
    X = with_categories(numeric(n, n_in, seed=nch), {2: [0, 1, 2, 3]}, seed=nch)
    X[n - 1, 0] = np.nan
    X[n // 2, n_in - 1] = np.inf
    check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma" if tmap else "rowthread/bulk")])


# ------------------------------------------------------------------------------------------ rowthread_kernel: dead tail
DEAD = [  # (n_in, steps, expected dead_tail)
    (64, "plain", 0),
    (32, "onehot-last-9", 2),
    (64, "onehot-last-15", 3),
    (32, "onehot-last-16", 4),
    (128, "drop-last-8", 2),
    (64, "drop-last-20", 5),
    (128, "onehot-last-6+drop-last-12", 4),
]


@pytest.mark.parametrize("n_in,steps,dead", DEAD, ids=[d[1] + f"-{d[0]}" for d in DEAD])
def test_rowthread_dead_tail(sms, n_in, steps, dead):
    """trailing chunks without a model input are skipped on the tensor-map loader (LIVE = NCH, NCH - 2, NCH - 4): trailing
    one-hot sources and trailing DropFeatures columns, NaN / Inf in them (never flagged); every tile height"""
    flow = Flow(n_in).imputer({"f0": 0.25})
    cats, dropped = {}, []
    for part in steps.split("+"):
        if part.startswith("onehot"):
            k = int(part.split("-")[-1])
            cats = {c: [0, 1, 2] for c in range(n_in - k, n_in)}
        elif part.startswith("drop"):
            k = int(part.split("-")[-1])
            dropped = list(range(n_in - k - len(cats), n_in - len(cats)))
    if cats:
        flow.one_hot({f"f{c}": v for c, v in cats.items()})
    if dropped:
        flow.drop([f"f{c}" for c in dropped])
    last_input = max(c for c in range(n_in) if c not in cats and c not in dropped)
    assert n_in // 4 - 1 - last_input // 4 == dead
    nch = n_in // 4
    models = scorers(flow.width, 2 if dead % 2 else 4, seed=n_in + dead)
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(nch, 2 if dead % 2 else 4), "TMA tensor-map loads")
    sizes = bands(sms)
    X = with_categories(numeric(sizes[-1], n_in, seed=dead), cats, seed=dead)
    for c in dropped:
        X[c::11, c] = [np.nan, np.inf, -np.inf][c % 3]
    X[3, last_input] = np.nan
    X[::5, 0] = np.nan
    check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma") for n in sizes[1:]])


# ------------------------------------------------------------------------------------------ rowthread_kernel: one-hot columns
FAST_CATS = [range(-3, 2), [7], range(8388600, 8388605), range(0, 16), range(10, 13), range(-1, 1), range(100, 104),
             range(0, 3), range(5, 25), range(-20, -10), range(1, 2), range(0, 8), range(3, 6), range(0, 2), range(40, 70),
             range(0, 4)]
# per-column paths: dense columns beside sparse ones, <= 4 categories searched inline, more in cat_val; a first code of
# 2^23 is not taken as dense
SEARCH_CATS = [range(-3, 2), [7, 3], range(8388608, 8388613), [3, 7, 11, 40], range(10, 13), [-1, 5, 6], [2, 4, 6, 8, 10, 12],
               range(0, 3), [100, 300], range(-20, -10), [0.5], range(0, 8), [1, 2, 4, 8, 16, 32, 64], range(0, 2),
               [8388607, 8388608], range(0, 4)]


def spread(n_in, k=16):
    """k one-hot source columns over all 8 chunk phases and every 32-column box: the first column, columns between
    numeric ones and the last column"""
    nch = n_in // 4
    chunks = [2 * i + (i // 4) % 2 for i in range(16)] if nch == 32 else list(range(min(nch, k)))
    return [4 * ch + i % 4 if 4 * ch + i % 4 < n_in else n_in - 1 for i, ch in enumerate(chunks)][:k]


@pytest.mark.parametrize("n_in", [128, 64, 32])
@pytest.mark.parametrize("path", ["cats_fast", "search"])
def test_rowthread_onehot_positions_and_index_paths(sms, n_in, path):
    """one-hot sources at every chunk phase and in every tensor-map box (swizzled reads), through cats_fast (consecutive
    integer codes: a negative first code, a single category, a first code just below 2^23) or the per-column paths (dense,
    inline search, cat_val search; 2^23 and above search).  Values: every category, first - 1, last + 1, +-0, 2.5, NaN with
    an Imputer fill that is a category / one that is not / none, +-Inf, +-2^31, +-3e9.  Every tile height, the padded
    tile (LDGSTS) and a host batch"""
    cols = spread(n_in)
    lists = FAST_CATS if path == "cats_fast" else SEARCH_CATS
    cats = {c: list(lists[i]) for i, c in enumerate(cols)}
    fills = {f"f{cols[0]}": -2.0, f"f{cols[1]}": 0.5}  # a category of its column / not one
    fills[f"f{[c for c in range(n_in) if c not in cats][0]}"] = 0.75
    flow = Flow(n_in).imputer(fills).one_hot({f"f{c}": v for c, v in cats.items()})
    ns = 2 if path == "cats_fast" else 4
    models = scorers(flow.width, ns, seed=n_in)
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(n_in // 4, ns), "TMA tensor-map loads")
    sizes = bands(sms)
    X = with_categories(numeric(sizes[-1], n_in, seed=n_in), cats, seed=n_in + ns, p_edge=0.4)
    first_num = [c for c in range(n_in) if c not in cats]
    X[::17, first_num[0]] = np.nan  # imputed
    X[5, first_num[-1]] = np.nan  # flags row 5
    E = check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma") for n in sizes[1:]])
    check_runs(plan, flow, models, X, [(Rows(X, offset=4), sizes[3], "rowthread/ldgsts"), ("host", 33, "rowthread/host")])
    onehot = [j for j, nm in enumerate(flow.program().out_names) if "_" in nm]
    assert E[:, onehot].sum(axis=0).min() > 0, "a category never occurs"


@pytest.mark.parametrize("case", ["1-col", "16-cols", "17-cols", "256-cats", "257-cats"])
def test_rowthread_onehot_limits(sms, case):
    """1 and 16 categorical columns stay on rowthread, 17 move to rows_kernel; 256 categories in all stay, 257 move"""
    n_in = 40
    if case.endswith(("col", "cols")):
        k = int(case.split("-")[0])
        cats = {c: [0, 1, 2] for c in range(1, 2 * k, 2)}
    else:
        k = int(case.split("-")[0])
        cats = {3: list(range(-50, 150)), 30: list(range(1000, 1000 + k - 200))}
    flow = Flow(n_in).one_hot({f"f{c}": v for c, v in cats.items()})
    models = scorers(flow.width, 3, seed=k)
    plan = flow.plan(models)
    stays = case in ("1-col", "16-cols", "256-cats")
    assert_kernel(plan, rowthread(16, 4) if stays else "rows_kernel<LINEAR,NS=4>")
    X = with_categories(numeric(5000, n_in, seed=k), cats, seed=k)
    X[9, 0] = np.nan
    check_runs(plan, flow, models, X, [(Rows(X), 5000, "rowthread/bulk" if stays else "rows")])


# ------------------------------------------------------------------------------------------ rowthread_kernel: epilogues
@pytest.mark.parametrize("weights", [[0.7, 0.0, 1.3, 0.25], [0.6, 0.0, 0.9], [0.1, 0.2, 0.0, 0.5, 1.7]])
def test_rowthread_fast_mean_vote(sms, weights):
    """the fast epilogue's mean vote with weights that are not uniform, include 0 and do not sum to 1 (NS = 4 / 8), on
    the tensor map (64 columns) and bulk copies (60 columns)"""
    for n_in in (64, 60):
        flow = Flow(n_in).one_hot({"f7": [0, 1, 2]})
        models = scorers(flow.width, len(weights), seed=n_in)
        vote = (nat.VOTE_MEAN, weights)
        plan = flow.plan(models, vote=vote)
        assert_kernel(plan, rowthread(16, 4 if len(weights) <= 4 else 8))
        n = bands(sms)[3]
        X = with_categories(numeric(n, n_in, seed=len(weights)), {7: [0, 1, 2]}, seed=1)
        X[50, 3] = np.nan
        check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma" if n_in == 64 else "rowthread/bulk"),
                                           ("host", 33, "rowthread/host")], vote=vote)


def logistic3(E, labels, seed):
    from sklearn.linear_model import LogisticRegression

    rng = np.random.default_rng(seed)
    z = E[:, 0] + 0.5 * E[:, 2] + 0.3 * rng.normal(size=len(E))
    y = np.asarray(labels)[np.digitize(z, np.quantile(z, [1 / 3, 2 / 3]))]
    return packing.pack_model(LogisticRegression(max_iter=300).fit(E, y))


EPILOGUES = ["binary", "argmax", "majority-ties", "majority-negative"]


@pytest.mark.parametrize("case", EPILOGUES)
def test_rowthread_generic_epilogue(sms, case):
    """the generic epilogue: binary `>` with non-contiguous and negative labels, a 3-class LogisticRegression between two
    binary models (its scores sit at offset 1, the third model's at 4: score_off differs from the model index), and
    majority votes with weighted ties and with a negative label (status bit 2)"""
    n_in = 32
    flow = Flow(n_in).imputer({"f5": 1.0}).one_hot({"f30": [0, 1, 2, 3]})
    n = bands(sms)[4]
    X = with_categories(numeric(n, n_in, seed=3), {30: [0, 1, 2, 3]}, seed=3)
    X[::9, 5] = np.nan
    X[77, 6] = np.nan
    E = flow.expand(X)
    w = flow.width
    b1 = linear(w, 1, seed=1, link=nat.LINK_BINARY_GT, classes=[-3, 5])
    b2 = linear(w, 1, seed=2, link=nat.LINK_BINARY_GT, classes=[0, 1] if case != "majority-negative" else [-1, 1])
    b3 = linear(w, 1, seed=3, link=nat.LINK_BINARY_GT, classes=[0, 1])
    vote = None
    if case == "binary":
        models = [b1, b2]
    elif case == "argmax":
        fit = E[:3000][np.isfinite(E[:3000]).all(axis=1)]
        models = [b1, logistic3(fit, [-4, 2, 9], seed=4), b2]
    else:
        b1 = linear(w, 1, seed=1, link=nat.LINK_BINARY_GT, classes=[1, 0])
        models = [b1, b2, b3]
        vote = (nat.VOTE_MAJORITY, [0.25, 0.25, 0.5])
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, rowthread(8, 8 if case == "argmax" else (2 if case == "binary" else 4)), "TMA tensor-map loads")
    runs = [(Rows(X), n, "rowthread/tma"), (Rows(X, offset=4), 5000, "rowthread/ldgsts"), ("host", 33, "rowthread/host")]
    check_runs(plan, flow, models, X, runs, vote=vote)
    ref = Ref(models, E)
    if case == "majority-ties":  # rows where models 0 + 1 outvote model 2 only by a tie of 0.5 vs 0.5
        assert ((ref.pred[:, 0] == ref.pred[:, 1]) & (ref.pred[:, 0] != ref.pred[:, 2])).any()
    if case == "majority-negative":
        out, st = run_device(plan, Rows(X), n)
        assert ((st & 2) != 0).any() and ((st & 2) == 0).any()


# ------------------------------------------------------------------------------------------ rowthread_kernel: status, strides
def test_rowthread_status_words(sms):
    """NaN / +-Inf in a model input of either per-thread column slice (TPR = 2: columns 0-31 and 32-63) flags its row
    only; in an imputed column, a dropped column or a one-hot source it flags nothing.  Bad rows sit at tile edges"""
    n_in = 64
    flow = Flow(n_in).imputer({"f10": 0.25}).one_hot({"f20": [0, 1], "f50": [4, 5, 6]}).drop(["f40"])
    models = scorers(flow.width, 3, seed=5)
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(16, 4), "TMA tensor-map loads")
    n = bands(sms)[4]
    X = with_categories(numeric(n, n_in, seed=6), {20: [0, 1], 50: [4, 5, 6]}, seed=6, p_edge=0.0)
    cells = {3: (5, np.nan), 4: (45, np.inf), 5: (31, -np.inf), 6: (32, np.nan), 127: (0, np.nan), 128: (63, -np.inf),
             7: (10, np.nan), 8: (40, np.inf), 9: (20, np.nan), 10: (50, -np.inf), 129: (40, np.nan), n - 1: (33, np.inf)}
    for r, (c, v) in cells.items():
        X[r, c] = v
    E = check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma"), (Rows(X, offset=4), n, "rowthread/ldgsts"),
                                           ("host", 130, "rowthread/host")])
    flagged = ~np.isfinite(E).all(axis=1)
    assert sorted(np.flatnonzero(flagged)) == [3, 4, 5, 6, 127, 128, n - 1]


@pytest.mark.parametrize("n_in,pad,want", [(64, 48, "rowthread/tma"), (60, 16, "rowthread/bulk"), (64, 4, "rowthread/ldgsts"),
                                           (63, 0, "rowthread/ldgsts"), (31, 0, "rowthread/ldgsts")])
def test_rowthread_strided_and_odd_rows(sms, n_in, pad, want):
    """rows `pad` bytes further apart than 4 * n_in: a multiple of 16 keeps the tensor map / bulk copies, 4 bytes take
    LDGSTS; rows of 63 and 31 columns (not whole 16-byte chunks) take LDGSTS"""
    nch = next(b for b in (4, 8, 16, 32) if 4 * b >= n_in)
    flow = Flow(n_in).imputer({"f1": 0.5}).one_hot({"f4": [0, 1, 2], f"f{n_in - 1}": [1, 3]})
    models = scorers(flow.width, 2, seed=n_in)
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(nch, 2))
    n = bands(sms)[4]
    X = with_categories(numeric(n, n_in, seed=n_in), {4: [0, 1, 2], n_in - 1: [1, 3]}, seed=pad)
    X[::13, 1] = np.nan
    X[21, 2] = np.nan
    check_runs(plan, flow, models, X, [(Rows(X, stride=4 * n_in + pad), m, want) for m in (33, n)])


# ------------------------------------------------------------------------------------------ rows_kernel<LINEAR, NS>
def all_mapped(flow_names, special):
    """MapValues keeps only the columns it maps: every column gets a map (`special` ones theirs, the others a key no
    row holds)"""
    return {n: special.get(n, {BIG: 0.0}) for n in flow_names}


ROWS_CASES = [  # (case, n_in, score columns, NS)
    ("value-map", 40, 1, 1), ("value-map", 64, 2, 2), ("range-map", 7, 1, 1), ("range-map", 20, 2, 2),
    ("chained-maps", 9, 3, 4), ("chained-maps", 44, 4, 4), ("map-onehot", 48, 5, 8), ("map-onehot", 24, 8, 8),
    ("wide", 129, 8, 8), ("wide", 300, 1, 1), ("17-cat-cols", 40, 4, 4), ("257-cats", 24, 8, 8),
    ("onehot-scores", 30, 12, 16), ("onehot-scores", 6, 9, 16), ("onehot-scores", 30, 32, 32), ("majority", 20, 12, 16),
]


def rows_case(case, n_in, n_scores):
    """flow, models, vote and the categorical columns of one rows_kernel case"""
    flow, cats, vote = Flow(n_in), {}, None
    nm = flow.names
    if case == "value-map":
        flow.map_values(all_mapped(nm, {n: {0: 10, 1: -2, 2: 0.5} for n in nm[::3]}))
    elif case == "range-map":
        flow.imputer({"f0": 0.25})
        flow.map_values(all_mapped(nm, {n: {"ranges": {1: ["-inf", -0.5], 2: [-0.5, 0.5], 3: [0.5, "inf"]}} for n in nm[::2]}))
    elif case == "chained-maps":  # the second map sees the first one's output; within a map the first hit wins
        flow.map_values(all_mapped(nm, {n: {0: 5, 5: 7, 1: 1} for n in nm[::2]}))
        flow.map_values(all_mapped(nm, {n: {5: 9, 7: 1, 1: 4} for n in nm[::2]}))
    elif case == "map-onehot":
        flow.map_values(all_mapped(nm, {"f0": {0: 10, 1: 11}, "f3": {"ranges": {1: ["-inf", 0], 2: [0, "inf"]}}}))
        cats = {0: [10, 11, 2], 3: [1, 2]}
        flow.one_hot({"f0": [10, 11, 2], "f3": [1, 2]})
    elif case == "wide":
        cats = {5: [0, 1, 2], n_in // 2: [3, 7], n_in - 1: [0, 1]}
        flow.imputer({"f1": 0.5}).one_hot({f"f{c}": v for c, v in cats.items()})
    elif case == "17-cat-cols":
        cats = {c: [0, 1, 2] for c in range(0, 34, 2)}
        flow.one_hot({f"f{c}": v for c, v in cats.items()})
    elif case == "257-cats":
        cats = {2: list(range(200)), 20: list(range(-57, 0))}
        flow.one_hot({f"f{c}": v for c, v in cats.items()})
    elif case in ("onehot-scores", "majority"):
        cats = {1: [0, 1, 2, 3]}
        flow.one_hot({"f1": [0, 1, 2, 3]})
    w = flow.width
    if case == "majority":
        models = [linear(w, 1, seed=s, link=nat.LINK_BINARY_GT, classes=[s % 3, 3 + s % 2]) for s in range(n_scores)]
        vote = (nat.VOTE_MAJORITY, list(np.random.default_rng(1).random(n_scores)))
    elif n_scores == 32:
        models = [linear(w, 16, seed=s, link=nat.LINK_ARGMAX, classes=list(range(-5, 27, 2))) for s in range(2)]
    else:
        models = scorers(w, n_scores, seed=n_in)
    return flow, models, vote, cats


def rows_data(case, n, n_in, cats, seed):
    X = numeric(n, n_in, seed)
    if case in ("value-map", "chained-maps", "map-onehot"):
        ints = np.random.default_rng(seed).integers(-1, 8, size=X.shape).astype(np.float32)
        X[:, ::2] = ints[:, ::2]
    X = with_categories(X, cats, seed)
    X[7, n_in - 1 if n_in - 1 not in cats else 0] = np.nan
    return X


@pytest.mark.parametrize("case,n_in,n_scores,ns", ROWS_CASES, ids=[f"{c[0]}-{c[1]}x{c[2]}" for c in ROWS_CASES])
def test_rows_kernel_linear(sms, case, n_in, n_scores, ns):
    """rows_kernel<LINEAR, NS> for each reason a plan lands there: value / range / chained maps, a MapValues feeding a
    OneHotEncoder, rows wider than 128 columns (fast and generic chunks side by side), 17 one-hot columns, 257 categories,
    9-32 scores behind a OneHotEncoder, a majority vote of 12 models.  NS = 1 ... 32 with 4 threads per row and with
    narrow rows cutting that to 2 and 1; every tile height of the small-batch shrink"""
    flow, models, vote, cats = rows_case(case, n_in, n_scores)
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, f"rows_kernel<LINEAR,NS={ns}>")
    sizes = bands(sms)
    X = rows_data(case, sizes[-1], n_in, cats, seed=n_in + n_scores)
    rows = Rows(X)
    check_runs(plan, flow, models, X, [(rows, n, "rows") for n in sizes] + [("host", 9, "rows")], vote=vote)


def test_seventeen_models_are_refused():
    """a plan holds at most 16 models: the 17th is a loud error"""
    flow = Flow(8)
    prog = flow.program()
    models = [linear(8, 1, seed=s, link=nat.LINK_BINARY_GT, classes=[0, 1]) for s in range(17)]
    with pytest.raises(nat.NativeError, match="more than 16 models"):
        prog.build_plan(models, vote=(nat.VOTE_MAJORITY, [1.0] * 17))
    prog.build_plan(models[:16], vote=(nat.VOTE_MAJORITY, [1.0] * 16))


def test_rows_kernel_widest_row(sms):
    """the widest row rows_kernel<LINEAR, NS=32> accepts (found by bisection of finalize) computes the reference; one
    column more is refused by the shared-memory check with a loud error"""
    def flow_of(n_in):
        return Flow(n_in).one_hot({f"f{n_in - 1}": [0, 1]})

    def models_of(flow):
        return [linear(flow.width, 16, seed=s, link=nat.LINK_ARGMAX, classes=list(range(16))) for s in range(2)]

    def accepted(n_in):
        flow = flow_of(n_in)
        try:
            flow.plan(models_of(flow))
        except nat.NativeError as e:
            assert "shared memory" in str(e), e
            return False
        return True

    lo, hi = 64, 4096
    assert accepted(lo) and not accepted(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if accepted(mid) else (lo, mid)
    flow = flow_of(lo)
    models = models_of(flow)
    plan = flow.plan(models)
    assert_kernel(plan, "rows_kernel<LINEAR,NS=32>")
    X = with_categories(numeric(3000, lo, seed=lo), {lo - 1: [0, 1]}, seed=1)
    X[11, 5] = np.inf
    check_runs(plan, flow, models, X, [(Rows(X), n, "rows") for n in (1, 33, 3000)])
    with pytest.raises(nat.NativeError, match="shared memory"):
        flow_of(lo + 1).plan(models_of(flow_of(lo + 1)))


# ------------------------------------------------------------------------------------------ rows_kernel<STORE>
STORE_CASES = [1, 3, 13, 64, 129]


def store_flow(n_in):
    f = Flow(n_in)
    nm = f.names
    if n_in == 1:
        f.imputer({"f0": 1.0}).map_values({"f0": {"ranges": {0: ["-inf", 0], 1: [0, 2]}}}).map_values({"f0": {0: 5, 1: 0}})
        return f.one_hot({"f0": [5, 0, 2.5]}), {}
    if n_in == 3:
        f.imputer(default=0.25).map_values({"f0": {1: 2, 2: 3}, "f2": {"ranges": {7: ["-inf", -1]}}})
        return f.map_values({"f0": {3: 4}, "f2": {7: -7}}), {}
    cats = {c: [0, 1, 2] for c in range(2, n_in, max(3, n_in // 8))}
    f.imputer({nm[0]: 0.5, nm[2]: 1.0}).one_hot({nm[c]: v for c, v in cats.items()})
    return f.drop([nm[1], nm[n_in - 2]] if n_in - 2 not in cats else [nm[1]]), cats


@pytest.mark.parametrize("n_in", STORE_CASES)
def test_store_plans_are_bit_exact(sms, n_in):
    """transform-only plans (rows_kernel<STORE>) against the oracle transforms bit for bit: Imputer, chained MapValues,
    OneHotEncoder, DropFeatures; status words 0, the row past the end untouched"""
    flow, cats = store_flow(n_in)
    plan = flow.program().build_plan([])
    assert_kernel(plan, "rows_kernel<STORE,NS=1>")
    n = bands(sms)[3]
    rng = np.random.default_rng(n_in)
    X = (rng.normal(size=(n, n_in)) * 2).astype(np.float32)
    X[:, ::2] = np.round(X[:, ::2])
    X = with_categories(X, cats, seed=n_in)
    X[::5, 0] = np.nan
    X[3, n_in - 1] = -0.0
    E = flow.expand(X).astype(np.float32)
    for rows, m in ((Rows(X), n), (Rows(X), 1), (Rows(X, offset=4), 777)):
        out, st = run_device(plan, rows, m)
        assert plan.last_kernel == "store"
        same = (out.view(np.uint32) == E[:m].view(np.uint32)) | (np.isnan(out) & np.isnan(E[:m]))
        assert same.all(), np.argwhere(~same)[:5]
        assert not st.any()


# ------------------------------------------------------------------------------------------ one plan on two kernels
def test_same_plan_on_rowthread_and_rows_kernel(sms):
    """one linear plan on rowthread (tensor map, LDGSTS, host; a 64-column plan never takes bulk copies), and again on
    rows_kernel, forced by a MapValues on every column whose key (2^100) no row holds: both within the bound of the same
    reference (not bitwise: the kernels split the sum differently)"""
    n_in = 64
    cats = {9: [0, 1, 2], 40: [1, 3, 5, 7, 9]}
    fast = Flow(n_in).imputer({"f0": 0.5}).one_hot({f"f{c}": v for c, v in cats.items()})
    slow = Flow(n_in).imputer({"f0": 0.5}).map_values(all_mapped(names(n_in), {})).one_hot({f"f{c}": v for c, v in cats.items()})
    models = scorers(fast.width, 3, seed=64)
    n = bands(sms)[4]
    X = with_categories(numeric(n, n_in, seed=8), cats, seed=8)
    X[::3, 0] = np.nan
    X[5, 1] = np.nan
    np.testing.assert_array_equal(fast.expand(X[:2000]), slow.expand(X[:2000]))
    p1 = fast.plan(models)
    assert_kernel(p1, rowthread(16, 4), "TMA tensor-map loads")
    E = check_runs(p1, fast, models, X, [(Rows(X), n, "rowthread/tma"), (Rows(X, offset=4), n, "rowthread/ldgsts"),
                                         ("host", 33, "rowthread/host")])
    ref = Ref(models, E)
    out_rt, _ = run_device(p1, Rows(X), n)
    p2 = slow.plan(models)
    assert_kernel(p2, "rows_kernel<LINEAR,NS=4>")
    out_rows, _ = run_device(p2, Rows(X), n)
    assert p2.last_kernel == "rows"
    ok = np.isfinite(E).all(axis=1)
    for out in (out_rt, out_rows):
        check_close(out[ok], ref.pred[ok], ref.bound[ok], "scores")
    check_close(out_rt[ok], out_rows[ok].astype(np.float64), 2 * ref.bound[ok] + U32 * np.abs(ref.pred[ok]), "rowthread vs rows")
