"""The mean vote folded into one linear model inside rowthread_kernel.  Needs an H100: `-m gpu`.

A mean vote of identity scorers is one linear model, sum_k v_k (b_k + w_k . x) = (sum_k v_k w_k) . x + sum_k v_k b_k, so
finalize folds the weights once (b2s_runtime.cu, fold_mean_vote) and the kernel computes one dot product per row instead
of NS.  Such plans report ", mean vote folded" in `plan.kernel`.  A row whose folded score is not finite is scored again
from the per-model tables, so that its stored value is the unfolded vote (NaN where the models' scores disagree in
sign); status words are those of the unfolded plan.  Plans whose weights reach 2^880 are not folded.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store.online import DeviceTable  # noqa: E402
from tests.device_check import Rows, assert_kernel, run_device, run_host  # noqa: E402
from tests.test_gpu_enrichment_paths import (NAN_INF, UNKNOWN, check_enriched, distinct_keys, enrich_dev,  # noqa: E402
                                             ask_keys, lookup_then_run, policy_of, ref_gather, table_values, upload_keys)
from tests.test_gpu_linear_paths import Flow, bands, check_runs, linear, numeric, rowthread, scorers, with_categories  # noqa: E402

FOLDED = ", mean vote folded"
CATS = {c: [0, 1, 2, 3] for c in range(56, 64)}  # the flagship's shape: 56 numeric columns, 8 one-hot sources of 4


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def flagship_flow(n_in=64):
    cats = {c - 64 + n_in: v for c, v in CATS.items()}
    flow = Flow(n_in).imputer({f"f{c}": 0.5 for c in range(0, n_in - 8, 3)}).one_hot({f"f{c}": v for c, v in cats.items()})
    return flow, cats


def ref_vote(models, E, w):
    """the unfolded vote in float64, elementwise (Inf * 0 = NaN as in the kernel): sum_k w_k (b_k + sum_c W_kc E_c)"""
    s = np.zeros(len(E))
    with np.errstate(invalid="ignore"):
        for (_, m), v in zip(models, w):
            s = s + v * ((E * m["W"][0][None, :]).sum(axis=1) + m["b"][0])
    return s


# ------------------------------------------------------------------------------------------ which plans fold
def test_which_plans_fold(sms):
    """the flagship plan (4 identity scorers, mean vote, rowthread<16, 4>) is folded; without a vote, with a majority vote,
    with classifier links and on the dense head (12 models) it is not"""
    flow, _ = flagship_flow()
    w = flow.width
    plan = flow.plan(scorers(w, 4, seed=1), vote=(nat.VOTE_MEAN, [0.25] * 4))
    assert_kernel(plan, rowthread(16, 4), "TMA tensor-map loads", FOLDED)
    assert FOLDED not in flow.plan(scorers(w, 4, seed=1)).kernel
    binary = [linear(w, 1, seed=s, link=nat.LINK_BINARY_GT, classes=[0, 1]) for s in range(3)]
    for vote in ((nat.VOTE_MAJORITY, [0.25, 0.25, 0.5]), (nat.VOTE_MEAN, [0.25, 0.25, 0.5])):
        p = flow.plan(binary, vote=vote)
        assert_kernel(p, rowthread(16, 4))
        assert FOLDED not in p.kernel, p.kernel
    dense = Flow(64).plan(scorers(64, 12, seed=2), vote=(nat.VOTE_MEAN, [1 / 12] * 12))
    assert "dense_head_kernel" in dense.kernel and FOLDED not in dense.kernel, dense.kernel
    one = flow.plan(scorers(w, 1, seed=3), vote=(nat.VOTE_MEAN, [1.0]))
    assert_kernel(one, rowthread(16, 1))
    assert FOLDED not in one.kernel


# ------------------------------------------------------------------------------------------ loaders and tile heights
@pytest.mark.parametrize("n_in", [64, 60])
def test_folded_on_every_loader(sms, n_in):
    """the flagship shape on the tensor map (64 columns) or bulk copies (60), LDGSTS, a host batch; every tile height;
    NaN in imputed and in plain model inputs, Inf in either thread's half of the row"""
    flow, cats = flagship_flow(n_in)
    models = scorers(flow.width, 4, seed=n_in)
    vote = (nat.VOTE_MEAN, [0.25] * 4)
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, rowthread(16, 4), FOLDED)
    sizes = bands(sms)
    X = with_categories(numeric(sizes[-1], n_in, seed=n_in), cats, seed=n_in)
    X[::7, 0] = np.nan  # imputed
    X[5, 1] = np.nan
    X[33, 40] = np.inf
    X[sizes[2] - 1, 2] = -np.inf
    tmap = n_in == 64
    runs = [(Rows(X), n, "rowthread/tma" if tmap else "rowthread/bulk") for n in sizes]
    runs += [(Rows(X, offset=4), n, "rowthread/ldgsts") for n in (33, sizes[3])]
    runs += [("host", 33, "rowthread/host")]
    check_runs(plan, flow, models, X, runs, vote=vote)


@pytest.mark.parametrize("weights", [[0.7, 0.0, 1.3, 0.25], [0.6, 0.0, 0.9], [0.1, 0.2, 0.0, 0.5, 1.7], [-1.0, 3.0]])
def test_folded_vote_weights(sms, weights):
    """weights that are not uniform, include 0, are negative or do not sum to 1; 3 models on NS = 4 and 5 on NS = 8 leave
    padded score slots; NS = 2"""
    flow, cats = flagship_flow()
    models = scorers(flow.width, len(weights), seed=len(weights))
    vote = (nat.VOTE_MEAN, weights)
    plan = flow.plan(models, vote=vote)
    ns = {2: 2, 3: 4, 4: 4, 5: 8}[len(weights)]
    assert_kernel(plan, rowthread(16, ns), FOLDED)
    n = bands(sms)[4]
    X = with_categories(numeric(n, 64, seed=7), cats, seed=7)
    X[50, 3] = np.nan
    check_runs(plan, flow, models, X, [(Rows(X), n, "rowthread/tma"), (Rows(X, offset=4), 5000, "rowthread/ldgsts"),
                                       ("host", 33, "rowthread/host")], vote=vote)


# ------------------------------------------------------------------------------------------ non-finite rows
def test_nonfinite_rows_store_the_unfolded_vote(sms):
    """+-Inf and NaN in columns whose weights differ in sign or are 0 in one model: the stored value has the class
    (NaN / +Inf / -Inf) of the unfolded vote, which the folded weights alone would not give (+Inf under +1 and -3 with
    votes 1/2, 1/2 is NaN unfolded, -Inf folded); status words flag exactly the non-finite rows"""
    n_in = 64
    flow, cats = flagship_flow(n_in)
    w = flow.width
    models = scorers(w, 2, seed=11)
    names = flow.program().out_names
    col = {c: names.index(f"f{c}") for c in (1, 2, 4, 34, 35, 37)}
    for c, ws in {1: (1.0, -3.0), 2: (1.0, 3.0), 4: (0.0, 2.0), 34: (2.0, -2.0), 35: (-1.0, -0.5), 37: (0.0, 0.0)}.items():
        for (_, m), wk in zip(models, ws):
            m["W"][0, col[c]] = wk
    vote = (nat.VOTE_MEAN, [0.5, 0.5])
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, rowthread(16, 2), FOLDED)
    n = bands(sms)[4]
    X = with_categories(numeric(n, n_in, seed=12), cats, seed=12, p_edge=0.0)
    bad = {}
    for i, (c, v) in enumerate([(c, v) for c in (1, 2, 4, 34, 35, 37) for v in (np.inf, -np.inf, np.nan)]):
        for r in (i, 127 - i, 128 + i, n - 1 - i, 1000 + 37 * i):
            X[r, c] = v
            bad[r] = True
    X[2000, 1], X[2000, 34] = np.inf, -np.inf  # two poisoned columns in different thread halves
    X[2001, 2], X[2001, 35] = np.inf, np.inf
    E = flow.expand(X)
    want = ref_vote(models, E, vote[1])
    flagged = ~np.isfinite(E).all(axis=1)
    assert flagged.sum() >= len(bad)
    folded_class = ref_vote([("linear", dict(W=sum(v * m["W"] for (_, m), v in zip(models, vote[1])), b=np.zeros(1)))],
                            E, [1.0])
    assert (np.isnan(want[flagged]) != np.isnan(folded_class[flagged])).any(), "no row where folding changes the class"
    for rows, m, lk in ((Rows(X), n, "rowthread/tma"), (Rows(X, offset=4), n, "rowthread/ldgsts"), ("host", 130, "rowthread/host")):
        out, st = run_host(plan, X[:m]) if rows == "host" else run_device(plan, rows, m)
        assert plan.last_kernel == lk, plan.last_kernel
        o, wv, f = out[:, 0].astype(np.float64), want[:m], flagged[:m]
        np.testing.assert_array_equal(np.isnan(o[f]), np.isnan(wv[f]))
        inf = f & ~np.isnan(wv)
        np.testing.assert_array_equal(o[inf], wv[inf])
        np.testing.assert_array_equal(st, np.where(f, 1, 0))


def test_enrichment_gather_is_folded(sms):
    """the fused gather loader with a folded plan: NaN / Inf stored (a policy on half the columns), unknown keys (all-NaN
    rows, UNKNOWN | NONFINITE), non-uniform votes; against the float64 reference and bit-equal to lookup + run"""
    F = 64
    rng = np.random.default_rng(64)
    tab_keys = distinct_keys(5000, rng)
    vals = table_values(len(tab_keys), F, rng, specials=NAN_INF, p=0.02)
    pol = policy_of("half", F, rng)
    table = DeviceTable(tab_keys, vals, pol)
    flow = Flow(F).imputer({"f3": 0.5})
    models = scorers(flow.width, 4, seed=65)
    vote = (nat.VOTE_MEAN, [0.1, 0.4, 0.0, 0.7])
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, rowthread(16, 4), FOLDED)
    for n in bands(sms):
        ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, n - 1), every=97)
        rows, found = ref_gather(tab_keys, vals, pol, ask)
        d_keys = upload_keys(ask)
        out, st = enrich_dev(table, plan, ask, d_keys=d_keys)
        check_enriched(out, st, flow, models, rows, found, vote=vote)
        assert n < 50 or (st & UNKNOWN).any()
        want = ref_vote(models, flow.expand(rows), vote[1])
        f = (st & 1) != 0
        np.testing.assert_array_equal(np.isnan(out[f, 0]), np.isnan(want[f]))
        out2, st2 = lookup_then_run(table, plan, ask, d_keys=d_keys)
        np.testing.assert_array_equal(out.view(np.uint32), out2.view(np.uint32))
        np.testing.assert_array_equal(st, st2)
    table.close()


# ------------------------------------------------------------------------------------------ the bound
BOUND = 2.0 ** 880
LARGE = [("weight", False), ("bias", False), ("onehot-weight", False), ("folded-magnitude", False), ("below", True)]


@pytest.mark.parametrize("case,folds", LARGE, ids=[c[0] for c in LARGE])
def test_large_weights_are_not_folded(sms, case, folds):
    """a weight, a bias or a one-hot weight at 2^880, or sum_k |v_k w_k| at 2^885 with every weight below 2^880, leaves
    the plan unfolded; weights of 2^879 fold"""
    flow, _ = flagship_flow()
    models = scorers(flow.width, 4, seed=9)
    votes = [0.25] * 4
    m = models[1][1]
    onehot = next(j for j, nm in enumerate(flow.program().out_names) if nm.startswith("f56_"))
    if case == "weight":
        m["W"][0, 3] = BOUND
    elif case == "bias":
        m["b"][0] = -BOUND
    elif case == "onehot-weight":
        m["W"][0, onehot] = BOUND
    elif case == "folded-magnitude":
        m["W"][0, 3] = 2.0 ** 875
        votes = [0.25, 2.0 ** 10, 0.25, 0.25]
    else:
        m["W"][0, 3] = BOUND / 2
    plan = flow.plan(models, vote=(nat.VOTE_MEAN, votes))
    assert_kernel(plan, rowthread(16, 4))
    assert (FOLDED in plan.kernel) == folds, plan.kernel
