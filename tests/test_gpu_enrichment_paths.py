"""Online enrichment on every path that can serve it, against plain float64 references.  Needs an H100: `-m gpu`.

A batch of entity keys reaches the scoring plan one of three ways (csrc/b2s_table.cu):
  * table_lookup_kernel (b2s_table_lookup_host / _device): one lane probes per key, then rows are copied by sub-warps of
    n_feat / 4 lanes when that is a power of two <= 32 (F = 4 ... 128: lanes_per_row 1 ... 32), by the whole warp in
    16-byte words for other multiples of 4 (F > 128 loops `c += 128`), and 4 bytes at a time when F % 4 != 0, the stride
    is not a multiple of 16 bytes or the rows' base is not 16-byte aligned;
  * the gather loader of rowthread_kernel<NCH, NS, TPR, LM = 1> (b2s_table_enrich_device, and b2s_table_enrich_host
    when the plan is fusable): each tile row's key is probed one tile ahead (g_probe_finish) and its row fetched with
    one bulk copy; the table's impute policy folds into the plan's Imputer operands.  `last_kernel` is "rowthread/bulk";
  * the fallback of b2s_table_enrich_host for plans the loader declines: lookup, the plan's launches (three for trees3),
    then mark_unknown_kernel.

References: gathered rows are a lookup of the table's keys in numpy, then `~isfinite -> policy` wherever the policy is
not NaN; unknown keys give an all-NaN row.  Rows are compared bit for bit (NaN payloads, +-FLT_MAX, -0.0 and denormals
survive), found flags and status words exactly.  Scores use the expanded rows E of oracle/batch.py and E @ W.T + b in
float64, held to the bound of tests/device_check.py (the dense head to its own bound, tests/test_gpu_dense_matrix.py).
"""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200.feature_store.online import DeviceTable  # noqa: E402
from tests import table_hash as th  # noqa: E402
from tests.device_check import SENT_F, SENT_I, assert_kernel, check_plan_output, names  # noqa: E402
from tests.test_gpu_linear_paths import Flow, all_mapped, bands, rowthread, scorers  # noqa: E402

UNKNOWN, NONFINITE = nat.ROW_UNKNOWN_KEY, nat.ROW_NONFINITE_INPUT
SENT_BITS = np.float32(SENT_F).view(np.uint32)
# stored values the lookup must copy as they are unless a policy applies: NaN payloads (quiet, negative, signalling),
# +-Inf (always imputed where a policy is set), +-FLT_MAX, -0.0 and denormals (never imputed)
SPECIALS = np.array([0x7FC12345, 0xFFC0BEEF, 0x7F800001, 0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x80000000,
                     0x00000001, 0x807FFFFF], dtype=np.uint32).view(np.float32)
NAN_INF = np.array([np.nan, np.inf, -np.inf], dtype=np.float32)


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


# ------------------------------------------------------------------------------------------ tables, keys and references
def distinct_keys(n, rng, exclude=None):
    keys = np.unique(rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=2 * n + 16, dtype=np.int64))
    if exclude is not None:
        keys = keys[~np.isin(keys, exclude)]
    return rng.permutation(keys)[:n]


def table_values(n_keys, F, rng, specials=SPECIALS, p=0.08):
    """normal values; row j < len(specials) is all specials[j], and a fraction p of the other cells a random special"""
    vals = rng.normal(size=(n_keys, F)).astype(np.float32)
    hit = rng.random(vals.shape) < p
    vals[hit] = rng.choice(specials, size=int(hit.sum()))
    k = min(len(specials), n_keys)
    vals[:k] = specials[:k, None]
    return vals


def policy_of(kind, F, rng):
    """the table's impute vector: none, every column, or the even columns (the odd ones keep what is stored)"""
    if kind == "none":
        return None
    pol = rng.normal(size=F).astype(np.float32)
    if kind == "half":
        pol[1::2] = np.nan
    return pol


def ask_keys(tab_keys, n, rng, unknown_rows=(), every=None):
    """n keys drawn from the table, with keys it does not hold at `unknown_rows` and every `every`-th row"""
    ask = tab_keys[rng.integers(0, len(tab_keys), size=n)]
    rows = [r for r in unknown_rows if 0 <= r < n]
    if every:
        rows += list(range(every // 2, n, every))
    rows = np.unique(np.asarray(rows, dtype=np.int64))
    if len(rows):
        ask[rows] = distinct_keys(len(rows), rng, exclude=tab_keys)
    return ask


def ref_gather(tab_keys, vals, policy, ask):
    """(rows, found): the table's rows for the asked keys, NaN rows for unknown keys, then the policy"""
    order = np.argsort(tab_keys)
    srt = tab_keys[order]
    pos = np.minimum(np.searchsorted(srt, ask), len(srt) - 1)
    found = srt[pos] == ask
    rows = np.where(found[:, None], vals[order[pos]], np.float32(np.nan)).astype(np.float32)
    if policy is not None:
        fill = ~np.isfinite(rows) & ~np.isnan(policy)[None, :]
        rows = np.where(fill, policy[None, :], rows)
    return rows, found


def assert_rows(got, want, found, tag=""):
    """bit-exact, except that an unknown key's NaN is any NaN"""
    g, w = got.view(np.uint32), want.view(np.uint32)
    same = (g == w) | (~found[:, None] & np.isnan(got) & np.isnan(want))
    assert same.all(), (tag, int((~same).sum()), np.argwhere(~same)[:5], g[~same][:5], w[~same][:5])


def capacity_of(table):
    cap = C.c_int64()
    nat.check(nat.load().b2s_table_info(table._h, None, None, C.byref(cap)))
    return cap.value


# ------------------------------------------------------------------------------------------ running the three paths
def upload_keys(ask):
    return nat.DeviceBuffer(8 * len(ask)).upload(np.asarray(ask, dtype=np.int64))


def lookup_dev(table, ask, stride=None, offset=0, d_keys=None):
    """b2s_table_lookup_device into rows `stride` bytes apart, `offset` bytes past a buffer filled with sentinels: the
    pad words of every row, the words before row 0, row n and found[n] must keep them.  -> (rows, found, rows buffer)"""
    n, F = len(ask), table.n_feat
    stride = 4 * F if stride is None else stride
    words = stride // 4
    buf0 = np.full(offset // 4 + (n + 1) * words, SENT_BITS, dtype=np.uint32)
    d_rows = nat.DeviceBuffer(buf0.nbytes).upload(buf0)
    d_found = nat.DeviceBuffer(4 * (n + 1)).upload(np.full(n + 1, SENT_I, dtype=np.int32))
    d_keys = d_keys or upload_keys(ask)
    table.lookup_device(d_keys.ptr, n, d_rows.ptr + offset, stride, d_found.ptr)
    raw = d_rows.download(np.uint32, buf0.shape)
    found = d_found.download(np.int32, (n + 1,))
    assert (raw[:offset // 4] == SENT_BITS).all(), "a word before row 0 was written"
    rows = raw[offset // 4:].reshape(n + 1, words)
    assert (rows[:n, F:] == SENT_BITS).all(), "a pad word was written"
    assert (rows[n] == SENT_BITS).all() and found[n] == SENT_I, "a row past the end was written"
    assert set(np.unique(found[:n]).tolist()) <= {0, 1}
    return np.ascontiguousarray(rows[:n, :F]).view(np.float32), found[:n].astype(bool), d_rows


def sentinel_out(plan, n):
    sent = SENT_I if plan.out_is_int else SENT_F
    out0 = np.full((n + 1, plan.out_cols), sent, dtype=plan.out_dtype)
    return nat.DeviceBuffer(out0.nbytes).upload(out0), nat.DeviceBuffer(4 * (n + 1)).upload(np.full(n + 1, -1, dtype=np.int32))


def download_out(plan, d_out, d_st, n):
    sent = SENT_I if plan.out_is_int else SENT_F
    out = d_out.download(plan.out_dtype, (n + 1, plan.out_cols))
    st = d_st.download(np.int32, (n + 1,))
    assert (out[n] == sent).all() and st[n] == -1, "a row past the end was written"
    return out[:n], st[:n]


def enrich_dev(table, plan, ask, d_keys=None):
    """b2s_table_enrich_device: one launch, served by the gather loader"""
    n = len(ask)
    d_keys = d_keys or upload_keys(ask)
    d_out, d_st = sentinel_out(plan, n)
    before = nat.launch_count()
    assert table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr) is True
    assert nat.launch_count() - before == 1
    assert plan.last_kernel == "rowthread/bulk", plan.last_kernel
    return download_out(plan, d_out, d_st, n)


def lookup_then_run(table, plan, ask, d_keys=None):
    """b2s_table_lookup_device, then b2s_run_device on the rows it wrote; UNKNOWN folded in from the found flags"""
    n = len(ask)
    _, found, d_rows = lookup_dev(table, ask, d_keys=d_keys)
    d_out, d_st = sentinel_out(plan, n)
    plan.run_device(d_rows.ptr, n, 4 * table.n_feat, d_out.ptr, d_st.ptr)
    out, st = download_out(plan, d_out, d_st, n)
    return out, st | np.where(found, 0, UNKNOWN).astype(np.int32)


def check_enriched(out, st, flow, models, rows, found, vote=None):
    """outputs against the float64 reference of the plan over the reference rows; UNKNOWN exactly where no key matched"""
    check_plan_output(out, st, models, flow.expand(rows), vote=vote)
    np.testing.assert_array_equal((st & UNKNOWN) != 0, ~found)
    assert not (st & ~(UNKNOWN | NONFINITE | 2)).any()


def tile_rows(n, sms):
    """the row-thread kernel's tile height for n rows: halved from 128 while there are fewer tiles than SMs, down to 32"""
    tr = 128
    while tr > 32 and -(-n // tr) < sms:
        tr //= 2
    return tr


# ------------------------------------------------------------------------------------------ table_lookup_kernel
LOOKUP_F = {  # F -> copy path (lanes_per_row for the sub-warp path)
    4: "subwarp-1", 8: "subwarp-2", 16: "subwarp-4", 32: "subwarp-8", 64: "subwarp-16", 128: "subwarp-32",
    12: "warp-1", 20: "warp-1", 48: "warp-1", 132: "warp-2", 260: "warp-3",
    1: "scalar", 3: "scalar", 13: "scalar", 63: "scalar", 129: "scalar",
}


@pytest.mark.parametrize("policy", ["none", "all", "half"])
@pytest.mark.parametrize("F", list(LOOKUP_F))
def test_lookup_copy_paths(sms, F, policy):
    """every copy path of table_lookup_kernel (sub-warps of 1 ... 32 lanes per row, the warp-per-row loop once, twice and
    three times, the scalar path) under no policy, a policy on every column and one on half of them, bit for bit,
    through lookup_host and lookup_device; n = 1, 31, 32, 33, and (half policy) a ragged batch on which every warp runs
    at least two grid-stride iterations (8 CTAs of 256 threads per SM at most)"""
    rng = np.random.default_rng(F * 3 + len(policy))
    tab_keys = distinct_keys(3000, rng)
    vals = table_values(len(tab_keys), F, rng)
    pol = policy_of(policy, F, rng)
    table = DeviceTable(tab_keys, vals, pol)
    sizes = [1, 31, 32, 33] + ([2 * 8 * 256 * sms + 77] if policy == "half" else [])
    for n in sizes:
        ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, n - 1), every=29)
        if n == 1:
            ask = tab_keys[:1]  # the all-specials row
        want, found = ref_gather(tab_keys, vals, pol, ask)
        got, got_found, _ = lookup_dev(table, ask)
        np.testing.assert_array_equal(got_found, found)
        assert_rows(got, want, found, f"device n={n}")
        got, got_found = table.lookup(ask)
        np.testing.assert_array_equal(got_found, found)
        assert_rows(got, want, found, f"host n={n}")
    table.close()


def test_lookup_device_strides(sms):
    """F = 64 into rows 4F + 4 bytes apart (scalar path), 4F + 16 (16-byte path), and 4F + 16 from a base 4 bytes off
    16-byte alignment (a column offset of a wider matrix: scalar path); pad words, the words before the base, row n
    and found[n] keep their sentinels.  Misaligned or missing pointers are refused before anything is launched"""
    F = 64
    rng = np.random.default_rng(64)
    tab_keys = distinct_keys(4000, rng)
    vals = table_values(len(tab_keys), F, rng)
    pol = policy_of("half", F, rng)
    table = DeviceTable(tab_keys, vals, pol)
    for n in (33, 5000):
        ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, 32, n - 1), every=41)
        want, found = ref_gather(tab_keys, vals, pol, ask)
        for stride, offset in ((4 * F + 4, 0), (4 * F + 16, 0), (4 * F + 16, 4), (4 * F + 16, 8), (4 * F, 12)):
            got, got_found, _ = lookup_dev(table, ask, stride=stride, offset=offset)
            np.testing.assert_array_equal(got_found, found)
            assert_rows(got, want, found, f"n={n} stride={stride} offset={offset}")

    n = 64
    d_keys = nat.DeviceBuffer(8 * n + 16).upload(np.zeros(n + 2, dtype=np.int64))
    d_rows = nat.DeviceBuffer(4 * F * (n + 1) + 16)
    d_found = nat.DeviceBuffer(4 * n + 16)
    flow = Flow(F)
    models = scorers(F, 2, seed=1)
    plan = flow.plan(models)
    d_out, d_st = nat.DeviceBuffer(8 * n + 16), nat.DeviceBuffer(4 * n + 16)
    before = nat.launch_count()
    refused = [
        lambda: table.lookup_device(d_keys.ptr + 4, n, d_rows.ptr, 4 * F, d_found.ptr),
        lambda: table.lookup_device(None, n, d_rows.ptr, 4 * F, d_found.ptr),
        lambda: table.lookup_device(d_keys.ptr, n, None, 4 * F, d_found.ptr),
        lambda: table.lookup_device(d_keys.ptr, n, d_rows.ptr + 2, 4 * F, d_found.ptr),
        lambda: table.lookup_device(d_keys.ptr, n, d_rows.ptr, 4 * F, d_found.ptr + 2),
        lambda: table.lookup_device(d_keys.ptr, n, d_rows.ptr, 4 * F + 2, d_found.ptr),
        lambda: table.enrich_device(plan, d_keys.ptr + 4, n, d_out.ptr, d_st.ptr),
        lambda: table.enrich_device(plan, d_keys.ptr, n, d_out.ptr + 2, d_st.ptr),
        lambda: table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr + 1),
    ]
    for call in refused:
        with pytest.raises(nat.NativeError, match="aligned|null|bad"):
            call()
    assert nat.launch_count() == before, "a refused call launched a kernel"
    table.close()


# ------------------------------------------------------------------------------------------ probe chains
def identity_models(F):
    """F one-score models, model j = feature j: the fused scores are the gathered rows themselves"""
    out = []
    for j in range(F):
        W = np.zeros((1, F))
        W[0, j] = 1.0
        out.append(("linear", dict(W=W, b=np.zeros(1), link=nat.LINK_IDENTITY, classes=None)))
    return out


I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
EDGE_KEYS = np.array([0, -1, 1, I64_MIN, I64_MAX], dtype=np.int64)
LAYOUTS = ["wrap-cluster", "load-half-8", "load-half-4096", "one-key", "edge-keys-present", "edge-keys-absent"]


def layout(case, rng):
    """(table keys, absent keys): absent keys are homed where they have to walk the table's chains"""
    if case == "wrap-cluster":  # n keys homed at cap - 3: one chain over cap - 3, cap - 2, cap - 1, 0, ..., n - 4
        n = 1000
        cap = th.capacity(n)
        keys = th.keys_with_home_slots(np.full(n, cap - 3), cap, rng)
        inside = (cap - 3 + rng.integers(0, n, size=2000)) % cap
        absent = th.keys_with_home_slots(inside, cap, rng, exclude=keys)
        chain = th.probe_layout(keys, cap)
        assert chain[n - 4] == keys[-1] and (n - 3) not in chain
        return keys, absent
    if case.startswith("load-half"):
        n = int(case.split("-")[-1])
        cap = th.capacity(n)
        assert cap == 2 * n
        keys = th.keys_with_home_slots(rng.integers(0, cap, size=n), cap, rng)
        return keys, th.keys_with_home_slots(rng.integers(0, cap, size=2000), cap, rng, exclude=keys)
    if case == "one-key":
        keys = th.keys_with_home_slots([5], 16, rng)
        absent = th.keys_with_home_slots(np.concatenate([np.full(1000, 5), rng.integers(0, 16, size=1000)]), 16, rng,
                                         exclude=keys)
        return keys, absent
    cap = th.capacity(len(EDGE_KEYS) + 4 if case == "edge-keys-present" else 4)
    others = th.keys_with_home_slots([0, 0, cap - 1, 1], cap, rng, exclude=EDGE_KEYS)  # chains through slot 0
    absent = th.keys_with_home_slots(rng.integers(0, cap, size=2000), cap, rng, exclude=np.concatenate([EDGE_KEYS, others]))
    if case == "edge-keys-present":
        return np.concatenate([EDGE_KEYS, others]), absent
    return others, np.concatenate([EDGE_KEYS, absent])


@pytest.mark.parametrize("case", LAYOUTS)
def test_hash_layouts(sms, case):
    """tables laid out with keys of chosen home slots: a chain wrapping past the last slot, absent keys walking it, load
    factor exactly 0.5, a single key, the keys 0 (homed at slot 0, beside empty slots that hold key 0), +-1, INT64_MIN
    and INT64_MAX present and absent.  Every key and the absent ones through the lookup kernel and the fused loader
    (identity models: the scores are the rows)"""
    rng = np.random.default_rng(LAYOUTS.index(case))
    keys, absent = layout(case, rng)
    F = 8
    vals = rng.normal(size=(len(keys), F)).astype(np.float32)
    table = DeviceTable(keys, vals)
    assert capacity_of(table) == th.capacity(len(keys))
    ask = rng.permutation(np.concatenate([keys, absent]))
    want, found = ref_gather(keys, vals, None, ask)
    assert found.sum() == len(keys)
    got, got_found, _ = lookup_dev(table, ask)
    np.testing.assert_array_equal(got_found, found)
    assert_rows(got, want, found, case)
    plan = Flow(F).plan(identity_models(F))
    assert_kernel(plan, rowthread(4, 8))
    out, st = enrich_dev(table, plan, ask)
    assert_rows(out, want, found, f"{case} fused")
    np.testing.assert_array_equal(st, np.where(found, 0, UNKNOWN | NONFINITE))
    table.close()


# ------------------------------------------------------------------------------------------ the fused gather loader
N_SCORES = {1: (1, 1), 2: (2, 2), 4: (3, 4), 8: (5, 8)}  # per NS: score columns at the ragged and at the full width
RAGGED_F = {4: 12, 8: 20, 16: 36, 32: 100}  # partial rows inside an NCH tile
LARGE_NS = {4: 1, 8: 2, 16: 4, 32: 8}  # the instantiation that also runs >= 3 tiles per CTA


@pytest.mark.parametrize("ns", [1, 2, 4, 8])
@pytest.mark.parametrize("nch", [4, 8, 16, 32])
def test_fused_gather_instantiations(sms, nch, ns):
    """rowthread_kernel<NCH, NS, TPR, 1> gathering from a table: F = 4 NCH and a ragged F, a table policy on half the
    columns, a plan Imputer, NaN / Inf stored; 1 and 33 rows and a ragged batch in each tile-height band (32 / 64 / 128);
    unknown keys at rows 0, TR - 1, TR, n - 1 and every 97th row (every tile, so every pipeline stage); an all-unknown
    batch; for one NS per NCH a batch of >= 3 tiles per CTA (16 CTAs per SM at most), whose key look-ahead runs past the
    last tile.  Against the float64 reference and bit-equal to lookup_device + run_device"""
    sizes = bands(sms)
    for F in (4 * nch, RAGGED_F[nch]):
        rng = np.random.default_rng(nch * 10 + ns + F)
        tab_keys = distinct_keys(5000, rng)
        vals = table_values(len(tab_keys), F, rng, specials=NAN_INF, p=0.05)
        pol = policy_of("half", F, rng)
        table = DeviceTable(tab_keys, vals, pol)
        flow = Flow(F).imputer({f"f{F // 2 + 1}": 0.5, f"f{F - 2}": -1.5})
        models = scorers(flow.width, N_SCORES[ns][F == 4 * nch], seed=nch + ns + F)
        plan = flow.plan(models)
        assert_kernel(plan, rowthread(nch, ns))
        runs = [(n, "mixed") for n in sizes] + [(sizes[3], "all-unknown")]
        if F == 4 * nch and ns == LARGE_NS[nch]:
            runs.append((3 * 16 * 128 * sms + 77, "mixed"))
        for n, kind in runs:
            tr = tile_rows(n, sms)
            if kind == "all-unknown":
                ask = distinct_keys(n, rng, exclude=tab_keys)
            else:
                ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, tr - 1, tr, n - 1), every=97)
            rows, found = ref_gather(tab_keys, vals, pol, ask)
            d_keys = upload_keys(ask)
            out, st = enrich_dev(table, plan, ask, d_keys=d_keys)
            check_enriched(out, st, flow, models, rows, found)
            out2, st2 = lookup_then_run(table, plan, ask, d_keys=d_keys)
            np.testing.assert_array_equal(out.view(np.uint32), out2.view(np.uint32))
            np.testing.assert_array_equal(st, st2)
        table.close()


def test_fused_impute_fold(sms):
    """every combination on one column of table policy {set, NaN} x plan Imputer {present, absent} x DropFeatures
    {dropped, kept}, over stored NaN payloads, +-Inf and +-FLT_MAX: the policy applies first, then the plan"""
    F = 32
    rng = np.random.default_rng(32)
    tab_keys = distinct_keys(3000, rng)
    vals = table_values(len(tab_keys), F, rng, specials=SPECIALS[:7], p=0.1)
    combos = [(c % 2 == 0, (c // 2) % 2 == 0, (c // 4) % 2 == 0) for c in range(F)]  # (policy, imputer, dropped)
    pol = np.where([p for p, _, _ in combos], rng.normal(size=F), np.nan).astype(np.float32)
    fills = {f"f{c}": float(rng.normal()) for c, (_, imp, _) in enumerate(combos) if imp}
    dropped = [f"f{c}" for c, (_, _, d) in enumerate(combos) if d]
    flow = Flow(F).imputer(fills).drop(dropped)
    models = scorers(flow.width, 4, seed=5)
    for _, m in models:
        m["W"] = m["W"] * 1e-3  # FLT_MAX inputs: scores stay inside float32
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(8, 4))
    table = DeviceTable(tab_keys, vals, pol)
    n = bands(sms)[4]
    ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, 1, n - 1), every=53)
    ask[2:2 + 7] = tab_keys[:7]  # the all-special rows
    rows, found = ref_gather(tab_keys, vals, pol, ask)
    out, st = enrich_dev(table, plan, ask)
    check_enriched(out, st, flow, models, rows, found)
    assert (st & NONFINITE).any() and not (st & NONFINITE).all()
    out2, st2 = lookup_then_run(table, plan, ask)
    check_enriched(out2, st2, flow, models, rows, found)
    table.close()


def test_fused_onehot_without_policy(sms):
    """one-hot sources gathered from a table without a policy: category codes, codes outside the vocabulary, NaN (with
    an Imputer fill that is a category on one source and none on the other)"""
    F = 24
    rng = np.random.default_rng(24)
    tab_keys = distinct_keys(4000, rng)
    vals = table_values(len(tab_keys), F, rng, specials=NAN_INF, p=0.03)
    cats = {3: [0, 1, 2, 3], 10: [5, 7, 9]}
    for c, v in cats.items():
        vals[:, c] = rng.choice(np.array(v + [-1, 4, 6, 2.5, np.nan], dtype=np.float32), size=len(tab_keys))
    flow = Flow(F).imputer({"f3": 1.0}).one_hot({f"f{c}": v for c, v in cats.items()})
    models = scorers(flow.width, 2, seed=24)
    plan = flow.plan(models)
    assert_kernel(plan, rowthread(8, 2))
    table = DeviceTable(tab_keys, vals)
    for n in bands(sms)[1:]:
        ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, n - 1), every=61)
        rows, found = ref_gather(tab_keys, vals, None, ask)
        out, st = enrich_dev(table, plan, ask)
        check_enriched(out, st, flow, models, rows, found)
        out2, st2 = lookup_then_run(table, plan, ask)
        np.testing.assert_array_equal(out.view(np.uint32), out2.view(np.uint32))
        np.testing.assert_array_equal(st, st2)
    E = flow.expand(rows)
    onehot = [j for j, nm in enumerate(flow.program().out_names) if "_" in nm]
    assert E[:, onehot].sum(axis=0).min() > 0, "a category never occurs"
    table.close()


# ------------------------------------------------------------------------------------------ the three-launch fallback
DECLINED = ["dense-12x64", "map-values", "onehot-policy", "f13", "trees3"]


def declined_case(case, rng):
    """(F, flow, models, policy, the kernel the plan finalizes to, what serves the fallback's launch, plan launches)"""
    if case == "dense-12x64":
        flow = Flow(64)
        return 64, flow, scorers(64, 12, seed=12), policy_of("half", 64, rng), "dense_head_kernel", "dense", 1
    if case == "map-values":
        F = 20
        flow = Flow(F).map_values(all_mapped(names(F), {"f0": {0: 10, 1: -2}, "f4": {"ranges": {1: ["-inf", 0], 2: [0, "inf"]}}}))
        return F, flow, scorers(flow.width, 2, seed=20), policy_of("half", F, rng), "rows_kernel<LINEAR,NS=2>", "rows", 1
    if case == "onehot-policy":
        F = 16
        flow = Flow(F).one_hot({"f2": [0, 1, 2]})
        pol = policy_of("all", F, rng)
        pol[2] = 1.0  # NaN in the one-hot source becomes category 1
        return F, flow, scorers(flow.width, 3, seed=16), pol, rowthread(4, 4), "rowthread/bulk", 1
    if case == "trees3":  # scikit-learn trees (NaN flags its row), read by the tree prep kernel through a tensor map
        from tests.test_gpu_tree_paths import gbr, pk

        F = 32
        models = [pk(gbr(F, 5, 15, seed=3)), pk(gbr(F, 4, 10, seed=4))]
        return F, Flow(F), models, policy_of("half", F, rng), "t3_prep_kernel + trees3_kernel<", "trees3/tma", 3
    F = 13
    flow = Flow(F).imputer({"f1": 0.5})
    return F, flow, scorers(F, 3, seed=13), policy_of("half", F, rng), rowthread(4, 4), "rowthread/ldgsts", 1


@pytest.mark.parametrize("case", DECLINED)
def test_declined_plans_through_enrich_host(sms, case):
    """plans the gather loader declines (the dense head with 12 scores, MapValues on rows_kernel, a one-hot source under a
    table policy, 13 columns, trees3): b2s_table_enrich_device launches nothing, b2s_table_enrich_host gathers, runs the
    plan and marks unknown keys (2 + the plan's launches, reported in stats and counted by the library)"""
    rng = np.random.default_rng(DECLINED.index(case))
    F, flow, models, pol, kernel, served, plan_launches = declined_case(case, rng)
    tab_keys = distinct_keys(6000, rng)
    vals = table_values(len(tab_keys), F, rng, specials=NAN_INF, p=0.05)
    if case == "map-values":
        vals[:, 0] = rng.choice(np.array([0, 1, 2, np.nan], dtype=np.float32), size=len(tab_keys))
    if case == "onehot-policy":
        vals[:, 2] = rng.choice(np.array([0, 1, 2, 5, np.nan], dtype=np.float32), size=len(tab_keys))
    plan = flow.plan(models)
    assert_kernel(plan, kernel)
    table = DeviceTable(tab_keys, vals, pol)
    n = bands(sms)[4]
    ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, n - 1), every=37)
    rows, found = ref_gather(tab_keys, vals, pol, ask)
    d_keys = upload_keys(ask)
    d_out, d_st = sentinel_out(plan, n)
    before = nat.launch_count()
    assert table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr) is False
    assert nat.launch_count() == before
    before = nat.launch_count()
    out, st, stats = table.enrich(plan, ask, with_stats=True)
    assert nat.launch_count() - before == 2 + plan_launches
    assert stats["kernels"] == 2 + plan_launches and stats["rows"] == n
    assert plan.last_kernel == served, plan.last_kernel
    np.testing.assert_array_equal((st & UNKNOWN) != 0, ~found)
    if case != "dense-12x64":
        check_enriched(out, st, flow, models, rows, found)
        return
    from tests.test_gpu_dense_matrix import score_bound

    E = flow.expand(rows)
    W = np.concatenate([m["W"] for _, m in models])
    b = np.concatenate([m["b"] for _, m in models])
    ok = np.isfinite(E).all(axis=1)
    np.testing.assert_array_equal((st & NONFINITE) != 0, ~ok)
    want = E[ok] @ W.T + b
    err = np.abs(out[ok].astype(np.float64) - want)
    assert (err <= score_bound(E[ok], W, b, 16, 2, False)).all()
    table.close()


def test_enrich_host_staging(sms):
    """one table, plans of 1 and 8 output columns, batches that grow and shrink the staging in both directions, keys
    pinned and pageable"""
    F = 16
    rng = np.random.default_rng(16)
    tab_keys = distinct_keys(5000, rng)
    vals = table_values(len(tab_keys), F, rng, specials=NAN_INF, p=0.05)
    pol = policy_of("half", F, rng)
    table = DeviceTable(tab_keys, vals, pol)
    flow = Flow(F).imputer({"f3": 0.25})
    plans = {}
    for cols in (1, 8):
        models = scorers(F, cols, seed=cols)
        plans[cols] = (flow.plan(models), models)
        assert plans[cols][0].out_cols == cols
    for i, (cols, n) in enumerate([(1, 5000), (8, 100), (8, 6000), (1, 7000), (8, 4096), (1, 1), (8, 9000)]):
        plan, models = plans[cols]
        ask = ask_keys(tab_keys, n, rng, unknown_rows=(0, n - 1), every=31)
        if i % 2:
            pinned = nat.pinned_empty((n,), np.int64)
            pinned[:] = ask
            ask = pinned
        rows, found = ref_gather(tab_keys, vals, pol, np.asarray(ask))
        out, st, stats = table.enrich(plan, ask, with_stats=True)
        assert stats["kernels"] == 1 and stats["rows"] == n
        assert plan.last_kernel == "rowthread/bulk"
        check_enriched(out, st, flow, models, rows, found)
    table.close()


def test_bench_shape(sms):
    """the enrich_ens4 workload at a reduced size: 1 Mi keys x 64 features, 5 % NaN, a $mean policy, four linear models
    and a mean vote, 1 Mi keys asked, one fused launch"""
    F, n_keys = 64, 1 << 20
    rng = np.random.default_rng(4)
    vals = rng.normal(size=(n_keys, F)).astype(np.float32)
    vals[rng.random(vals.shape) < 0.05] = np.nan
    tab_keys = rng.permutation(n_keys).astype(np.int64) * 7919 + 13
    pol = np.nanmean(vals, axis=0).astype(np.float32)
    table = DeviceTable(tab_keys, vals, pol)
    coefs = np.random.default_rng(5).normal(size=(4, F))
    models = [("linear", dict(W=coefs[i:i + 1], b=np.array([0.25 * i]), link=nat.LINK_IDENTITY, classes=None)) for i in range(4)]
    vote = (nat.VOTE_MEAN, [0.25] * 4)
    flow = Flow(F)
    plan = flow.plan(models, vote=vote)
    assert_kernel(plan, rowthread(16, 4))
    ask = ask_keys(tab_keys, 1 << 20, rng, every=1009)
    rows, found = ref_gather(tab_keys, vals, pol, ask)
    out, st = enrich_dev(table, plan, ask)
    check_enriched(out, st, flow, models, rows, found, vote=vote)
    assert not (st & NONFINITE).any()
    table.close()
