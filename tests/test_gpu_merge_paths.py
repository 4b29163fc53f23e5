"""The fused ensemble-merge on every kernel family, on one GPU: merge targets (b2s_plan_set_merge_targets) and a world-1
communicator (b2s_comm_*, MergeComm).  Needs an H100: `-m gpu`.

Every scoring kernel has its own store of the merged rows: vote_and_store / store_word (rows_kernel, t3_vote_kernel), the
row-thread epilogue and the dense head's epilogue, each followed by merge_signal.  The oracle of a merged row is the same
plan's b2s_run_device output into local memory over the same rows, bit for bit (votes and status words); that output is
itself held to the float64 expectation of test_gpu_host_batches.make_plan.  So merged rows are checked against both the
reference and the single-GPU answer.

Communicator layout (world 1): kCommHeader = 512 bytes -- flags (64 words, this rank's at word 0), the CTA counter (word
64) and the timeout word (65) -- then four slots of world x max_rows x out_cols words; step e (1-based) lands in slot e & 3.
The header is read after a stream synchronisation and before any wait is enqueued wherever the test knows where it is, so
that a broken signal fails an assert instead of running into the wait's timeout.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import api  # noqa: E402
from mlrun_b200.feature_store.online import DeviceTable  # noqa: E402
from mlrun_b200.sharding import MergeComm, ShardedGraphServer  # noqa: E402
from mlrun_b200.synthetic import flow3_workload, tree_workload  # noqa: E402
from tests.device_check import SENT_F, SENT_I, Rows, assert_kernel, run_device  # noqa: E402
from tests.test_gpu_dense_matrix import U, build as dense_plan, regressors, score_bound  # noqa: E402
from tests.test_gpu_host_batches import KINDS, N_MAX, Expect, make_plan, numeric_rows  # noqa: E402

ERR_INVALID, ERR_UNSUPPORTED = r"error -1:", r"error -6:"
COMM_HEADER = 512        # kCommHeader: flags, CTA counter, timeout word
COUNTER, TIMEOUT = 64, 65  # words of the header
COMM_ROWS = 4097         # MergeComm rounds it up to 4100 (row blocks start 16-byte aligned)


def dense_mean():
    """a third dense epilogue next to KINDS' scores and argmax: 13 identity scorers, mean vote (out_cols 1)"""
    rng = np.random.default_rng(13)
    W, b, w = rng.normal(size=(13, 64)), rng.normal(size=13), rng.uniform(0.0, 1.0, 13)
    X = numeric_rows(N_MAX, 64, 65)
    X64 = X.astype(np.float64)
    ok = np.isfinite(X64).all(axis=1)
    with np.errstate(invalid="ignore"):
        sc = X64 @ W.T + b
        sb = score_bound(X64, W, b, 16, 2, False)
        want, tol = sc @ w, sb @ w + U * (np.abs(sc) + sb) @ w
    return dense_plan(64, regressors(W, b), vote=(nat.VOTE_MEAN, w)), X, Expect(want[:, None], tol[:, None], ok[:, None], ~ok)


# kind -> (parts of the plan kernel, device last_kernel, kernels per batch): every plan with a vote to merge
MERGING = {k: (v[0], v[1], v[3]) for k, v in KINDS.items() if k != "store"}
MERGING["dense-mean"] = ("dense_head_kernel", "dense", 1)


class Plan:
    """one plan of a kind, its batch on the device and b2s_run_device's local output over the whole batch, held to the
    float64 expectation"""

    def __init__(self, kind):
        self.kind = kind
        self.kernel, self.dev_kernel, self.k = MERGING[kind]
        self.plan, X, self.expect = dense_mean() if kind == "dense-mean" else make_plan(kind)
        self.X = np.ascontiguousarray(X, dtype=np.float32)
        assert_kernel(self.plan, *([self.kernel] if isinstance(self.kernel, str) else self.kernel))
        self.rows = Rows(self.X)
        self.out, self.st = run_device(self.plan, self.rows)
        assert self.plan.last_kernel == self.dev_kernel, (kind, self.plan.last_kernel)
        self.expect.check(self.out, self.st, slice(0, N_MAX), f"{kind} run_device")
        self.sent = SENT_I if self.plan.out_is_int else SENT_F
        self.oc = self.plan.out_cols
        self._local = {}

    def local(self, n):
        """b2s_run_device into local memory over rows [0, n) -> (votes, status, last_kernel); the same rows of the whole
        batch's run, bit for bit"""
        if n not in self._local:
            out, st = run_device(self.plan, self.rows, n)
            np.testing.assert_array_equal(out.view(np.uint32), self.out[:n].view(np.uint32), err_msg=f"{self.kind} n={n}")
            np.testing.assert_array_equal(st, self.st[:n])
            self._local[n] = (out, st, self.plan.last_kernel)
        return self._local[n]

    def sentinels(self, rows):
        return np.full((rows, self.oc), self.sent, dtype=self.plan.out_dtype)


_PLANS = {}


def plan_of(kind):
    if kind not in _PLANS:
        nat.init(0)
        assert nat.device_info()["cc"] == (9, 0)
        _PLANS[kind] = Plan(kind)
    return _PLANS[kind]


@pytest.fixture(scope="module", autouse=True)
def close_plans():
    yield
    for p in _PLANS.values():
        p.plan.close()
    _PLANS.clear()


@pytest.fixture(scope="module")
def sms():
    nat.init(0)
    return nat.device_info()["sm_count"]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def sync():
    nat.check(nat.load().b2s_device_sync())


def d2h(ptr, shape, dtype):
    out = np.empty(shape, dtype=dtype)
    nat.check(nat.load().b2s_memcpy_d2h(out.ctypes.data, ptr, out.nbytes))
    return out


def h2d(ptr, arr):
    arr = np.ascontiguousarray(arr)
    nat.check(nat.load().b2s_memcpy_h2d(ptr, arr.ctypes.data, arr.nbytes))


def tile_edge(p, sms):
    """rows at which each family's grid runs out of tiles: 128-row tiles over one CTA per SM (row-thread, rows, dense
    head); 64-row trees3 tiles over four per SM, which is also the vote kernel's 256 rows over 4 x SMs blocks"""
    return 256 * sms if p.dev_kernel.startswith("trees3") else 128 * sms


# ------------------------------------------------------------------------------------------ merge targets
TARGETS = {"1": 1, "2": 2, "8": 8, "aliased": 1}  # "aliased": two targets that are the same buffer


@pytest.mark.parametrize("kind", list(MERGING))
@pytest.mark.parametrize("targets", list(TARGETS))
def test_merge_targets_hold_the_local_rows(kind, targets, sms):
    """every target holds the local run's rows at [off, off + n), bit for bit, and sentinels outside them; the local
    output is not written, the status words and last_kernel are the local run's; offsets 0, 1, 3 (not 16-byte aligned)
    and one that ends the block a row before the end of the buffer; batches of 1, 31, 129 rows, both sides of the
    family's tile edge and the whole batch.  set_merge_targets([], 0) then restores local output"""
    p = plan_of(kind)
    plan = p.plan
    edge = tile_edge(p, sms)
    sizes = [1, 31, 129, edge - 1, edge + 1, N_MAX]
    local = {n: p.local(n) for n in sizes}  # before any target is set
    try:
        for n in sizes:
            want, want_st, want_kernel = local[n]
            R = n + 1024
            bufs = [nat.DeviceBuffer(R * p.oc * 4) for _ in range(TARGETS[targets])]
            ptrs = [b.ptr for b in bufs] * (2 if targets == "aliased" else 1)
            d_out = nat.DeviceBuffer((n + 1) * p.oc * 4)
            d_st = nat.DeviceBuffer((n + 1) * 4)
            for off in (0, 1, 3, R - n - 1):
                tag = f"{kind} targets={targets} n={n} off={off}"
                for b in bufs:
                    b.upload(p.sentinels(R))
                d_out.upload(p.sentinels(n + 1))
                d_st.upload(np.full(n + 1, -1, dtype=np.int32))
                plan.set_merge_targets(ptrs, off)
                plan.run_device(p.rows.ptr, n, p.rows.stride, d_out.ptr, d_st.ptr)
                assert plan.last_kernel == want_kernel, (tag, plan.last_kernel)
                mine = d_out.download(plan.out_dtype, (n + 1, p.oc))
                assert (bits(mine) == bits(p.sentinels(1))).all(), (tag, "the local output was written")
                st = d_st.download(np.int32, (n + 1,))
                np.testing.assert_array_equal(st[:n], want_st, err_msg=tag)
                assert st[n] == -1, tag
                for g, b in enumerate(bufs):
                    got = b.download(plan.out_dtype, (R, p.oc))
                    np.testing.assert_array_equal(bits(got[off:off + n]), bits(want), err_msg=f"{tag} target {g}")
                    assert (bits(got[:off]) == bits(p.sentinels(1))).all(), (tag, g, "rows before the block")
                    assert (bits(got[off + n:]) == bits(p.sentinels(1))).all(), (tag, g, "rows after the block")
    finally:
        plan.set_merge_targets([], 0)
    out, st = run_device(plan, p.rows, 129)
    np.testing.assert_array_equal(bits(out), bits(p.local(129)[0]))
    np.testing.assert_array_equal(st, p.local(129)[1])


def test_merge_target_refusals():
    """a transform-only plan has no vote to merge (-6); more than 8 targets or a negative offset are invalid (-1)"""
    nat.init(0)
    store = make_plan("store")[0]
    p = plan_of("rt4x1")
    buf = nat.DeviceBuffer(4 * 1024)
    try:
        with pytest.raises(nat.NativeError, match=ERR_UNSUPPORTED):
            store.set_merge_targets([buf.ptr], 0)
        with pytest.raises(nat.NativeError, match=ERR_INVALID):
            p.plan.set_merge_targets([buf.ptr] * 9, 0)
        with pytest.raises(nat.NativeError, match=ERR_INVALID):
            p.plan.set_merge_targets([buf.ptr], -1)
        store.set_merge_targets([], 0)  # no targets: nothing to refuse
        # the refusals left the plan's local output in place
        out, st = run_device(p.plan, p.rows, 31)
        np.testing.assert_array_equal(bits(out), bits(p.out[:31]))
    finally:
        p.plan.set_merge_targets([], 0)
        store.close()


# ------------------------------------------------------------------------------------------ a world-1 communicator
class CommView:
    """the host's view of a world-1 communicator's allocation, found from the pointer of a step's response"""

    def __init__(self, p, comm, ptr, epoch):
        self.slot_words = comm.world * comm.max_rows * p.oc
        self.base = ptr - COMM_HEADER - (epoch & 3) * self.slot_words * 4
        self.p = p

    def slot_ptr(self, e):
        return self.base + COMM_HEADER + (e & 3) * self.slot_words * 4

    def header(self):
        return d2h(self.base, (COMM_HEADER // 4,), np.uint32)

    def slots(self):
        return d2h(self.base + COMM_HEADER, (4, self.slot_words // self.p.oc, self.p.oc), self.p.plan.out_dtype)

    def fill_slots(self):
        h2d(self.base + COMM_HEADER, np.stack([self.p.sentinels(self.slot_words // self.p.oc)] * 4))


def check_header(view, e, tag):
    h = view.header()
    assert h[0] == e, (tag, "flag", int(h[0]))
    assert not h[1:64].any(), (tag, "flags of ranks that do not exist")
    assert h[COUNTER] == 0, (tag, "the last CTA did not reset the counter", int(h[COUNTER]))
    assert h[TIMEOUT] == 0, (tag, "timeout word", int(h[TIMEOUT]))


# (rows of the step, first batch row): every slot is written three times, empty steps among them
STEPS = [(1, 0), (129, 5), (4097, 1000), (0, 0), (31, 9000), (4100, 20000), (2048, 40001), (0, 0), (1, 77),
         (4097, 60000), (257, 100), (0, 0), (5, 131)]


@pytest.mark.parametrize("kind", list(MERGING))
@pytest.mark.parametrize("fused", [None, 0, 1])
def test_comm_steps_on_one_rank(kind, fused):
    """13 steps of 0 ... 4100 rows on MergeComm(0, 1, 4097, ...): after each step (and a synchronisation) its slot holds
    the local run's rows, the rows past n and the other three slots what they held, flag 0 the epoch, the counter and
    the timeout word 0; the local output is not written, the status words are the local run's.  wait(lag) gives the
    step's slot and epoch ((None, 0) before there is one), and each step launches the plan's kernels per batch (one
    signal kernel for an empty step) plus one wait kernel exactly when the fused wait does not cover it.  Then an
    oversized shard and a communicator of the wrong width are refused without a step"""
    p = plan_of(kind)
    plan = p.plan
    comm = MergeComm(0, 1, COMM_ROWS, p.oc, exchange=None)
    assert comm.max_rows == 4100
    comm.set_fused_wait(fused)
    comm.attach(plan)
    lag = 1 if fused == 1 else 0  # pipelined callers wait for the previous step
    d_out = nat.DeviceBuffer((comm.max_rows + 1) * p.oc * 4).upload(p.sentinels(comm.max_rows + 1))
    d_st = nat.DeviceBuffer((comm.max_rows + 1) * 4)
    view, model, fused_epoch = None, None, 0
    try:
        for i, (n, lo) in enumerate(STEPS):
            e = i + 1
            tag = f"{kind} fused={fused} step {e} ({n} rows)"
            d_st.upload(np.full(comm.max_rows + 1, -1, dtype=np.int32))
            before = nat.launch_count()
            plan.run_device(p.rows.ptr + lo * p.rows.stride, n, p.rows.stride, d_out.ptr, d_st.ptr)
            assert nat.launch_count() - before == (p.k if n else 1), (tag, "launches of the step")
            if fused is not None and e > fused:
                fused_epoch = e - fused
            sync()
            if view is not None:
                check_header(view, e, tag)
            w = e - lag
            before = nat.launch_count()
            ptr, epoch = comm.wait(lag=lag)
            covered = w == 0 or (fused_epoch and fused_epoch >= w)
            assert nat.launch_count() - before == (0 if covered else 1), (tag, "wait kernels")
            if w == 0:
                assert (ptr, epoch) == (None, 0), tag
            else:
                assert epoch == w, (tag, epoch)
                if view is not None:
                    assert ptr == view.slot_ptr(w), tag
            if view is None:  # the first step: find the allocation from its response, then sentinels in every slot
                if ptr is None:
                    ptr, epoch = comm.wait(lag=0)
                    assert epoch == e
                view = CommView(p, comm, ptr, e)
                sync()
                comm.check()
                check_header(view, e, tag)
                np.testing.assert_array_equal(bits(view.slots()[e & 3][:n]), bits(p.out[lo:lo + n]), err_msg=tag)
                view.fill_slots()
                model = np.stack([p.sentinels(comm.max_rows)] * 4)
            else:
                sync()
                comm.check()
                model[e & 3][:n] = p.out[lo:lo + n]
                got = view.slots()
                for s in range(4):
                    np.testing.assert_array_equal(bits(got[s]), bits(model[s]), err_msg=f"{tag} slot {s}")
            assert plan.last_kernel == p.dev_kernel or n == 0, (tag, plan.last_kernel)
            local = d_out.download(plan.out_dtype, (comm.max_rows + 1, p.oc))
            assert (bits(local) == bits(p.sentinels(1))).all(), (tag, "the local output was written")
            st = d_st.download(np.int32, (comm.max_rows + 1,))
            np.testing.assert_array_equal(st[:n], p.st[lo:lo + n], err_msg=tag)
            assert (st[n:] == -1).all(), tag
        e = len(STEPS)
        # refused without a step: a shard larger than the communicator's row block ...
        before = nat.launch_count()
        with pytest.raises(nat.NativeError, match=ERR_INVALID):
            plan.run_device(p.rows.ptr, comm.max_rows + 1, p.rows.stride, d_out.ptr, d_st.ptr)
        assert nat.launch_count() == before
        sync()
        check_header(view, e, f"{kind} after an oversized shard")
        # ... and a communicator whose rows have another width: the plan stays attached to the first one
        other = MergeComm(0, 1, 64, p.oc + 1, exchange=None)
        try:
            with pytest.raises(nat.NativeError, match=ERR_INVALID):
                other.attach(plan)
            assert other.wait(lag=0) == (None, 0)
        finally:
            other.close()
        check_header(view, e, f"{kind} after a refused attach")
        plan.run_device(p.rows.ptr, 3, p.rows.stride, d_out.ptr, d_st.ptr)
        sync()
        check_header(view, e + 1, f"{kind} the step after the refusals")
        np.testing.assert_array_equal(bits(view.slots()[(e + 1) & 3][:3]), bits(p.out[:3]))
        assert comm.wait(lag=0)[1] == e + 1
        sync()
        comm.check()
    finally:
        comm.detach(plan)
        comm.close()
    out, st = run_device(plan, p.rows, 31)  # detached: local output again
    np.testing.assert_array_equal(bits(out), bits(p.out[:31]))


def test_comm_refuses_a_transform_only_plan():
    """attaching a plan that has no vote to merge is refused (-6) and takes no step"""
    nat.init(0)
    store = make_plan("store")[0]
    comm = MergeComm(0, 1, 64, store.out_cols, exchange=None)
    try:
        with pytest.raises(nat.NativeError, match=ERR_UNSUPPORTED):
            comm.attach(store)
        assert comm.wait(lag=0) == (None, 0)
    finally:
        comm.close()
        store.close()


# ------------------------------------------------------------------------------------------ ShardedGraphServer, world 1
def sharded_workload(which):
    if which == "flow3":
        wl = flow3_workload(n_rows=5000, n_num=56, n_cat=8, seed=7, n_models=4)
        return wl.build_server(api, engine="sync"), wl.names, wl.X, "rowthread_kernel"
    tw = tree_workload(n_rows=5000, n_feat=32, n_models=4, n_trees=20, depth=5, seed=52, n_fit=1500)
    return tw.build_server(api), None, tw.X, "trees3_kernel"


@pytest.mark.parametrize("which", ["flow3", "trees3"])
@pytest.mark.parametrize("fused", [0, 1, None])
def test_sharded_graph_server_on_one_rank(which, fused):
    """ShardedGraphServer(server, 0, 1, ...): run_batch gives the server's own run_batch rows bit for bit, and an empty
    batch is a step of its own (the epoch advances, the response is that step's slot)"""
    nat.init(0)
    server, names, X, kernel = sharded_workload(which)
    batches = [X[:4097], X[100:101], X[:0], X[2000:2129], X[:0], X[:0], X[3000:4000]]
    want = [server.run_batch(b, names=names) if len(b) else None for b in batches]
    sharded = ShardedGraphServer(server, 0, 1, 4097, None, names=names, fused_wait=fused)
    assert kernel in sharded.plan.kernel, sharded.plan.kernel
    try:
        slot_of = {}
        for i, Xb in enumerate(batches):
            e = i + 1
            merged = sharded.run_batch(Xb)
            ptr, epoch = sharded.comm.wait(lag=0)
            assert epoch == e, (which, fused, i, epoch)
            slot_of.setdefault(e & 3, ptr)
            assert ptr == slot_of[e & 3] and len(set(slot_of.values())) == len(slot_of), (which, i, "slot")
            if want[i] is not None:
                got = sharded.rows_of(merged, 0, len(Xb))
                np.testing.assert_array_equal(bits(got), bits(want[i]), err_msg=f"{which} fused={fused} batch {i}")
        sync()
        sharded.comm.check()
    finally:
        sharded.close()
    np.testing.assert_array_equal(bits(server.run_batch(batches[0], names=names)), bits(want[0]))


# ------------------------------------------------------------------------------------------ enrichment of merging plans
@pytest.mark.parametrize("kind", ["linear", "trees"])  # the fused gather (row-thread) and the gather-first path (trees3)
@pytest.mark.parametrize("how", ["targets", "comm"])
def test_enrichment_refuses_merging_plans(kind, how):
    """with merge targets or an attached communicator the kernels would store the votes there and not into the
    enrichment's output: enrich and enrich_device refuse the plan (-6 / False) with no launch, the targets untouched and
    no step; without them the same calls give the plan's output over the looked-up rows"""
    p = plan_of(kind)
    plan = p.plan
    rng = np.random.default_rng(3)
    keys = np.arange(20000, dtype=np.int64) * 7 + 3
    table = DeviceTable(keys, p.X[:20000])
    pick = rng.integers(0, 20000, size=3000)
    ask = keys[pick]
    n = len(ask)
    d_keys = nat.DeviceBuffer(8 * n).upload(ask)
    d_out = nat.DeviceBuffer(n * p.oc * 4).upload(p.sentinels(n))
    d_st = nat.DeviceBuffer(4 * n).upload(np.full(n, -1, dtype=np.int32))
    target = comm = None
    if how == "targets":
        target = nat.DeviceBuffer((n + 8) * p.oc * 4).upload(p.sentinels(n + 8))
        plan.set_merge_targets([target.ptr], 2)
    else:
        comm = MergeComm(0, 1, n, p.oc, exchange=None)
        comm.attach(plan)
    try:
        before = nat.launch_count()
        with pytest.raises(nat.NativeError, match=ERR_UNSUPPORTED):
            table.enrich(plan, ask)
        assert table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr) is False
        sync()
        assert nat.launch_count() == before, "a refused enrichment launched"
        if target is not None:
            assert (bits(target.download(plan.out_dtype, (n + 8, p.oc))) == bits(p.sentinels(1))).all()
        else:
            assert comm.wait(lag=0) == (None, 0), "a refused enrichment took a step of the communicator"
        assert (bits(d_out.download(plan.out_dtype, (n, p.oc))) == bits(p.sentinels(1))).all()
        assert (d_st.download(np.int32, (n,)) == -1).all()
    finally:
        if comm is not None:
            comm.detach(plan)
            comm.close()
        else:
            plan.set_merge_targets([], 0)
    out, st = table.enrich(plan, ask)
    np.testing.assert_array_equal(bits(out), bits(p.out[pick]))
    np.testing.assert_array_equal(st, p.st[pick])
    fused = table.enrich_device(plan, d_keys.ptr, n, d_out.ptr, d_st.ptr)
    assert fused == (kind == "linear")
    if fused:
        np.testing.assert_array_equal(bits(d_out.download(plan.out_dtype, (n, p.oc))), bits(p.out[pick]))
        np.testing.assert_array_equal(d_st.download(np.int32, (n,)), p.st[pick])
    table.close()
