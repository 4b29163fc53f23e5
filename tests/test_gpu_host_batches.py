"""Every host path of a plan (b2s_run_host and the coalescing ring) against b2s_run_device on the same rows.  Needs an
H100: `-m gpu`.

b2s_run_host takes a batch one of three ways: at most 64 KiB of rows is read by the kernels from pinned host memory (the
caller's, or the staging copy of pageable rows); a larger batch is copied in first; a pinned batch of at least 2 x 65 536
rows runs as a pipeline of 65 536-row chunks.  Results and status words are written straight to pinned memory, or copied
back per chunk.  Strided rows are packed into the staging area first.  A ring batch is the same batch from its pinned
slot.  Whichever path a batch takes, its votes and status words are those of b2s_run_device, bit for bit.

Plans whose votes go to merge targets or an attached communicator write nothing locally: the host entry points refuse
them (B2S_ERR_UNSUPPORTED, -6), before anything is enqueued, and b2s_run_device serves them.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from mlrun_b200 import _native as nat  # noqa: E402
from mlrun_b200 import packing  # noqa: E402
from mlrun_b200.feature_store.steps import OneHotEncoder  # noqa: E402
from mlrun_b200.lowering import ColumnProgram  # noqa: E402
from mlrun_b200.sharding import MergeComm  # noqa: E402
from mlrun_b200.synthetic import flow3_workload, tree_workload  # noqa: E402
from tests.device_check import ROW_NONFINITE, SENT_F, Rows, run_device  # noqa: E402

CHUNK = 65536            # rows per chunk of a pipelined host batch
PIPE = 2 * CHUNK + 3000  # the smallest pinned batch that is pipelined, plus a ragged last chunk
REFUSED = r"error -6: .*b2s_run_device"


@pytest.fixture(scope="module")
def workloads():
    nat.init(0)
    assert nat.device_info()["cc"] == (9, 0)
    # no Imputer in front: the NaN values flag their rows (B2S_ROW_NONFINITE_INPUT) on every path
    wl = flow3_workload(n_rows=PIPE, n_num=56, n_cat=8, seed=51, n_models=1, nan_frac=0.002)
    tw = tree_workload(n_rows=PIPE, n_feat=32, n_models=4, n_trees=20, depth=5, seed=52, n_fit=1500)
    tw.X[::997, 5] = np.nan
    return {"linear": wl, "trees": tw}


def build_plan(kind, wl):
    if kind == "linear":
        prog = ColumnProgram(wl.names)
        prog.apply(OneHotEncoder(mapping={k: list(v) for k, v in wl.onehot_mapping.items()}))
        plan = prog.build_plan([packing.pack_model(m) for m in wl.sklearn_models()])
        assert plan.kernel.startswith("rowthread_kernel<"), plan.kernel
        return plan, 1
    plan = ColumnProgram([f"f{i}" for i in range(32)]).build_plan([packing.pack_model(m) for m in wl.models],
                                                                  vote=(nat.VOTE_MEAN, [0.25] * 4))
    assert plan.kernel.startswith("t3_prep_kernel + trees3_kernel<"), plan.kernel
    return plan, 3


def host_rows(how, X):
    """the same rows as the host path `how` takes them"""
    if how == "pipelined":
        pinned = nat.pinned_empty(X.shape, np.float32)
        pinned[:] = X
        return pinned
    if how.startswith("strided"):
        wide = np.zeros((len(X), X.shape[1] + 16), dtype=np.float32)
        wide[:, :X.shape[1]] = X
        return wide[:, :X.shape[1]]
    return np.ascontiguousarray(X)


def check_batch(out, st, stats, want, want_st, n, kernels):
    np.testing.assert_array_equal(out.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(st, want_st)
    assert want_st.any(), "the batch has no flagged row"
    assert stats["rows"] == n and stats["kernels"] == kernels
    assert stats["nonfinite_rows"] == int(((want_st & ROW_NONFINITE) != 0).sum())


# (host path, rows): zero-copy input (16 KiB of rows), copied in (1 MiB), pipelined in three chunks, and strided rows
# packed into the staging area, read from there by the kernels or copied in from there
HOST_CASES = [("zero-copy", 64), ("copied", 4096), ("pipelined", PIPE), ("strided-zero-copy", 64), ("strided", 4096)]


@pytest.mark.parametrize("kind", ["linear", "trees"])
@pytest.mark.parametrize("how,n", HOST_CASES, ids=[h for h, _ in HOST_CASES])
def test_run_host_matches_run_device(workloads, kind, how, n):
    wl = workloads[kind]
    plan, k = build_plan(kind, wl)
    X = wl.X[:n]
    want, want_st = run_device(plan, Rows(X))
    out, st, stats = plan.run(host_rows(how, X), with_status=True, with_stats=True)
    if kind == "linear" and how == "zero-copy":
        assert plan.last_kernel == "rowthread/host", plan.last_kernel
    chunks = -(-n // CHUNK) if how == "pipelined" else 1
    check_batch(out, st, stats, want, want_st, n, k * chunks)


@pytest.mark.parametrize("kind", ["linear", "trees"])
@pytest.mark.parametrize("n", [64, 4096])
def test_submit_wait_matches_run_device(workloads, kind, n):
    """one ticket per batch: the batch is the ticket's rows, read from the ring's pinned slot (64) or copied in (4096)"""
    wl = workloads[kind]
    plan, k = build_plan(kind, wl)
    X = wl.X[:n]
    want, want_st = run_device(plan, Rows(X))
    for _ in range(2):  # the second batch reuses a slot of the first
        out, st, stats = plan.wait(plan.submit(np.ascontiguousarray(X)), with_status=True, with_stats=True)
        check_batch(out, st, stats, want, want_st, n, k)


@pytest.mark.parametrize("how", ["targets", "comm"])
def test_merging_plans_are_refused_on_host_entry_points(workloads, how):
    """with merge targets or an attached communicator the kernels store their votes there and not into the batch's
    results: b2s_run_host (small and pipelined) and a ring batch refuse the plan; b2s_run_device still fills the target"""
    wl = workloads["linear"]
    want, _ = run_device(build_plan("linear", wl)[0], Rows(wl.X[:64]))
    plan, _ = build_plan("linear", wl)
    comm = target = None
    if how == "targets":
        target = nat.DeviceBuffer(4 * (PIPE + 1)).upload(np.full(PIPE + 1, SENT_F, dtype=np.float32))
        plan.set_merge_targets([target.ptr], 1)
    else:
        comm = MergeComm(0, 1, PIPE, plan.out_cols, exchange=None)
        comm.attach(plan)
    try:
        for X in (np.ascontiguousarray(wl.X[:64]), host_rows("pipelined", wl.X)):
            with pytest.raises(nat.NativeError, match=REFUSED):
                plan.run(X)
        ticket = plan.submit(np.ascontiguousarray(wl.X[:64]))
        with pytest.raises(nat.NativeError, match=REFUSED):
            plan.wait(ticket)

        local, _ = run_device(plan, Rows(wl.X[:64]))
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
