"""Multi-GPU (one process per GPU): event sharding + the fused P2P ensemble-merge.  Needs >= 2 GPUs; the
single-GPU `-m gpu` run skips it (the same sharding logic is covered over gloo in test_boundary_cpu.py)."""

import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["REPO_ROOT"])
from mlrun_b200 import _native as nat, api
from mlrun_b200.sharding import shard_bounds
from mlrun_b200.synthetic import flow3_workload
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
nat.init(rank)
wl = flow3_workload(n_rows=10000, n_num=56, n_cat=8, seed=7, n_models=4)     # the same batch on every rank
server = wl.build_server(api, engine="sync")
plan = server.compile(wl.names).plan
full_ref = plan.run(wl.X)                                                      # single-GPU answer
lo, hi = shard_bounds(len(wl.X), rank, world)
merged = nat.DeviceBuffer(len(wl.X) * plan.out_cols * 4)
handles = [None] * world
dist.all_gather_object(handles, nat.ipc_export(merged.ptr))
peers = [merged.ptr if r == rank else nat.ipc_open(handles[r]) for r in range(world)]
plan.set_merge_targets(peers, lo)
shard = nat.DeviceBuffer((hi - lo) * 256).upload(wl.X[lo:hi])
plan.run_device(shard.ptr, hi - lo, 256, None)
nat.load().b2s_device_sync()
dist.barrier()
got = merged.download(np.float32, (len(wl.X), plan.out_cols))
assert np.array_equal(got, full_ref), (rank, np.abs(got - full_ref).max())
dist.barrier()
dist.destroy_process_group()
sys.stdout.write(f"[merge ok on rank {rank}]\n")
sys.stdout.flush()
'''


def test_fused_p2p_merge_two_gpus(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    out = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
         "--master-port", "29621", str(script)],
        capture_output=True, text=True, env=dict(os.environ, REPO_ROOT=ROOT), timeout=300)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "[merge ok on rank 0]" in out.stdout and "[merge ok on rank 1]" in out.stdout, out.stdout[-2000:]


_SHARDED = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["REPO_ROOT"])
from mlrun_b200 import _native as nat, api
from mlrun_b200.sharding import ShardedGraphServer, shard_bounds, torch_exchange
from mlrun_b200.synthetic import flow3_workload
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
nat.init(rank)

def check(server, names, batches, label):
    full = [server.run_batch(X, names=names) for X in batches]          # single-GPU answers (same on every rank)
    max_rows = max(shard_bounds(len(X), 0, world)[1] for X in batches)
    for fused in (0, 1, None):      # the three ways of waiting: launch's last CTA (own step / previous step), wait kernel
        check_one(server, names, batches, label, full, max_rows, fused)
    dist.barrier()
    sys.stdout.write(f"[{label} ok on rank {rank}]\n")  # one write per rank: the ranks share the pipe
    sys.stdout.flush()


def check_one(server, names, batches, label, full, max_rows, fused):
    sharded = ShardedGraphServer(server, rank, world, max_rows, torch_exchange(dist), names=names, fused_wait=fused)
    for step, X in enumerate(batches * 3):                              # several steps: both buffer parities, reused
        lo, hi = shard_bounds(len(X), rank, world)
        merged = sharded.run_batch(X[lo:hi])
        for r in range(world):
            rlo, rhi = shard_bounds(len(X), r, world)
            got = sharded.rows_of(merged, r, rhi - rlo)
            want = full[step % len(batches)][rlo:rhi]
            assert np.array_equal(got, want), (label, fused, step, rank, r, np.abs(got.astype(np.float64) - want).max())
    # pipelined steps (lag 1): three launches back to back, each followed by the wait for the launch BEFORE it, then the
    # drain; nothing synchronises in between, so step e's votes and flags cross NVLink while e + 1 is scored.  The four
    # response slots keep all three responses intact until they are read; four groups walk every slot three times.
    d_in = [nat.DeviceBuffer(sharded.max_rows * sharded.plan.n_in * 4) for _ in range(3)]
    seq = batches * 6
    for g0 in range(0, len(seq), 3):
        group = seq[g0:g0 + 3]
        for j, X in enumerate(group):
            lo, hi = shard_bounds(len(X), rank, world)
            d_in[j].upload(np.ascontiguousarray(X[lo:hi]))
        ptrs = []
        for j, X in enumerate(group):
            lo, hi = shard_bounds(len(X), rank, world)
            ptr, epoch = sharded.run_device(d_in[j].ptr, hi - lo, lag=1)
            assert ptr is not None  # (the lockstep steps above were steps of the same communicator)
            if j > 0:
                ptrs.append(ptr)
        ptrs.append(sharded.drain()[0])
        nat.check(nat.load().b2s_device_sync())
        sharded.comm.check()
        for j, X in enumerate(group):
            merged = np.empty((world * sharded.max_rows, sharded.plan.out_cols), dtype=sharded.plan.out_dtype)
            nat.check(nat.load().b2s_memcpy_d2h(merged.ctypes.data, ptrs[j], merged.nbytes))
            for r in range(world):
                rlo, rhi = shard_bounds(len(X), r, world)
                got = sharded.rows_of(merged, r, rhi - rlo)
                want = full[(g0 + j) % len(batches)][rlo:rhi]
                assert np.array_equal(got, want), (label, "lag1", fused, g0 + j, rank, r)
    sharded.close()

# (a) the metric workload: Imputer -> OneHotEncoder -> VotingEnsemble(4 linear) on the row-thread kernel
wl = flow3_workload(n_rows=10001, n_num=56, n_cat=8, seed=7, n_models=4)
server = wl.build_server(api, engine="sync")
rng = np.random.default_rng(5)
# the 1-row batch leaves rank 1 an empty shard: it stores nothing but still takes the step
check(server, wl.names, [wl.X, wl.X[rng.permutation(len(wl.X))[:7777]], wl.X[:1]], "flow3")

# (b) BASELINE configs[3]: a router of 8 mixed linear / tree scorers over 64 raw features (tree parts kernel + vote kernel)
from sklearn.ensemble import GradientBoostingRegressor
from sklearn.linear_model import Ridge
frng = np.random.default_rng(11)
Xf = frng.normal(size=(3000, 64)).astype(np.float32)
y = 2 * Xf[:, 0] + np.sin(Xf[:, 1]) + Xf[:, 2] * Xf[:, 3]
fn = api.new_function("router8", kind="serving")
graph = fn.set_topology("router", api.VotingEnsemble(vote_type="regression"))
for i in range(8):
    m = (GradientBoostingRegressor(n_estimators=25, max_depth=6, random_state=i, subsample=0.5) if i % 2 == 0 else Ridge(alpha=1.0 + i)).fit(Xf, y)
    graph.add_route(f"m{i}", class_name="SKLearnModelServer", model=m, model_path="")
server8 = fn.to_mock_server(namespace={"SKLearnModelServer": api.SKLearnModelServer})
X8 = frng.normal(size=(65536, 64)).astype(np.float32)
check(server8, [f"f{i}" for i in range(64)], [X8, X8[:30011], X8[:1]], "router8")

# (c) the dense head (wgmma): one 16-class LogisticRegression, argmax in the epilogue's float32 fast path
from sklearn.linear_model import LogisticRegression
from mlrun_b200 import packing
from mlrun_b200.lowering import ColumnProgram


class PlanServer:
    """a compiled plan behind the two calls ShardedGraphServer makes of a server; its single-GPU answer is b2s_run_device
    on device rows (the kernel the shards run, whatever the batch size)"""

    def __init__(self, plan):
        self.plan = plan

    def compile(self, names=None):
        return self

    def run_batch(self, X, names=None):
        X = np.ascontiguousarray(X, dtype=np.float32)
        d_in = nat.DeviceBuffer(X.nbytes).upload(X)
        d_out = nat.DeviceBuffer(len(X) * self.plan.out_cols * 4)
        self.plan.run_device(d_in.ptr, len(X), X.shape[1] * 4, d_out.ptr)
        assert self.plan.last_kernel == "dense", self.plan.last_kernel
        return d_out.download(self.plan.out_dtype, (len(X), self.plan.out_cols))


drng = np.random.default_rng(3)
centres = drng.normal(size=(16, 64)) * 1.5
yd = drng.integers(0, 16, size=6000)
logit = LogisticRegression(max_iter=300).fit((centres[yd] + drng.normal(size=(6000, 64))).astype(np.float32), yd * 3 + 5)
dplan = ColumnProgram([f"f{i}" for i in range(64)]).build_plan([packing.pack_model(logit)])
assert "dense_head_kernel" in dplan.kernel, dplan.kernel
Xd = (centres[drng.integers(0, 16, size=20001)] + drng.normal(size=(20001, 64))).astype(np.float32)
check(PlanServer(dplan), None, [Xd, Xd[:4321], Xd[:1]], "dense")
dist.destroy_process_group()
'''


def test_sharded_graph_server_with_completion_flags(tmp_path):
    """the product API of the sharded router: no barrier, no collective -- readers wait on the per-rank completion flags.
    The row-thread, trees3 and dense-head plans, merged rows bit-equal to the single-GPU answer, a 1-row batch among
    them (rank 1's shard empty)"""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "sharded.py"
    script.write_text(_SHARDED)
    out = subprocess.run(
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
         "--master-port", "29622", str(script)],
        capture_output=True, text=True, env=dict(os.environ, REPO_ROOT=ROOT), timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    for label in ("flow3", "router8", "dense"):
        for r in range(2):
            assert f"[{label} ok on rank {r}]" in out.stdout, out.stdout[-2000:]
