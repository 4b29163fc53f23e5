"""The ensemble-merge protocol of b2s_comm_* (csrc/b2s_runtime.cu: comm struct, launch wiring; csrc/b2s_device.cuh: merge_signal)
as a randomly scheduled model: N ranks, every rank's stream is a sequence of

    K(e): store this rank's block of step e into slot e % SLOTS of EVERY rank's response buffer (one store per target, in any
          interleaving with the other ranks), then publish flag[target][me] = e on every target, then -- fused wait -- poll
          flag[me][*] >= e - LAG
    R(w): read the merged response of step w = e - LAG on this rank (enqueued on the stream behind K(e), like a caller's D2H copy)

The checks are the two claims DESIGN.md section 7 makes for four slots and lag <= 1: every read sees every rank's block of
exactly its step (no rank is ever more than SLOTS - 1 steps ahead of a reader), and the schedule never deadlocks.  With two
slots the same schedule does let a fast rank overwrite a block a slow reader has not read: the model must catch that.

A rank whose shard of a step is empty (a batch of fewer rows than ranks, mlrun_b200.sharding.shard_bounds) stores nothing
but still publishes the step's flag: its block of that step is not part of the response, and nobody waits for rows."""
import random

import pytest

from mlrun_b200.sharding import shard_bounds


def simulate(world, steps, slots, lag, seed, empty=frozenset(), skip=False):
    """empty: the (rank, step) pairs whose shard has no rows.  Such a rank stores nothing in that step and publishes its
    flag; skip=True instead lets it take no step at all (no flag, and every later launch of it one epoch lower)"""
    rnd = random.Random(seed)
    flags = [[0] * world for _ in range(world)]           # flags[target][source]
    merged = [[[0] * world for _ in range(slots)] for _ in range(world)]  # merged[target][slot][source] = step stored
    # per rank program: list of micro-ops
    prog = []
    for me in range(world):
        ops = []
        e = 0  # this rank's epoch
        for step in range(1, steps + 1):
            if skip and (me, step) in empty:
                continue
            e += 1
            targets = [(me + 1 + g) % world for g in range(world)]  # right-hand neighbour first, as the launch wiring does
            if (me, step) not in empty:
                ops += [("store", t, e) for t in targets]
            ops += [("flag", t, e) for t in targets]
            if e > lag:
                ops.append(("wait", e - lag))
                ops.append(("read", e - lag))
        for w in range(max(e - lag + 1, 1), e + 1):  # drain: the last `lag` steps
            ops.append(("wait", w))
            ops.append(("read", w))
        prog.append(ops)
    pc = [0] * world
    torn = []
    idle_rounds = 0
    while any(pc[r] < len(prog[r]) for r in range(world)):
        r = rnd.randrange(world)
        if rnd.random() < 0.3:  # bursts: one rank runs ahead for a while
            burst = rnd.randrange(1, 6 * world)
        else:
            burst = 1
        progressed = False
        for _ in range(burst):
            if pc[r] >= len(prog[r]):
                break
            op = prog[r][pc[r]]
            if op[0] == "store":
                merged[op[1]][op[2] % slots][r] = op[2]
            elif op[0] == "flag":
                flags[op[1]][r] = op[2]
            elif op[0] == "wait":
                if min(flags[r]) < op[1]:
                    break  # still polling
            else:  # read
                got = merged[r][op[1] % slots]
                if any(v != op[1] for src, v in enumerate(got) if (src, op[1]) not in empty):
                    torn.append((r, op[1], list(got)))
            pc[r] += 1
            progressed = True
        idle_rounds = 0 if progressed else idle_rounds + 1
        if idle_rounds > 100000:
            return "deadlock", torn
    return "done", torn


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("lag", [0, 1])
def test_four_slots_never_tear_and_never_deadlock(world, lag):
    for seed in range(40):
        state, torn = simulate(world, steps=24, slots=4, lag=lag, seed=seed)
        assert state == "done" and not torn, (seed, state, torn[:2])


@pytest.mark.parametrize("slots", [2, 3])
def test_the_model_catches_too_few_slots(slots):
    """pipelined steps (lag 1) need four slots: a reader of step w has published w + 1 before it reads, so a fast rank may
    already store step w + 3 -- with two or three slots that lands on the block being read.  Lockstep (lag 0) needs two."""
    caught = 0
    for seed in range(20):
        state, torn = simulate(8, steps=24, slots=slots, lag=1, seed=seed)
        assert state == "done"
        caught += bool(torn)
        assert not simulate(8, steps=24, slots=slots, lag=0, seed=seed)[1]
    assert caught == 20


def empty_shards(world, steps, seed):
    """(rank, step) pairs left empty by shard_bounds when about a third of the batches have fewer rows than ranks"""
    rnd = random.Random(seed)
    empty = set()
    for step in range(1, steps + 1):
        n = rnd.randrange(world) if rnd.random() < 0.35 else rnd.randrange(world, 4 * world)
        empty |= {(r, step) for r in range(world) if shard_bounds(n, r, world)[0] == shard_bounds(n, r, world)[1]}
    return empty


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("lag", [0, 1])
def test_empty_shards_publish_their_flags_and_never_tear_or_deadlock(world, lag):
    """batches of fewer rows than ranks (0 rows included) among ordinary ones: every rank still takes every step"""
    for seed in range(40):
        empty = empty_shards(world, 24, seed)
        assert any(r == world - 1 for r, _ in empty)
        state, torn = simulate(world, steps=24, slots=4, lag=lag, seed=seed, empty=empty)
        assert state == "done" and not torn, (seed, state, torn[:2])


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("lag", [0, 1])
def test_a_rank_that_skips_its_empty_step_deadlocks_the_schedule(world, lag):
    """a rank that launches nothing for an empty shard publishes no flag for it, and its later epochs lag one behind the
    other ranks': they wait for its last step for ever (on the device, until B2S_COMM_TIMEOUT_MS)"""
    for seed in range(3):
        state, _ = simulate(world, steps=24, slots=4, lag=lag, seed=seed, empty={(world - 1, 5)}, skip=True)
        assert state == "deadlock", seed
