"""The fp8 all-to-all's schedule, ids, failure accounting and plan limits, on the CPU.

A model plays the mesh: every rank posts its shards in ``phase_order``, one record at a time, each on the queue pair to
its destination with the ids ``posted_ids`` gives; ranks take turns in a random order.  Every rank must receive every id
outside its own slot exactly once, R per source queue pair, and its slots must complete in ``arrival_slots`` order when
the ranks go phase by phase.  The per-pair accounting (``alltoall_fp8.reap``) must leave nothing after a clean run and
exactly the missing rank's receives after a run in which one rank never contributes."""
import random

import pytest

from rocnrdma_b200.parallel import alltoall_fp8 as A2A
from rocnrdma_b200.parallel import ring_fp8 as RF
from rocnrdma_b200.parallel.allgather_fp8 import arrival_slots


def _simulate(N, R, seed, skip=()):
    """Returns, per rank, the (source, id) pairs it received in arrival order, and ``posted_to[s][d]``."""
    rng = random.Random(seed)
    todo = [[(d, i) for d in A2A.phase_order(s, N)[1:] for i in A2A.posted_ids(s, N, R)[d]] if s not in skip else []
            for s in range(N)]
    got = [[] for _ in range(N)]
    posted_to = [[0] * N if s not in skip else [] for s in range(N)]
    while any(todo):
        s = rng.choice([q for q in range(N) if todo[q]])
        d, i = todo[s].pop(0)
        got[d].append((s, i))
        posted_to[s][d] += 1
    return got, posted_to


@pytest.mark.parametrize("N", range(2, 9))
@pytest.mark.parametrize("R", [1, 3])
def test_every_rank_receives_every_id_outside_its_slot_once(N, R):
    for seed in range(4):
        got, posted_to = _simulate(N, R, seed)
        for q in range(N):
            ids = [i for _, i in got[q]]
            assert sorted(ids) == sorted(set(range(N * R)) - set(range(q * R, (q + 1) * R))), q
            for s in range(N):
                if s != q:
                    from_s = [i for src, i in got[q] if src == s]
                    assert len(from_s) == R and from_s == A2A.received_ids(q, N, R)[s]
            assert sum(posted_to[q]) == (N - 1) * R and posted_to[q][q] == 0


@pytest.mark.parametrize("N", range(2, 9))
def test_each_phase_is_a_permutation(N):
    """At phase j every rank sends to exactly one peer and receives from exactly one; phase 0 is the own shard."""
    for j in range(N):
        dests = [A2A.phase_order(s, N)[j] for s in range(N)]
        assert sorted(dests) == list(range(N))
        assert all(dests[s] == (s + j) % N for s in range(N))
    assert all(A2A.phase_order(s, N)[0] == s for s in range(N))


@pytest.mark.parametrize("N", range(2, 9))
def test_slots_complete_in_arrival_order(N):
    """Phase by phase, rank q's slot from rank s fills at phase (q - s) mod N: the order q, q-1, ..., q+1, which the
    GEMM's a_order and the unpacks follow."""
    for q in range(N):
        filled = [s for j in range(N) for s in range(N) if A2A.phase_order(s, N)[j] == q]
        assert filled == arrival_slots(q, N)


@pytest.mark.parametrize("N", range(2, 9))
def test_ids_are_the_landing_layout(N):
    """The immediate of record r from rank s is s * R + r on every destination: slot s of its landing region."""
    R = 5
    for s in range(N):
        ids = A2A.posted_ids(s, N, R)
        assert sorted(ids) == [d for d in range(N) if d != s]
        assert all(v == list(range(s * R, (s + 1) * R)) for v in ids.values())
    for q in range(N):
        assert sorted(A2A.received_ids(q, N, R)) == [s for s in range(N) if s != q]


@pytest.mark.parametrize("N", range(2, 9))
def test_a_clean_run_leaves_nothing_behind(N):
    R = 3
    _, posted_to = _simulate(N, R, seed=N)
    for q in range(N):
        stale, backlog = A2A.reap(q, R, posted_to, (N - 1) * R)
        assert stale == 0 and backlog == [0] * N


@pytest.mark.parametrize("N", range(2, 9))
def test_a_skipped_rank_leaves_its_receives_on_its_pairs(N):
    """Rank k never runs: every other rank has R receive WQEs left on its queue pair from k and no stale completion;
    rank k itself received everything and has nothing left."""
    R, k = 3, N - 1
    _, posted_to = _simulate(N, R, seed=N, skip=(k,))
    for q in range(N):
        received = (N - 2) * R if q != k else (N - 1) * R
        stale, backlog = A2A.reap(q, R, posted_to, received)
        assert stale == 0
        assert backlog == [R if (s == k and q != k) else 0 for s in range(N)]


def test_late_records_become_stale_completions():
    """A consumer that stopped early (it timed out) leaves the records that landed after it on the shared CQ."""
    N, R = 4, 2
    posted_to = [[0, R, R, R], [R, 0, R, R], [R, R, 0, R], [R, R, R, 0]]
    stale, backlog = A2A.reap(0, R, posted_to, 4)
    assert stale == 3 * R - 4 and backlog == [0] * N


@pytest.mark.parametrize("N", range(2, 9))
def test_capacity_and_queue_pairs(N):
    """R <= 16384 / (2(N-1)); the mesh of N(N-1) send and N(N-1) receive queue pairs fits the context's default 256."""
    R = A2A.max_records(N)
    assert 2 * (N - 1) * R <= RF.MAX_QUEUE_DEPTH < 2 * (N - 1) * (R + 1)
    assert 2 * N * (N - 1) <= 256
    assert A2A.MAX_WORLD == 8 <= RF.MAX_IN_PROCESS


def test_plan_refuses_bad_worlds_and_shapes():
    with pytest.raises(ValueError, match="2..8"):
        A2A.AllToAllFp8(None, 8192, 8192, 0, 9)
    with pytest.raises(ValueError, match="at least 2"):
        A2A.AllToAllFp8(None, 8192, 8192, 0, 1)
    with pytest.raises(ValueError, match="multiple of chunk_elems"):
        A2A.AllToAllFp8(None, 8192 * 3, 8192 * 2, 0, 2)
    with pytest.raises(ValueError, match="receive CQ"):
        A2A.AllToAllFp8(None, 8192 * (A2A.max_records(4) + 1), 8192, 0, 4)
