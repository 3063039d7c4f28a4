"""The fp8 ring all-gather's schedule, its plan's limits, K7's ordered tile walk and the gather's reference, on the CPU.

The schedule model runs N ranks that each relay ``relay_slots(q)`` in order, a slot only once they hold it, and checks
that every rank ends with every shard exactly once, in the order the GEMM walks it."""
import random

import pytest
import torch

from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import allgather_fp8 as AG
from rocnrdma_b200.parallel import ring_fp8 as RF


# ------------------------------------------------------------------ the ring schedule
def _simulate(N, R, seed):
    """Every rank relays its slots in order, each record once it holds it; ranks take turns in a random order.  Returns
    the ids each rank received, in arrival order, and the ids each rank posted."""
    rng = random.Random(seed)
    held = [set(range(q * R, (q + 1) * R)) for q in range(N)]
    todo = [[s * R + r for s in AG.relay_slots(q, N) for r in range(R)] for q in range(N)]
    got = [[] for _ in range(N)]
    posted = [[] for _ in range(N)]
    while any(todo):
        ready = [q for q in range(N) if todo[q] and todo[q][0] in held[q]]
        assert ready, f"the ring deadlocks: {[t[:1] for t in todo]}"
        q = rng.choice(ready)
        i = todo[q].pop(0)
        posted[q].append(i)
        nxt = (q + 1) % N
        assert i not in held[nxt], f"rank {nxt} receives id {i} twice"
        held[nxt].add(i)
        got[nxt].append(i)
    return got, posted, held


@pytest.mark.parametrize("N", range(2, 9))
@pytest.mark.parametrize("R", [1, 3])
def test_every_rank_receives_every_other_shard_once(N, R):
    for seed in range(5):
        got, posted, held = _simulate(N, R, seed)
        for q in range(N):
            own = set(range(q * R, (q + 1) * R))
            assert sorted(got[q]) == sorted(set(range(N * R)) - own), q
            assert held[q] == set(range(N * R))
            assert len(got[q]) == (N - 1) * R


@pytest.mark.parametrize("N", range(2, 9))
def test_relay_order_is_the_arrival_order(N):
    R = 2
    got, posted, _ = _simulate(N, R, seed=N)
    for q in range(N):
        slots = AG.relay_slots(q, N)
        assert slots[0] == q and (q + 1) % N not in slots
        assert slots == [(q - k) % N for k in range(N - 1)]
        arrival = AG.arrival_slots(q, N)
        assert sorted(arrival) == list(range(N)) and arrival[:N - 1] == slots and arrival[-1] == (q + 1) % N
        # what a rank receives comes in its arrival order after its own slot, and it posts in that order too
        assert got[q] == [s * R + r for s in arrival[1:] for r in range(R)]
        assert posted[q] == [s * R + r for s in slots for r in range(R)]
        # and the relay of rank q is what rank q + 1 receives, in the same order
        assert got[(q + 1) % N] == posted[q]


# ------------------------------------------------------------------ the plan's limits
class _NoGpu:
    device = 0


@pytest.mark.parametrize("N", range(2, 9))
def test_queue_capacity_matches_the_refusal(N):
    m = AG.max_records(N)
    assert RF._pow2(2 * (N - 1) * m) <= RF.MAX_QUEUE_DEPTH < RF._pow2(2 * (N - 1) * (m + 1))
    chunk = P.TILE_ELEMS
    with pytest.raises(ValueError, match="receive queue"):
        AG.RingAllgatherFp8(_NoGpu(), (m + 1) * chunk, chunk, 0, N)


def test_plan_refuses_bad_geometry():
    for args, what in [((8192, 8192, 0, 1), "at least 2"), ((3 * 8192, 2 * 8192, 0, 2), "multiple of chunk"),
                       ((8192, 100, 0, 2), "multiple of 8192"), ((8192, 8192, 2, 2), "outside")]:
        with pytest.raises(ValueError, match=what):
            AG.RingAllgatherFp8(_NoGpu(), *args)


@pytest.mark.parametrize("N", range(2, 9))
def test_budget_arithmetic(monkeypatch, N):
    monkeypatch.setattr(RF, "_sms", lambda ctx: 132)
    for engine in (8, 16, 32):
        g = RF._default_grid(None, engine, N, AG.RingAllgatherFp8.WAITERS)
        RF._check_budget(None, engine, N, g, AG.RingAllgatherFp8.WAITERS)      # the default always fits
        for grid in range(1, 130):
            fits = engine + N * (grid + 2) <= 132
            if fits:
                RF._check_budget(None, engine, N, grid, 2)
            else:
                with pytest.raises(ValueError, match="SM budget"):
                    RF._check_budget(None, engine, N, grid, 2)


# ------------------------------------------------------------------ K7's ordered walk
def _row_walk(n_tiles, n_blks):
    return [(t // n_blks, t % n_blks) for t in range(n_tiles)]


def _ordered_walk(order, bpr, n_blks, n_rec):
    """tile_coords<1, true> of gemm_mxfp8.cu, walk index t -> (m_blk, n_blk)."""
    per_rec = bpr * n_blks
    out = []
    for t in range(len(order) * per_rec):
        rec = min(order[t // per_rec] & 0xFFFFFFFF, n_rec)
        out.append((rec * bpr + (t % per_rec) // n_blks, t % n_blks))
    return out


@pytest.mark.parametrize("rows_per_rec", [128, 256, 512])
@pytest.mark.parametrize("N", [128, 200, 1000, 4096])
def test_identity_order_is_the_row_walk(rows_per_rec, N):
    n_rec, bpr, n_blks = 6, rows_per_rec // 128, -(-N // 128)
    assert _ordered_walk(list(range(n_rec)), bpr, n_blks, n_rec) == _row_walk(n_rec * bpr * n_blks, n_blks)


@pytest.mark.parametrize("rows_per_rec", [128, 256, 512])
@pytest.mark.parametrize("N", [128, 200, 1000, 4096])
def test_any_order_covers_every_tile_once(rows_per_rec, N):
    rng = random.Random(rows_per_rec * 7 + N)
    bpr, n_blks = rows_per_rec // 128, -(-N // 128)
    for n_rec in (1, 2, 5, 16):
        order = list(range(n_rec))
        rng.shuffle(order)
        walk = _ordered_walk(order, bpr, n_blks, n_rec)
        assert sorted(walk) == sorted(_row_walk(n_rec * bpr * n_blks, n_blks))
        # record by record, in the given order, with every tile of a record before the next record
        per_rec = bpr * n_blks
        for i, rec in enumerate(order):
            assert {m // bpr for m, _ in walk[i * per_rec:(i + 1) * per_rec]} == {rec}
        # and the persistent CTAs' strided share of the walk covers it too
        grid = 7
        shares = [walk[u::grid] for u in range(grid)]
        assert sorted(t for s in shares for t in s) == sorted(walk)


def test_an_entry_outside_the_records_only_reaches_rows_past_m():
    n_rec, bpr, n_blks = 4, 2, 3
    for bad in (4, 1000, -1):
        walk = _ordered_walk([0, bad, 2, 3], bpr, n_blks, n_rec)
        assert all(m >= n_rec * bpr for m, _ in walk[bpr * n_blks:2 * bpr * n_blks])


# ------------------------------------------------------------------ the reference
@pytest.mark.parametrize("N", [2, 3, 5])
@pytest.mark.parametrize("chunk", [8192, 16384])
def test_ref_allgather_is_each_shard_packed_and_unpacked(N, chunk):
    g = torch.Generator().manual_seed(N * chunk)
    shards = [(torch.randn(2 * chunk, generator=g) * 3 ** s).to(torch.bfloat16) for s in range(N)]
    out, recs = P.ref_allgather_fp8(shards, chunk)
    n, rb = 2 * chunk, P.staging_bytes(2 * chunk, chunk)
    assert out.dtype == torch.bfloat16 and out.numel() == N * n and recs.numel() == N * rb
    for s, x in enumerate(shards):
        want = P.ref_pack_fp8(x, chunk)
        assert torch.equal(recs[s * rb:(s + 1) * rb], want)
        assert torch.equal(out[s * n:(s + 1) * n].view(torch.int16), P.ref_unpack_fp8(want, n, chunk).view(torch.int16))


# ------------------------------------------------------------------ the ordered K7 inside the gather (test_gpu_allgather_fp8_shapes.py)
@pytest.mark.parametrize("N", [2, 3, 5, 8])
def test_gather_schedule_walk_is_the_ordered_walk(N):
    """Every rank's model walk is ``_ordered_walk`` of its arrival order, and its CTAs' strided shares cover it once."""
    from test_gpu_allgather_fp8_shapes import OrderedGatherSchedule
    for K, rows_per_rec, R, Nb, grid in [(64, 128, 2, 200, 7), (4096, 512, 1, 4096, 0), (32, 256, 3, 1, 1),
                                         (160, 256, 2, 391, 300)]:
        for q in range(N):
            s = OrderedGatherSchedule(N, q, K, rows_per_rec, R, Nb, grid)
            order = [sl * R + r for sl in AG.arrival_slots(q, N) for r in range(R)]
            assert s.order == order
            assert s.coords() == _ordered_walk(order, rows_per_rec // 128, -(-Nb // 128), N * R)
            assert sorted(t for ts in s.tiles for t in ts) == list(range(s.n_tiles))
            assert s.place(s.walk[0][0]) == 0 and s.place(s.walk[-1][0]) == N - 1


def test_gather_schedule_hand_counted_walks():
    from test_gpu_allgather_fp8_shapes import OrderedGatherSchedule
    # N 2, rank 1, two 128-row blocks a record, two column blocks, grid 3: records 1 then 0, four tiles each
    s = OrderedGatherSchedule(2, 1, 64, 256, 1, 200, 3)
    assert s.walk == [(1, 2, 0), (1, 2, 1), (1, 3, 0), (1, 3, 1), (0, 0, 0), (0, 0, 1), (0, 1, 0), (0, 1, 1)]
    assert s.tiles == [[0, 3, 6], [1, 4, 7], [2, 5]]
    f = s.facts()
    assert f == {"multi_block_records": True, "cta_crosses_slots": True, "cta_starts_remote": False,
                 "record_shared": True, "ragged_n": True, "odd_n": False, "partial_k": True, "mid_ring_entry": True,
                 "clamped_grid": False}
    # N 3, rank 0, one tile a record, grid 7 clamped to 3: each CTA one record, in the arrival order 0, 2, 1
    s = OrderedGatherSchedule(3, 0, 4096, 128, 1, 1, 7)
    assert s.grid == 3 and s.tiles == [[0], [1], [2]] and s.walk == [(0, 0, 0), (2, 2, 0), (1, 1, 0)]
    assert [s.place(r) for r, _, _ in s.walk] == [0, 1, 2]
    f = s.facts()
    assert f["clamped_grid"] and f["cta_starts_remote"] and not f["cta_crosses_slots"] and not f["record_shared"]
    assert not f["mid_ring_entry"] and not f["partial_k"] and f["odd_n"] and f["ragged_n"]
    # N 4, rank 2, R 2, grid 1: one CTA walks slots 2, 1, 0, 3, every record of a slot before the next slot
    s = OrderedGatherSchedule(4, 2, 512, 128, 2, 128, 1)
    assert [r for r, _, _ in s.walk] == [4, 5, 2, 3, 0, 1, 6, 7] and s.tiles == [list(range(8))]
    f = s.facts()
    assert f["cta_crosses_slots"] and not f["cta_starts_remote"] and not f["record_shared"]
    assert not f["mid_ring_entry"] and not f["ragged_n"] and not f["partial_k"]       # k_blks 4: every tile from stage 0
    assert OrderedGatherSchedule(4, 2, 384, 128, 2, 128, 1).facts()["mid_ring_entry"]   # k_blks 3: the second from stage 3


def test_gather_geometry_cases_cover_every_fact_and_parameter():
    """The GPU geometry cases: each claims facts of both walks, the same on every rank; together they cover every fact,
    N = 2..8, Nb from 1 to 4096, grids 1, 3, 7, the default and one above the tile count, and signal_every 1, 3, 8."""
    from test_gpu_allgather_fp8_shapes import GEMM_FACTS, GEOMETRY_CASES, UNPACK_FACTS, case_facts, gather_grid
    seen_k, seen_u = set(), set()
    for (N, K, rows_per_rec, R, Nb, grid, sig), k, u in GEOMETRY_CASES:
        assert k and u, "every case claims facts"
        assert (rows_per_rec * K) % P.TILE_ELEMS == 0 and rows_per_rec % 128 == 0 and K % 32 == 0
        for q in range(N):
            assert case_facts(N, K, rows_per_rec, R, Nb, grid, rank=q) == (k, u), (N, K, rows_per_rec, R, Nb, grid, q)
        assert 16 + N * (gather_grid(N, grid) + 2) <= 132, "SM budget"
        seen_k |= k
        seen_u |= u
    assert seen_k == set(GEMM_FACTS) and seen_u == set(UNPACK_FACTS)
    cases = [c for c, _, _ in GEOMETRY_CASES]
    assert {c[0] for c in cases} == set(range(2, 9))
    assert min(c[4] for c in cases) == 1 and max(c[4] for c in cases) == 4096
    assert {1, 3, 7, 0} <= {c[5] for c in cases}
    assert {1, 3, 8} <= {c[6] for c in cases}
