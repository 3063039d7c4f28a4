"""The fp8 ring reduce-scatter's schedule, the GEMM walk its plan builds and its limits, on the CPU.

The schedule model runs N ranks whose step k posts the records of shard (q-1-k) mod N, a step only once the records it
adds have arrived, and checks that every rank receives every id once, reads what the previous rank wrote one step
earlier, and ends with its own shard."""
import random

import pytest

from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import reduce_scatter_fp8 as RS
from rocnrdma_b200.parallel import ring_fp8 as RF


def _simulate(N, R, seed):
    """Ranks take turns in a random order; a rank's next step runs once every record it adds has landed.  Returns, per
    rank, the ids received in arrival order, and per (rank, id) the (writer, writer's step, shard) it came from."""
    rng = random.Random(seed)
    steps = [RS.schedule(q, N) for q in range(N)]
    nxt = [0] * N
    landed = [dict() for _ in range(N)]          # id -> (writer rank, writer step, shard)
    got = [[] for _ in range(N)]
    while any(k < N for k in nxt):
        ready = [q for q in range(N) if nxt[q] < N and (steps[q][nxt[q]].read_slot is None or
                 all(steps[q][nxt[q]].read_slot * R + r in landed[q] for r in range(R)))]
        assert ready, f"the ring deadlocks at steps {nxt}"
        q = rng.choice(ready)
        k = nxt[q]
        st = steps[q][k]
        if st.read_slot is not None:
            for r in range(R):
                writer, wstep, shard = landed[q][st.read_slot * R + r]
                assert writer == (q - 1) % N and wstep == k - 1 and shard == st.shard, (q, k, r)
        if st.send_slot is not None:
            d = (q + 1) % N
            for r in range(R):
                i = st.send_slot * R + r
                assert i not in landed[d], f"rank {d} receives id {i} twice"
                landed[d][i] = (q, k, st.shard)
                got[d].append(i)
        nxt[q] += 1
    return got


@pytest.mark.parametrize("N", range(2, 9))
@pytest.mark.parametrize("R", [1, 3])
def test_every_rank_receives_every_id_once(N, R):
    for seed in range(4):
        got = _simulate(N, R, seed)
        for q in range(N):
            assert sorted(got[q]) == list(range((N - 1) * R)), q


@pytest.mark.parametrize("N", range(2, 9))
def test_the_last_step_is_the_own_shard(N):
    for q in range(N):
        st = RS.schedule(q, N)
        assert [s.shard for s in st] == [(q - 1 - k) % N for k in range(N)]
        assert st[-1].shard == q and st[-1].send_slot is None and st[0].read_slot is None
        assert sorted(s.shard for s in st) == list(range(N))


@pytest.mark.parametrize("N", range(2, 9))
@pytest.mark.parametrize("R", [1, 2, 3])
def test_gemm_ids_follow_the_schedule(N, R):
    for q in range(N):
        walk, add, send = RS.gemm_ids(q, N, R)
        assert sorted(walk) == list(range(N * R)), "every m-block of the product once"
        for k, st in enumerate(RS.schedule(q, N)):
            for r in range(R):
                p = k * R + r
                assert walk[p] == st.shard * R + r
                assert add[p] == (-1 if k == 0 else (k - 1) * R + r)
                assert send[p] == (k * R + r if k < N - 1 else -1)
        # the j-th bf16 position stores rows [128 j, 128 j + 128) of out: rank q's own shard, in row order
        assert [walk[p] for p in range(N * R) if send[p] < 0] == [q * R + r for r in range(R)]
        sends = [s for s in send if s >= 0]
        assert sorted(sends) == list(range((N - 1) * R))


class _NoGpu:
    device = 0


@pytest.mark.parametrize("N", range(2, 9))
def test_queue_capacity_refused_before_allocation(N):
    m = RS.max_records(N)
    assert RF._pow2(2 * (N - 1) * m) <= RF.MAX_QUEUE_DEPTH < RF._pow2(2 * (N - 1) * (m + 1))
    chunk = P.TILE_ELEMS
    with pytest.raises(ValueError, match="receive queue"):
        RS.RingReduceScatterFp8(_NoGpu(), (m + 1) * chunk, chunk, 0, N)


def test_plan_refuses_bad_geometry():
    for args, what in [((8192, 8192, 0, 1), "at least 2"), ((3 * 8192, 2 * 8192, 0, 2), "multiple of chunk"),
                       ((8192, 100, 0, 2), "multiple of 8192"), ((8192, 8192, 2, 2), "outside")]:
        with pytest.raises(ValueError, match=what):
            RS.RingReduceScatterFp8(_NoGpu(), *args)


@pytest.mark.parametrize("N", range(2, 9))
def test_sm_budget_arithmetic(monkeypatch, N):
    """engine + N (grid + 1): the plan's one waiter beside its grid is the consumer.  The budget itself is checked when
    the plans are linked (link_in_process, connect), once the ranks on the GPU are known."""
    monkeypatch.setattr(RF, "_sms", lambda ctx: 132)
    assert RS.RingReduceScatterFp8.WAITERS == 1
    for engine in (8, 16, 32):
        RF._check_budget(None, engine, N, RF._default_grid(None, engine, N, 1), 1)
        for grid in range(1, 130):
            if engine + N * (grid + 1) <= 132:
                RF._check_budget(None, engine, N, grid, 1)
            else:
                with pytest.raises(ValueError, match="SM budget"):
                    RF._check_budget(None, engine, N, grid, 1)


def _raster(P, n_blks, group_m):
    """tile_coords of gemm_send.cu: tile t -> (walk position, n-block); group_m positions advance together across the
    n-blocks, the position fastest inside a group, the last group possibly short."""
    out = []
    for t in range(P * n_blks):
        per_group = group_m * n_blks
        grp, r = t // per_group, t % per_group
        m0 = grp * group_m
        gm = min(group_m, P - m0)
        out.append((m0 + r % gm, r // gm))
    return out


def _cta_steps_in_order(N, R, n_blks, group_m, grid):
    """True when every CTA (round robin: CTA u takes tiles u, u + grid, ...) meets its tiles in step order."""
    tiles = _raster(N * R, n_blks, group_m)
    for u in range(grid):
        steps = [tiles[t][0] // R for t in range(u, len(tiles), grid)]
        if steps != sorted(steps):
            return False
    return True


@pytest.mark.parametrize("n_blks", [1, 2, 3])
def test_raster_model_covers_every_tile_once(n_blks):
    for P, g in ((6, 4), (8, 4), (5, 2), (7, 1)):
        assert sorted(_raster(P, n_blks, g)) == [(m, n) for m in range(P) for n in range(n_blks)]


@pytest.mark.parametrize("R", range(1, 13))
def test_each_cta_meets_its_tiles_in_step_order(R):
    """The plan's group_m divides R, so a raster group never holds two steps and every CTA's tiles are in step order,
    whatever the grid and the n-blocks: the order the deadlock argument needs (DESIGN.md 3.4)."""
    g = next(v for v in (4, 2, 1) if R % v == 0)
    for N in (2, 3, 8):
        for n_blks in (1, 2, 3, 32):
            for grid in (1, 2, 3, 7, 28, 57):
                assert _cta_steps_in_order(N, R, n_blks, g, grid), (N, n_blks, grid)


def test_a_group_that_straddles_steps_breaks_the_order():
    """The model is not vacuous: group_m = 4 with R = 3 and two n-blocks puts a step-1 tile of a CTA before step-0
    tiles of the same CTA (steps 0, 0, 0, 1, 0, 0, 0, 1 along the raster)."""
    tiles = _raster(2 * 3, 2, 4)
    assert [m // 3 for m, _ in tiles][:8] == [0, 0, 0, 1, 0, 0, 0, 1]
    assert not _cta_steps_in_order(2, 3, 2, 4, grid=2)
