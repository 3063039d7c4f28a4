"""The fp8 ring reduce-scatter's schedule, the GEMM walk its plan builds and its limits, on the CPU.

The schedule model runs N ranks whose step k posts the records of shard (q-1-k) mod N, a step only once the records it
adds have arrived, and checks that every rank receives every id once, reads what the previous rank wrote one step
earlier, and ends with its own shard."""
import random
from typing import NamedTuple

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


# ------------------------------------------------------------------ the fused walk (test_gpu_reduce_scatter_fp8_shapes.py)
H100_SMS = 132
BN, BK, STAGES = 256, 64, 3             # gemm_send.cu: the tile's columns, its k-block and the operand ring's stages


class Tile(NamedTuple):
    """One tile of the walk: walk position p, its step, n-block, m-block of ``a``, landed record added (-1: none), record
    posted (-1: none) and, for a bf16 position, the 128-row block of ``out`` it stores (``j_out``; -1 otherwise)."""
    p: int
    step: int
    n_blk: int
    m_blk: int
    add: int
    send: int
    j_out: int


class ReduceScatterWalk:
    """``run_gemm``'s one ``gemm_reduce_send`` on rank ``rank`` of N, for R 128-row panels per shard, an Nb-column
    product and K_l = K: the grid clamped to the SMs and to the tiles (``rn_k_gemm_reduce_send``), CTA u's tiles u,
    u + grid, ... (``next_seg`` without stream-K), each mapped by ``tile_coords`` with the plan's ``group_m`` to a walk
    position and an n-block, and each walk position through ``gemm_ids`` to its step, m-block and ids.  ``tiles[u]``
    lists CTA u's tiles in the order it meets them."""

    def __init__(self, N, R, Nb, K, grid, rank=0, sms=H100_SMS):
        self.N, self.R, self.Nb, self.K = N, R, Nb, K
        self.P, self.n_blks, self.k_blks = N * R, -(-Nb // BN), -(-K // BK)
        self.n_tiles = self.P * self.n_blks
        self.group_m = next(g for g in (4, 2, 1) if R % g == 0)          # RingReduceScatterFp8
        self.requested = sms if grid <= 0 or grid > sms else grid
        self.grid = min(self.requested, self.n_tiles)
        walk, add, send = RS.gemm_ids(rank, N, R)
        raster = _raster(self.P, self.n_blks, self.group_m)
        self.tiles = []
        for u in range(self.grid):
            mine = []
            for t in range(u, self.n_tiles, self.grid):
                p, n = raster[t]
                j_out = sum(1 for i in range(p) if send[i] < 0) if send[p] < 0 else -1
                mine.append(Tile(p, p // R, n, walk[p], add[p], send[p], j_out))
            self.tiles.append(mine)

    def facts(self):
        owners = {}
        for u, ts in enumerate(self.tiles):
            for t in ts:
                owners.setdefault(t.p, set()).add(u)

        def bf16_after_posts(ts):
            posted = False
            for t in ts:
                if t.send >= 0:
                    posted = True
                elif posted and t.j_out > 0:
                    return True
            return False

        return {
            "cta_crosses_steps": any(len({t.step for t in ts}) >= 2 for ts in self.tiles),
            "panel_shared": any(len(us) >= 2 for us in owners.values()),
            "cta_starts_gated": any(ts[0].add >= 0 for ts in self.tiles),
            "bf16_after_posts": any(bf16_after_posts(ts) for ts in self.tiles),
            "ragged_n": self.Nb % BN != 0,
            "narrow_n": self.Nb < 128,
            "partial_k": self.K % BK != 0,
            # a CTA's second tile starts at stage k_blks mod 3 of the operand ring: not stage 0
            "mid_ring_entry": self.k_blks % STAGES != 0 and any(len(ts) >= 2 for ts in self.tiles),
            "clamped_grid": self.requested > self.n_tiles,
            "one_cta_walks_every_step": any(len({t.step for t in ts}) == self.N for ts in self.tiles),
        }


WALK_FACTS = ("cta_crosses_steps", "panel_shared", "cta_starts_gated", "bf16_after_posts", "ragged_n", "narrow_n",
              "partial_k", "mid_ring_entry", "clamped_grid", "one_cta_walks_every_step")


@pytest.mark.parametrize("N", [2, 3, 5, 8])
def test_walk_model_covers_every_tile_in_step_order(N):
    """Every rank's model walk holds every (walk position, n-block) once, each CTA meets its tiles in step order, the
    bf16 positions store out's row blocks 0..R-1 in turn, and the facts are the same on every rank."""
    for R, Nb, K, grid in [(1, 64, 8, 1), (3, 320, 200, 2), (4, 512, 64, 3), (2, 4096, 640, 0), (6, 256, 128, 500)]:
        facts = None
        for q in range(N):
            w = ReduceScatterWalk(N, R, Nb, K, grid, rank=q)
            assert sorted((t.p, t.n_blk) for ts in w.tiles for t in ts) == [(p, n) for p in range(N * R)
                                                                              for n in range(w.n_blks)]
            for ts in w.tiles:
                assert [t.step for t in ts] == sorted(t.step for t in ts), (R, Nb, grid, q)
                for t in ts:
                    assert (t.send < 0) == (t.step == N - 1) and (t.add < 0) == (t.step == 0)
                    assert t.j_out == (t.p - (N - 1) * R if t.step == N - 1 else -1)
                    assert t.m_blk == RS.schedule(q, N)[t.step].shard * R + t.p % R
            facts = facts or w.facts()
            assert w.facts() == facts


def test_walk_model_hand_counted_walks():
    # N 2, R 1, Nb 64, K 8, grid 1: one CTA, positions 0 (posted as record 0) then 1 (adds record 0, bf16 row block 0)
    w = ReduceScatterWalk(2, 1, 64, 8, 1, rank=0)
    assert w.grid == 1 and w.group_m == 1 and w.k_blks == 1
    assert w.tiles == [[Tile(0, 0, 0, 1, -1, 0, -1), Tile(1, 1, 0, 0, 0, -1, 0)]]
    f = w.facts()
    assert f["cta_crosses_steps"] and f["one_cta_walks_every_step"] and f["narrow_n"] and f["ragged_n"]
    assert f["partial_k"] and f["mid_ring_entry"]                    # k_blks 1: the second tile enters at stage 1
    assert not f["panel_shared"] and not f["cta_starts_gated"] and not f["bf16_after_posts"] and not f["clamped_grid"]
    # N 2, R 4 (group_m 4), Nb 512 (two n-blocks), K 192 (three k-blocks), grid 3: tile t is position 4 (t // 8) + t % 4,
    # n-block (t // 8) % 2; rank 0's step 0 is shard 1 (m-blocks 4..7), its step 1 shard 0 (bf16 row blocks 0..3)
    w = ReduceScatterWalk(2, 4, 512, 192, 3, rank=0)
    assert w.group_m == 4 and w.n_blks == 2 and w.grid == 3 and w.k_blks == 3
    assert [(t.p, t.n_blk) for t in w.tiles[0]] == [(0, 0), (3, 0), (2, 1), (5, 0), (4, 1), (7, 1)]
    assert [(t.p, t.n_blk) for t in w.tiles[1]] == [(1, 0), (0, 1), (3, 1), (6, 0), (5, 1)]
    assert [(t.p, t.n_blk) for t in w.tiles[2]] == [(2, 0), (1, 1), (4, 0), (7, 0), (6, 1)]
    assert [t.m_blk for t in w.tiles[0]] == [4, 7, 6, 1, 0, 3]
    assert [t.j_out for t in w.tiles[0]] == [-1, -1, -1, 1, 0, 3]
    assert [(t.add, t.send) for t in w.tiles[0]] == [(-1, 0), (-1, 3), (-1, 2), (1, -1), (0, -1), (3, -1)]
    f = w.facts()
    assert f["panel_shared"] and f["bf16_after_posts"] and f["cta_crosses_steps"] and f["one_cta_walks_every_step"]
    assert not f["cta_starts_gated"] and not f["mid_ring_entry"] and not f["ragged_n"] and not f["partial_k"]
    assert not f["narrow_n"] and not f["clamped_grid"]
    # N 3, R 1, grid 7 clamped to 3 tiles: each CTA one position, CTAs 1 and 2 start gated, none crosses a step
    w = ReduceScatterWalk(3, 1, 192, 1000, 7)
    assert w.grid == 3 and [[t.p for t in ts] for ts in w.tiles] == [[0], [1], [2]]
    f = w.facts()
    assert f["clamped_grid"] and f["cta_starts_gated"] and f["ragged_n"] and f["partial_k"]
    assert not f["cta_crosses_steps"] and not f["mid_ring_entry"] and not f["bf16_after_posts"]
    assert not f["panel_shared"] and not f["one_cta_walks_every_step"]
    # the default grid (all 132 SMs), 8 positions of 32 n-blocks, group_m 4 (128 tiles a group): CTA 0 takes tiles 0 and
    # 132, CTA 123 tiles 123 and 255, CTA 131 only tile 131
    w = ReduceScatterWalk(2, 4, 8192, 64, 0)
    assert w.grid == 132 and [(t.p, t.n_blk) for t in w.tiles[0]] == [(0, 0), (4, 1)]
    assert [(t.p, t.n_blk) for t in w.tiles[123]] == [(3, 30), (7, 31)]
    assert [(t.p, t.n_blk) for t in w.tiles[131]] == [(7, 0)]
    assert [u for u, ts in enumerate(w.tiles) if ts[0].add >= 0] == [128, 129, 130, 131]   # 128 step-0 tiles, 132 CTAs
    f = w.facts()
    assert f["panel_shared"] and f["cta_crosses_steps"] and f["bf16_after_posts"] and f["mid_ring_entry"]
    assert f["cta_starts_gated"] and not f["clamped_grid"] and not f["ragged_n"]


def test_geometry_cases_cover_every_fact_and_parameter():
    """The GPU geometry cases (test_gpu_reduce_scatter_fp8_shapes.py): each claims facts of the fused walk and of a
    reduce hop, the same on every rank; together they cover every walk fact, N = 2..8, every group_m, signal_every of
    1, of more than 1 and of more than R, and every reduce-hop fact a hop of ``run`` can have.  A hop runs the reduce
    with the addend and P = 1, whose steps hold G = 2 tiles, so a step never holds a run of two tiles beside a run of
    another record: ``boundary_in_step`` cannot occur."""
    from test_gpu_reduce_schedule import ReduceSchedule, variant_of
    from test_gpu_reduce_scatter_fp8_shapes import GEOMETRY_CASES, case_facts
    from test_gpu_ring_fp8_shapes import REDUCE_FACTS, ring_grid
    seen_w, seen_r, group_ms = set(), set(), set()
    for (N, K, R, Nb, grid, sig), w, r in GEOMETRY_CASES:
        assert w and r, "every case claims facts"
        assert Nb % 64 == 0 and K % 8 == 0
        for q in range(N):
            assert case_facts(N, K, R, Nb, grid, rank=q) == (w, r), (N, K, R, Nb, grid, q)
        assert 16 + N * (ring_grid(N, grid) + 1) <= 132, "SM budget"
        seen_w |= w
        seen_r |= r
        group_ms.add(ReduceScatterWalk(N, R, Nb, K, ring_grid(N, grid)).group_m)
    assert variant_of(1, True)[0] == 2
    assert not any(ReduceSchedule(128 * nb, r, 1, local=True, grid=g, ready=True).facts()["boundary_in_step"]
                   for nb in (64, 128, 320, 4096) for r in (1, 2, 5) for g in (1, 2, 3, 57))
    assert seen_w == set(WALK_FACTS) and seen_r == set(REDUCE_FACTS) - {"boundary_in_step"}
    cases = [c for c, _, _ in GEOMETRY_CASES]
    assert {c[0] for c in cases} == set(range(2, 9))
    assert group_ms == {1, 2, 4}
    assert any(ReduceScatterWalk(N, R, Nb, K, ring_grid(N, g)).n_blks >= 2 and R % 4 != 0 and R % 2 == 0
               for N, K, R, Nb, g, _ in cases), "group_m 2 with several n-blocks"
    assert any(ReduceScatterWalk(N, R, Nb, K, ring_grid(N, g)).n_blks > 2 for N, K, R, Nb, g, _ in cases)
    assert 1 in {c[5] for c in cases} and any(1 < sig <= R for _, _, R, _, _, sig in cases)
    assert any(sig > R for _, _, R, _, _, sig in cases)
