"""The fp8 ring all-gather and the all-gather GEMM on one GPU at the record geometries where their kernels' walks get
hard, at the largest plans the receive queue allows, at the benchmark's shapes, on the edge payload, over repeated runs
of one engine session, with a rank that never contributes to the GEMM, and as the first run of a fresh process.

* `OrderedGatherSchedule` mirrors ``launch_mx`` and ``mx_body<1, true>`` of gemm_mxfp8.cu as ``run_gemm`` launches
  them: the grid clamped to the tile count, CTA u's tiles u, u + grid, ..., each mapped through ``a_order`` (the plan's
  arrival order) to a record, one of its 128-row blocks and a 128-column block, and each record to its slot and that
  slot's place in the arrival order.  ``run``'s gated unpack of each slot (``unpack_fp8_kernel<false>`` with arrival
  words) walks a slot as test_gpu_ring_fp8_shapes.py's `UnpackSchedule` does.  Every geometry case asserts the facts
  of both walks it is there for; test_allgather_fp8_schedule.py checks the model against hand-counted walks.
* Shards from `exact_shard` (test_allgather_fp8_references.py) against ``_mx_exact_operand`` weights give K7 block
  partials of at most 11 significant bits, so every rank's C must equal ``ops.ref_gemm_mxfp8`` of the gathered records
  bit for bit.  ``out`` and the records must equal ``ops.ref_allgather_fp8`` (up to the sign of NaN on the edge
  payload).  Each rank receives and posts (N-1)R records a run, and its send queue grows by those records and one
  flush.

The rules of test_gpu_ring_fp8.py hold: every wait is bounded by 5 s or less, nothing allocates or synchronises the
device while the engine runs, landing regions start as poison, the guard words behind the arrival words stay zero, and
each case writes out its SM budget (engine CTAs + N x (grid + 2) of 132: the consumer and the relay wait beside the
grid).
"""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import gemm_mx as MX, pack as P
from rocnrdma_b200.parallel import allgather_fp8 as AG
from test_allgather_fp8_references import exact_shard, model_allgather, record_fields
from test_gpu_mx_range import _check_against_reference, _edge_matrix
from test_gpu_numerics import H100_SMS, _mx_exact_operand
from test_gpu_receive_fusion import _check_arrival_words
from test_gpu_ring_fp8 import WAIT_MS, _poison
from test_gpu_ring_fp8_shapes import ENGINE_CTAS, UnpackSchedule, _sm_budget, _spread_gpu, ring_grid
from test_ring_fp8_references import CHUNK, assert_bits_equal, edge_payload

pytestmark = pytest.mark.gpu

WAITERS = AG.RingAllgatherFp8.WAITERS
BM = BN = BK = 128
STAGES = 4                      # K7's operand ring


# ------------------------------------------------------------------ schedule model of the ordered K7 inside the gather
class OrderedGatherSchedule:
    """``gemm_mxfp8(a_order=plan.a_order, cta_group=1)`` over rank ``rank``'s landing region of N slots of R records of
    ``rows_per_rec`` x K, against Nb columns: ``tiles[u]`` lists CTA u's walk indices, ``walk[t]`` the (record, m-block,
    n-block) of walk index t."""

    def __init__(self, N, rank, K, rows_per_rec, R, Nb, grid, sms=H100_SMS):
        self.N, self.rank, self.R, self.K, self.Nb = N, rank, R, K, Nb
        self.bpr, self.n_blks, self.k_blks = rows_per_rec // BM, -(-Nb // BN), -(-K // BK)
        self.n_rec = N * R
        self.n_tiles = self.n_rec * self.bpr * self.n_blks
        self.requested = grid
        g = sms if grid <= 0 or grid > sms else grid                    # launch_mx: one CTA per SM at most
        self.grid = min(g, self.n_tiles)
        self.order = [s * R + r for s in AG.arrival_slots(rank, N) for r in range(R)]
        per_rec = self.bpr * self.n_blks
        self.walk = []
        for t in range(self.n_tiles):
            rec = self.order[t // per_rec]
            self.walk.append((rec, rec * self.bpr + (t % per_rec) // self.n_blks, t % self.n_blks))
        self.tiles = [list(range(u, self.n_tiles, self.grid)) for u in range(self.grid)]

    def slot(self, rec):
        return rec // self.R

    def place(self, rec):
        """The slot's place in this rank's arrival order: 0 for its own, N - 1 for the last to land."""
        return AG.arrival_slots(self.rank, self.N).index(self.slot(rec))

    def coords(self):
        """(m-block, n-block) of every walk index, as test_allgather_fp8_schedule.py's ``_ordered_walk`` gives them."""
        return [(m, n) for _, m, n in self.walk]

    def facts(self):
        owners = {}
        for u, ts in enumerate(self.tiles):
            for t in ts:
                owners.setdefault(self.walk[t][0], set()).add(u)
        return {
            "multi_block_records": self.bpr > 1,
            "cta_crosses_slots": any(len({self.slot(self.walk[t][0]) for t in ts}) >= 2 for ts in self.tiles),
            "cta_starts_remote": any(self.slot(self.walk[ts[0]][0]) != self.rank for ts in self.tiles),
            "record_shared": any(len(us) >= 2 for us in owners.values()),
            "ragged_n": self.Nb % BN != 0,
            "odd_n": self.Nb % 2 == 1,
            "partial_k": self.K % BK != 0,
            # the operand ring's stage of a CTA's second tile is k_blks mod 4: not stage 0
            "mid_ring_entry": self.k_blks % STAGES != 0 and any(len(ts) >= 2 for ts in self.tiles),
            "clamped_grid": self.requested > self.n_tiles,
        }


GEMM_FACTS = ("multi_block_records", "cta_crosses_slots", "cta_starts_remote", "record_shared", "ragged_n", "odd_n",
              "partial_k", "mid_ring_entry", "clamped_grid")
UNPACK_FACTS = ("record_raced", "waits_on_a_later_record", "partial_last_step", "clamped_grid")


def gather_grid(N, grid):
    """The grid of every launch of an in-process gather of N ranks: ``grid``, or the default beside two waiters."""
    return ring_grid(N, grid, WAITERS)


def case_facts(N, K, rows_per_rec, R, Nb, grid, rank=0):
    """The ordered K7's facts on ``rank`` and the gated unpack's (one slot, as every slot) at one geometry."""
    g = gather_grid(N, grid)
    k = OrderedGatherSchedule(N, rank, K, rows_per_rec, R, Nb, g).facts()
    u = UnpackSchedule(rows_per_rec * K, R, g).facts()
    return {f for f in GEMM_FACTS if k[f]}, {f for f in UNPACK_FACTS if u[f]}


# (N, K, rows per record, R, Nb, grid (0: default), signal_every), with the ordered K7's and the gated unpack's facts
GEOMETRY_CASES = [
    ((2, 32, 256, 3, 1, 1, 3),
     {"cta_crosses_slots", "mid_ring_entry", "multi_block_records", "odd_n", "partial_k", "ragged_n"},
     {"partial_last_step", "waits_on_a_later_record"}),
    ((2, 4096, 512, 2, 4096, 0, 1),
     {"cta_crosses_slots", "multi_block_records", "record_shared"},
     {"partial_last_step", "record_raced", "waits_on_a_later_record"}),
    ((3, 64, 128, 2, 200, 7, 1),
     {"cta_crosses_slots", "cta_starts_remote", "mid_ring_entry", "partial_k", "ragged_n", "record_shared"},
     {"clamped_grid", "partial_last_step"}),
    ((3, 640, 128, 3, 1000, 7, 3),
     {"cta_crosses_slots", "mid_ring_entry", "ragged_n", "record_shared"},
     {"partial_last_step", "record_raced", "waits_on_a_later_record"}),
    ((4, 96, 256, 3, 136, 3, 8),
     {"cta_crosses_slots", "mid_ring_entry", "multi_block_records", "partial_k", "ragged_n", "record_shared"},
     {"partial_last_step", "record_raced", "waits_on_a_later_record"}),
    ((4, 4096, 128, 2, 129, 0, 8),
     {"clamped_grid", "cta_starts_remote", "odd_n", "ragged_n", "record_shared"},
     {"partial_last_step", "record_raced", "waits_on_a_later_record"}),
    ((5, 160, 256, 2, 391, 0, 3),
     {"cta_crosses_slots", "cta_starts_remote", "mid_ring_entry", "multi_block_records", "odd_n", "partial_k",
      "ragged_n", "record_shared"},
     {"clamped_grid", "partial_last_step", "record_raced"}),
    ((6, 4096, 128, 1, 1, 17, 1),
     {"clamped_grid", "cta_starts_remote", "odd_n", "ragged_n"},
     {"partial_last_step", "record_raced"}),
    ((7, 1152, 128, 2, 256, 1, 8),
     {"cta_crosses_slots", "mid_ring_entry"},
     {"waits_on_a_later_record"}),
    ((8, 4096, 128, 1, 4096, 0, 3),
     {"cta_crosses_slots", "record_shared"},
     {"partial_last_step", "record_raced"}),
    ((8, 64, 128, 4, 1, 3, 1),
     {"cta_crosses_slots", "mid_ring_entry", "odd_n", "partial_k", "ragged_n"},
     {"partial_last_step", "waits_on_a_later_record"}),
]
GEOMETRY_IDS = [f"N{n}-K{k}-rows{r}-R{R}-Nb{nb}-grid{g or 'default'}-sig{s}" for (n, k, r, R, nb, g, s), _, _ in GEOMETRY_CASES]


# ------------------------------------------------------------------ running and checking
def _plans(ctx, N, chunk, R, grid=0, signal_every=1, timeout_ms=WAIT_MS):
    plans = [AG.RingAllgatherFp8(ctx, R * chunk, chunk, q, N, grid=grid, timeout_ms=timeout_ms,
                                 signal_every=signal_every, engine_ctas=ENGINE_CTAS) for q in range(N)]
    AG.link_in_process(plans)
    return plans


def _session(ctx, plans, runs):
    """``runs``: callables that each run every rank once (``run_in_process`` or ``run_gemm_in_process``), back to back
    in one engine session from poisoned landing regions.  Returns each run's results and each rank's send-queue WQE
    growth."""
    for p in plans:
        _poison(p.landing, p.chunk)
    wqe0 = [p.send_qp.counters()["n_wqe"] for p in plans]
    torch.cuda.synchronize()
    results = []
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        for run in runs:
            results.append(run())
    finally:
        ctx.engine_stop()
    return results, [p.send_qp.counters()["n_wqe"] - w for p, w in zip(plans, wqe0)]


def _check_runs(plans, results, growth):
    """Every launch OK, (N-1)R records received and posted a run, one flush a run, the words stamped, no guard word
    written, no work request in error."""
    N, R = plans[0].world, plans[0].R
    for res in results:
        for r in res:
            assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
            assert r.received == r.posted == (N - 1) * R, (r.rank, r.received, r.posted)
    assert growth == [len(results) * ((N - 1) * R + 1)] * N, growth
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0


def _same_on_every_rank(ts, what):
    for q, t in enumerate(ts):
        assert torch.equal(t.view(torch.int16), ts[0].view(torch.int16)), f"rank {q}'s {what} differs from rank 0's"


def _mismatch(c, ref):
    d = (c.view(torch.int16) != ref.view(torch.int16)).nonzero()
    if d.numel() == 0:
        return ""
    i, j = d[0].tolist()
    return f"{d.shape[0]} outputs differ, first at ({i}, {j}): got {c[i, j].item()}, want {ref[i, j].item()}"


def _check_exact_c(cs, recs, chunk, K, bq, bs, rows=None):
    """Every rank's C identical, and equal bit for bit to ``ref_gemm_mxfp8`` of the gathered records (on ``rows``
    only, when given)."""
    _same_on_every_rank(cs, "C")
    aq, as_ = record_fields(recs.cuda(), chunk, K)
    c = cs[0]
    if rows is not None:
        aq, as_, c = aq[rows], as_[rows], c[rows]
    ref = MX.ref_gemm_mxfp8(aq.contiguous(), as_.contiguous(), bq, bs)
    assert torch.equal(c.view(torch.int16), ref.view(torch.int16)), _mismatch(c, ref)


def _check_gather(plans, outs, want, want_rec):
    """Every rank's ``out`` and records bit for bit against the reference."""
    for q, p in enumerate(plans):
        assert torch.equal(outs[q].view(torch.int16), want.view(torch.int16)), f"rank {q}'s out differs from the reference"
        assert torch.equal(p.records(), want_rec), f"rank {q}'s gathered records"


def _bf16_full(shape, value=7.0):
    return torch.full(shape, value, dtype=torch.bfloat16, device="cuda")


# ------------------------------------------------------------------ 1. record geometries
@pytest.mark.parametrize("case,gemm_claims,unpack_claims", GEOMETRY_CASES, ids=GEOMETRY_IDS)
def test_allgather_geometry(ctx, case, gemm_claims, unpack_claims):
    """``run_gemm`` on exact shards, then ``run`` on other exact shards, in one engine session: C against the exact
    reference on every rank, ``out`` and the records against the gather's reference."""
    N, K, rows_per_rec, R, Nb, grid, sig = case
    assert case_facts(N, K, rows_per_rec, R, Nb, grid) == (gemm_claims, unpack_claims)
    _sm_budget(N, grid, WAITERS)
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    plans = _plans(ctx, N, chunk, R, grid, sig)
    g = torch.Generator().manual_seed(8000 + 100 * N + R)
    xg = [exact_shard(rows, K, g).cuda() for _ in range(N)]
    xr = [exact_shard(rows, K, g).reshape(-1).cuda() for _ in range(N)]   # other records: a slot read early differs
    bq, bs = _mx_exact_operand(Nb, K, g)
    b = MX.MxOperand.from_tensors(bq, bs)
    cs = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    outs = [_bf16_full((N * rows * K,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [lambda: AG.run_gemm_in_process(plans, xg, [b] * N, cs),
                                            lambda: AG.run_in_process(plans, xr, outs)])
    _check_runs(plans, results, growth)
    _check_exact_c(cs, ops.ref_allgather_fp8(xg, chunk)[1], chunk, K, bq, bs)
    _check_gather(plans, outs, *ops.ref_allgather_fp8(xr, chunk))


# ------------------------------------------------------------------ 2. the largest plans the receive queue allows
def _sample_rows(n_slots, R, rows_per_rec, seed):
    """Every row of the first and last record of each slot, and a seeded 1/64 of the other rows."""
    M = n_slots * R * rows_per_rec
    pick = torch.zeros(M, dtype=torch.bool)
    for s in range(n_slots):
        for r in (s * R, s * R + R - 1):
            pick[r * rows_per_rec:(r + 1) * rows_per_rec] = True
    g = torch.Generator().manual_seed(seed)
    pick[torch.randint(0, M, (M // 64,), generator=g)] = True
    return pick.nonzero().flatten().cuda()


@pytest.mark.parametrize("N,R", [(2, 8192), (8, 1170)])
def test_allgather_largest_legal_plan(ctx, N, R):
    """R = max_records(N) with chunk 8192: the receive queue at 16384 entries, and a relay of (N-1)R records through
    the 256-deep send queue.  ``run`` on spread shards, every element exact; at N = 2 also ``run_gemm`` with K = 64,
    128-row records and Nb = 136, C against K7 without an order in full and against the exact reference on sampled
    rows.  SMs: engine 16 + N x (default grid + 2) <= 132."""
    assert R == AG.max_records(N)
    _sm_budget(N, 0, WAITERS)
    chunk = 8192
    plans = _plans(ctx, N, chunk, R)
    assert plans[0].recv_qp.rq_depth == AG.MAX_QUEUE_DEPTH
    xs = _spread_gpu(N, R * chunk, seed=8500 + N)
    outs = [_bf16_full((N * R * chunk,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [lambda: AG.run_in_process(plans, xs, outs)])
    _check_runs(plans, results, growth)
    _check_gather(plans, outs, *ops.ref_allgather_fp8(xs, chunk))
    del outs
    if N != 2:
        return
    K, rows_per_rec, Nb = 64, 128, 136
    rows = R * rows_per_rec
    g = torch.Generator().manual_seed(8600)
    xg = [exact_shard(rows, K, g).cuda() for _ in range(N)]
    bq, bs = _mx_exact_operand(Nb, K, g)
    b = MX.MxOperand.from_tensors(bq, bs)
    cs = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    results, growth = _session(ctx, plans, [lambda: AG.run_gemm_in_process(plans, xg, [b] * N, cs)])
    _check_runs(plans, results, growth)
    want_rec = ops.ref_allgather_fp8(xg, chunk)[1]
    for q, p in enumerate(plans):
        assert torch.equal(p.records(), want_rec), f"rank {q}'s gathered records"
    c0 = torch.zeros_like(cs[0])
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_chunk_records(plans[0].records(), N * rows, K, chunk), b, c0,
                          cta_group=1).ok
    for q in range(N):
        assert torch.equal(cs[q].view(torch.int16), c0.view(torch.int16)), f"rank {q}'s C differs from K7 without an order"
    _check_exact_c(cs, want_rec, chunk, K, bq, bs, rows=_sample_rows(N, R, rows_per_rec, seed=8601))


# ------------------------------------------------------------------ 3. the benchmark's shapes
@pytest.mark.parametrize("Nb", [4096, 8192])
@pytest.mark.parametrize("N", [2, 4])
def test_allgather_at_the_benchmark_shape(ctx, N, Nb):
    """tools/allgather_bench.py's shapes: a total M of 8192, K = 4096, 256-row records, the default grid.  In one
    session: ``run_gemm`` on exact shards (C against the exact reference, computed on the GPU), ``run_gemm`` on the
    bench's own inputs (C identical on every rank and to K7 without an order, and within K7's fp64 bound on the
    first and last record of every slot), then ``run`` of the bench's inputs (``out`` and records exact)."""
    M, K = 8192, 4096
    chunk, rows = 256 * K, M // N
    R = rows * K // chunk
    _sm_budget(N, 0, WAITERS)
    plans = _plans(ctx, N, chunk, R)
    g = torch.Generator().manual_seed(8700 + N + Nb)
    xe = [exact_shard(rows, K, g).cuda() for _ in range(N)]
    xb = [torch.randn(rows, K, generator=g).to(torch.bfloat16).cuda() for _ in range(N)]
    eq, es = _mx_exact_operand(Nb, K, g)
    bq, bs = MX.quantize_mx(torch.randn(Nb, K, generator=g).to(torch.bfloat16).cuda())
    be, bb = MX.MxOperand.from_tensors(eq, es), MX.MxOperand.from_tensors(bq, bs)
    ce = [_bf16_full((M, Nb)) for _ in range(N)]
    cb = [_bf16_full((M, Nb)) for _ in range(N)]
    outs = [_bf16_full((M * K,)) for _ in range(N)]
    xb_flat = [x.reshape(-1) for x in xb]
    results, growth = _session(ctx, plans, [lambda: AG.run_gemm_in_process(plans, xe, [be] * N, ce),
                                            lambda: AG.run_gemm_in_process(plans, xb, [bb] * N, cb),
                                            lambda: AG.run_in_process(plans, xb_flat, outs)])
    _check_runs(plans, results, growth)
    _check_exact_c(ce, ops.ref_allgather_fp8(xe, chunk)[1], chunk, K, eq, es)
    del ce
    want, want_rec = ops.ref_allgather_fp8(xb_flat, chunk)
    _check_gather(plans, outs, want, want_rec)
    # the landing region now holds the bench inputs' records, which the second run_gemm multiplied
    _same_on_every_rank(cb, "C")
    c0 = torch.zeros_like(cb[0])
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_chunk_records(plans[0].records(), M, K, chunk), bb, c0, cta_group=1).ok
    assert torch.equal(cb[0].view(torch.int16), c0.view(torch.int16)), "C differs from K7 without an order"
    rows_per_rec = chunk // K
    pick = torch.cat([torch.arange(r * rows_per_rec, (r + 1) * rows_per_rec)
                      for s in range(N) for r in (s * R, s * R + R - 1)]).cuda()
    aq, as_ = record_fields(want_rec, chunk, K)
    _check_against_reference(cb[0][pick], aq[pick].contiguous(), as_[pick].contiguous(), bq, bs)


# ------------------------------------------------------------------ 4. the top of the range through the gather
def _records_equal_up_to_nan_sign(got, want, chunk, label):
    """K3 records byte for byte, except that a NaN code (0x7F / 0xFF) matches a NaN code of either sign."""
    g, w = got.reshape(-1, P.record_bytes(chunk)), want.reshape(-1, P.record_bytes(chunk))
    assert torch.equal(g[:, chunk:], w[:, chunk:]), f"{label}: scale bytes differ"
    gq, wq = g[:, :chunk], w[:, :chunk]
    nan = (wq & 0x7F) == 0x7F
    assert torch.equal((gq & 0x7F) == 0x7F, nan), f"{label}: NaN codes at other positions"
    assert torch.equal(gq[~nan], wq[~nan]), f"{label}: {int((gq[~nan] != wq[~nan]).sum())} codes differ"


@pytest.mark.parametrize("N", [3, 8])
def test_allgather_edge_payload(ctx, N):
    """``run`` on the edge payload of test_ring_fp8_references.py (NaN, +-Inf, blocks that overflow, bf16 max, bf16
    subnormals, zeros at the first and last block of records and tiles): ``out`` and the records equal the reference
    and the independent model up to the sign of NaN."""
    xs_cpu, _ = edge_payload(N, seed=8800 + N)
    n = xs_cpu[0].numel()
    _sm_budget(N, 0, WAITERS)
    plans = _plans(ctx, N, CHUNK, n // CHUNK)
    xs = [x.cuda() for x in xs_cpu]
    outs = [_bf16_full((N * n,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [lambda: AG.run_in_process(plans, xs, outs)])
    _check_runs(plans, results, growth)
    want, want_rec = ops.ref_allgather_fp8(xs_cpu, CHUNK)
    bits, codes, sc = model_allgather(xs_cpu, CHUNK)
    assert_bits_equal(want, bits, "the reference against the model")
    want_bits = want.view(torch.int16).numpy().astype(np.uint16)
    for q, p in enumerate(plans):
        got = outs[q].cpu()
        assert_bits_equal(got, want_bits, f"rank {q}'s out")
        assert_bits_equal(got, bits, f"rank {q}'s out against the model")
        _records_equal_up_to_nan_sign(p.records().cpu(), want_rec, CHUNK, f"rank {q}'s records")
    model_rec = torch.zeros_like(want_rec).reshape(-1, P.record_bytes(CHUNK))
    model_rec[:, :CHUNK] = torch.from_numpy(codes.reshape(-1, CHUNK))
    model_rec[:, CHUNK:CHUNK + CHUNK // 32] = torch.from_numpy(sc.reshape(-1, CHUNK // 32))
    _records_equal_up_to_nan_sign(plans[0].records().cpu(), model_rec, CHUNK, "rank 0's records against the model")
    assert bool(torch.isnan(outs[0]).any()), "no NaN travelled the gather"


TOP_BLOCK = 5


def top_exact_shard(rows, K, g):
    """``exact_shard`` with its block TOP_BLOCK of every row at 2^120: scale byte 241, still without error in K3."""
    x = exact_shard(rows, K, g)
    x[:, 32 * TOP_BLOCK:32 * TOP_BLOCK + 32] = exact_shard(rows, 32, g, 120, 120)
    return x


@pytest.mark.parametrize("N", [3, 8])
def test_allgather_gemm_top_of_the_range(ctx, N):
    """``run_gemm`` on shards of ``_edge_matrix`` (NaN, +-Inf, the top of the range with scale bytes 246 and 247,
    2^-67, bf16 subnormals, zero blocks), against ordinary weights and then weights scaled by 2^60, whose scale-byte
    sums pass 381 and take K7's second scaling path: C identical on every rank, finite where the reference is, and the
    reference's Inf and NaN elsewhere.  Then an exact case past the fp32 scale range: exact shards whose block
    ``TOP_BLOCK`` sits at 2^120 (scale byte 241) against exact weights whose block ``TOP_BLOCK`` has scale byte 150, so
    its scale product is 2^137.  Where that block's partial is nonzero C is +-Inf; where it is zero the output is the
    finite sum of the other blocks, bit for bit (an fp32 product of the two scales would make it NaN)."""
    K, rows_per_rec, R, Nb = 512, 128, 2, 200
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    _sm_budget(N, 0, WAITERS)
    plans = _plans(ctx, N, chunk, R)
    g = torch.Generator().manual_seed(8900 + N)
    xa_cpu = [_edge_matrix(rows, K, g, finite_only=False) for _ in range(N)]
    xa = [x.cuda() for x in xa_cpu]
    scales = (1.0, 2.0 ** 60)
    bw = [MX.quantize_mx((torch.randn(Nb, K, generator=g) * s).to(torch.bfloat16).cuda()) for s in scales]
    ob = [MX.MxOperand.from_tensors(q, s) for q, s in bw]
    cs = [[_bf16_full((N * rows, Nb)) for _ in range(N)] for _ in scales]
    xt = [top_exact_shard(rows, K, g).cuda() for _ in range(N)]
    tq, ts = _mx_exact_operand(Nb, K, g)
    ts[:, TOP_BLOCK] = 150
    ct = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    results, growth = _session(ctx, plans, [lambda: AG.run_gemm_in_process(plans, xt, [MX.MxOperand.from_tensors(tq, ts)] * N, ct),
                                            lambda: AG.run_gemm_in_process(plans, xa, [ob[0]] * N, cs[0]),
                                            lambda: AG.run_gemm_in_process(plans, xa, [ob[1]] * N, cs[1])])
    _check_runs(plans, results, growth)
    rec_t = ops.ref_allgather_fp8(xt, chunk)[1]
    tq_a, ts_a = record_fields(rec_t, chunk, K)
    assert int(ts_a[:, TOP_BLOCK].min()) == 241 and int(ts_a[:, TOP_BLOCK].max()) == 241
    ref_t = MX.ref_gemm_mxfp8(tq_a.contiguous(), ts_a.contiguous(), tq, ts)
    fin = torch.isfinite(ref_t)
    assert fin.any() and torch.isinf(ref_t).any() and not torch.isnan(ref_t).any(), "the exact top case is vacuous"
    _check_exact_c(ct, rec_t, chunk, K, tq, ts)
    want_rec = ops.ref_allgather_fp8(xa_cpu, chunk)[1]
    for q, p in enumerate(plans):
        _records_equal_up_to_nan_sign(p.records().cpu(), want_rec, chunk, f"rank {q}'s records")
    aq, as_ = record_fields(want_rec.cuda(), chunk, K)
    aq, as_ = aq.contiguous(), as_.contiguous()
    assert {0, 246, 247}.issubset(set(as_.unique().tolist()))
    for (bq, bs), c, s in zip(bw, cs, scales):
        _same_on_every_rank(c, "C")
        n_inf, n_nan = _check_against_reference(c[0], aq, as_, bq, bs)
        assert n_nan > 0, "no NaN block reached the product"
        if s > 1:
            assert n_inf > 0, "no output overflows"
            assert int(as_.max()) + int(bs.max()) > 381, "no stage leaves the first scaling path"


# ------------------------------------------------------------------ 5. repeated runs in one engine session
def test_allgather_repeated_runs_one_engine_session(ctx):
    """N = 4, grid 3, signal_every 3, with the engine started once: ``run`` into ``out``, ``run_gemm``, ``run`` in
    place, ``run_gemm`` with other weights.  The unpacks' and the GEMM's counters share the scratch slot's bottom with
    each other and its top with the relay's; the four runs' receives pass the receive queue's depth, so its index
    wraps."""
    N, K, rows_per_rec, R, Nb, grid = 4, 64, 128, 5, 200, 3
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    n = rows * K
    _sm_budget(N, grid, WAITERS)
    plans = _plans(ctx, N, chunk, R, grid, signal_every=3)
    assert 4 * plans[0].n_recv > plans[0].recv_qp.rq_depth
    g = torch.Generator().manual_seed(9000)
    x1, x2, x3, x4 = ([exact_shard(rows, K, g).cuda() for _ in range(N)] for _ in range(4))
    b2, b4 = (_mx_exact_operand(Nb, K, g) for _ in range(2))
    outs1 = [_bf16_full((N * n,)) for _ in range(N)]
    outs3 = [_bf16_full((N * n,)) for _ in range(N)]
    for q in range(N):
        outs3[q][q * n:(q + 1) * n].copy_(x3[q].reshape(-1))
    c2 = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    c4 = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    x1f = [x.reshape(-1) for x in x1]
    x3f = [outs3[q][q * n:(q + 1) * n] for q in range(N)]
    ob2, ob4 = MX.MxOperand.from_tensors(*b2), MX.MxOperand.from_tensors(*b4)
    want1, want3 = ops.ref_allgather_fp8(x1f, chunk)[0], ops.ref_allgather_fp8([x.reshape(-1) for x in x3], chunk)[0]
    results, growth = _session(ctx, plans, [lambda: AG.run_in_process(plans, x1f, outs1),
                                            lambda: AG.run_gemm_in_process(plans, x2, [ob2] * N, c2),
                                            lambda: AG.run_in_process(plans, x3f, outs3),
                                            lambda: AG.run_gemm_in_process(plans, x4, [ob4] * N, c4)])
    _check_runs(plans, results, growth)
    for q in range(N):
        assert torch.equal(outs1[q].view(torch.int16), want1.view(torch.int16)), f"rank {q}'s first out"
        assert torch.equal(outs3[q].view(torch.int16), want3.view(torch.int16)), f"rank {q}'s in-place out"
    _check_exact_c(c2, ops.ref_allgather_fp8(x2, chunk)[1], chunk, K, *b2)
    rec4 = ops.ref_allgather_fp8(x4, chunk)[1]
    _check_exact_c(c4, rec4, chunk, K, *b4)
    for q, p in enumerate(plans):
        assert torch.equal(p.records(), rec4), f"rank {q}'s gathered records"


# ------------------------------------------------------------------ 6. a rank that never contributes to the GEMM
def test_allgather_gemm_rank_that_never_contributes(ctx):
    """Rank 1 posts its receives but never runs its main and compute streams: the ordered K7 of the ranks that wait
    for its shard gives up in its loaders and ends TIMEOUT, no wait is longer than timeout_ms and the run ends within
    2N x timeout_ms.  The next ``run_gemm``, with all ranks, equals the exact reference."""
    N, K, rows_per_rec, R, Nb, tmo = 3, 64, 128, 2, 136, 300
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    _sm_budget(N, 0, WAITERS)
    plans = _plans(ctx, N, chunk, R, timeout_ms=tmo)
    g = torch.Generator().manual_seed(9100)
    x1, x2 = ([exact_shard(rows, K, g).cuda() for _ in range(N)] for _ in range(2))
    bq, bs = _mx_exact_operand(Nb, K, g)
    b = MX.MxOperand.from_tensors(bq, bs)
    c1 = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    c2 = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        res = AG.run_gemm_in_process(plans, x1, [b] * N, c1, skip={1})
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    for q in (0, 2):
        assert res[q].status == "TIMEOUT", (q, res[q].status, res[q].failed)
        gemm = [l for l in res[q].launches if l.name == "gemm"]
        assert len(gemm) == 1 and gemm[0].status == "TIMEOUT", (q, gemm)
    for r in res:
        for l in r.launches:
            assert l.status in ("OK", "TIMEOUT"), (r.rank, l)
    assert dt < 2 * N * tmo / 1000 + 1.0, f"the failed run took {dt:.2f} s"
    for p in plans:
        assert p.send_qp.counters()["n_err"] == 0
    results, growth = _session(ctx, plans, [lambda: AG.run_gemm_in_process(plans, x2, [b] * N, c2)])
    for r in results[0]:
        assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
        assert r.received == r.posted == (N - 1) * R, (r.rank, r.received, r.posted)
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0
    _check_exact_c(c2, ops.ref_allgather_fp8(x2, chunk)[1], chunk, K, bq, bs)


# ------------------------------------------------------------------ 7. the first run of a fresh process
_FIRST_RUN = """
import sys
import torch
sys.path.insert(0, {root!r})
import rocnrdma_b200 as rn
from rocnrdma_b200 import ops
from rocnrdma_b200.parallel import allgather_fp8 as AG
ctx = rn.Context(device=0)
N, R, chunk = {N}, {R}, 8192
plans = [AG.RingAllgatherFp8(ctx, R * chunk, chunk, q, N, timeout_ms=2000) for q in range(N)]
AG.link_in_process(plans)
xs = [torch.randn(R * chunk, device="cuda").to(torch.bfloat16) for _ in range(N)]
outs = [torch.zeros(N * R * chunk, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
torch.cuda.synchronize()
ctx.engine_start(ctas=16, idle_timeout_ms=5000)
try:
    res = AG.run_in_process(plans, xs, outs)
finally:
    ctx.engine_stop()
want = ops.ref_allgather_fp8(xs, chunk)[0]
print("statuses", *[r.status for r in res])
print("exact", all(torch.equal(o.view(torch.int16), want.view(torch.int16)) for o in outs))
ctx.close()
"""


@pytest.mark.parametrize("N,R", [(2, 3), (3, 5)])
def test_allgather_first_run_of_a_fresh_process(N, R):
    """The first run in a new process, with slots whose arrival words start 24 or 40 bytes into the words, so that
    setting them is not torch's vectorised fill.  The plan loads every fill kernel its runs use before the engine
    starts: a kernel's first load waits for the resident engine (DESIGN.md 3.2), which here held the relays of every
    rank after the first until the engine went idle, and the run ended TIMEOUT.  A process of its own, because a
    kernel loaded by any earlier test would hide it."""
    assert any((q * R * 8) % 16 for q in range(N))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", _FIRST_RUN.format(root=root, N=N, R=R)], capture_output=True, text=True,
                       timeout=300, cwd=root)
    assert p.returncode == 0, p.stderr[-3000:]
    assert f"statuses {' '.join(['OK'] * N)}" in p.stdout and "exact True" in p.stdout, p.stdout
