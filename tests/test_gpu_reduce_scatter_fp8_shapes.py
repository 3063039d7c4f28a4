"""The fp8 ring reduce-scatter and the GEMM-reduce-scatter on one GPU at the walk geometries where the fused kernel's
raster and gates get hard, with every landed code under every scale byte, at the largest plans the receive queue
allows, at the benchmark's shapes, on the edge payload, at the ends of the fused add's range and over repeated runs of
one engine session.

* `ReduceScatterWalk` (test_reduce_scatter_fp8_schedule.py) mirrors ``rn_k_gemm_reduce_send`` as ``run_gemm`` launches
  it: the grid clamped to the SMs and the tiles, CTA u's tiles u, u + grid, ..., each mapped by ``tile_coords`` with
  the plan's ``group_m`` to a walk position, and each position through ``gemm_ids`` to its step, ids and ``j_out``.
  ``run``'s reduce hops run test_gpu_reduce_schedule.py's `ReduceSchedule` with the addend and P = 1.  Every geometry
  case asserts the facts of both walks it is there for.
* GEMM operands are small integers times a power of two per row of ``a`` and of ``b``: every fp32 partial is exact in
  any order of the adds, and block scales still spread widely.  The reference partials are computed in fp64 and cast
  to fp32, and every rank's ``out`` must equal ``ops.ref_reduce_scatter_fp8`` bit for bit (NaN sign free where NaN is
  expected).  Each rank receives and posts (N-1)R records a run; its send queue grows by those records and one flush
  a ``run_gemm`` (the kernel's last CTA), N-1 a ``run`` (the pack's and those of hops 0..N-3: the last hop only
  writes ``out``).

The rules of test_gpu_ring_fp8.py hold: every wait is bounded by 5 s or less, nothing allocates or synchronises the
device while the engine runs, landing regions start as poison, the guard words behind the arrival words stay zero, and
each case writes out its SM budget (engine CTAs + N x (grid + 1) of 132: the consumer waits beside the grid).
"""
import gc

import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.parallel import reduce_scatter_fp8 as RS
from test_gpu_receive_fusion import _check_arrival_words
from test_gpu_reduce_schedule import SWEEP, ReduceSchedule, _assert_bf16_bits, bf16_rne_bits, decode_fp32, sweep_records
from test_gpu_reduce_scatter_fp8 import _Op, _want
from test_gpu_ring_fp8 import WAIT_MS, _poison
from test_gpu_ring_fp8_shapes import ENGINE_CTAS, REDUCE_FACTS, _edge_band, _sm_budget, _spread_gpu, ring_grid
from test_reduce_scatter_fp8_references import (_records_of, edge_payload_fp32, model_reduce_scatter,
                                                records_equal_up_to_nan_sign)
from test_reduce_scatter_fp8_schedule import WALK_FACTS, ReduceScatterWalk
from test_ring_fp8_references import CHUNK, assert_bits_equal, edge_payload, encode

pytestmark = pytest.mark.gpu

BM = 128
GEMM, RUN = "run_gemm", "run"


@pytest.fixture(autouse=True)
def _release_cached_memory():
    """After each test (and after its context closes): return the caching allocator's free segments to the driver.
    These cases allocate and free gigabytes; left cached, those segments would serve later tests' allocations, and a
    test that needs a fresh segment of its own (test_gpu_revocation.py) would get a piece of an old one instead."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def case_facts(N, K, R, Nb, grid, rank=0):
    """The fused walk's facts on ``rank`` and a reduce hop's at one geometry, as the in-process plans launch them."""
    g = ring_grid(N, grid)
    w = ReduceScatterWalk(N, R, Nb, K, g, rank=rank).facts()
    r = ReduceSchedule(BM * Nb, R, 1, local=True, grid=g, ready=True).facts()
    return {f for f in WALK_FACTS if w[f]}, {f for f in REDUCE_FACTS if r[f]}


# (N, K_l, R, Nb, grid (0: default), signal_every), with the fused walk's and the reduce hop's facts
GEOMETRY_CASES = [
    ((2, 8, 2, 64, 1, 1),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "narrow_n", "one_cta_walks_every_step", "partial_k",
      "ragged_n"},
     {"step_completes_two", "waits_on_a_later_record"}),
    ((2, 200, 3, 320, 2, 3),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step", "panel_shared",
      "partial_k", "ragged_n"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((3, 64, 4, 512, 3, 1),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step", "panel_shared"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((3, 1000, 2, 192, 7, 5),
     {"clamped_grid", "cta_starts_gated", "partial_k", "ragged_n"},
     {"partial_last_step", "record_shared"}),
    ((4, 128, 6, 256, 0, 1),
     {"clamped_grid", "cta_starts_gated"},
     {"partial_last_step", "record_shared"}),
    ((4, 4096, 1, 1088, 5, 1),
     {"cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step", "panel_shared", "ragged_n"},
     {"multi_tile_run", "partial_last_step", "record_shared"}),
    ((5, 96, 1, 64, 20, 3),
     {"clamped_grid", "cta_starts_gated", "narrow_n", "partial_k", "ragged_n"},
     {"partial_last_step"}),
    ((6, 640, 2, 4096, 0, 1),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step", "panel_shared"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((7, 1152, 1, 320, 1, 8),
     {"cta_crosses_steps", "one_cta_walks_every_step", "ragged_n"},
     {"multi_tile_run", "partial_last_step"}),
    ((8, 64, 4, 256, 3, 1),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((8, 4096, 2, 768, 0, 3),
     {"bf16_after_posts", "cta_crosses_steps", "cta_starts_gated", "mid_ring_entry", "panel_shared"},
     {"partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((2, 64, 5, 8192, 0, 1),
     {"bf16_after_posts", "cta_crosses_steps", "mid_ring_entry", "one_cta_walks_every_step", "panel_shared"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
]
GEOMETRY_IDS = [f"N{n}-K{k}-R{r}-Nb{nb}-grid{g or 'default'}-sig{s}" for (n, k, r, nb, g, s), _, _ in GEOMETRY_CASES]


# ------------------------------------------------------------------ operands, running and checking
def exact_operands(N, M, Nb, K, g, e=12):
    """Rank q's ``a`` [M, K] and ``b`` [Nb, K]: integers in [-2, 2] times 2^e_i per row of ``a`` and 2^e_j per row of
    ``b``, e_i and e_j uniform in [-e, e].  A partial is 2^(e_i + e_j) times a sum of at most 4K in magnitude: exact in
    fp32 whatever the order of the adds."""
    def one(rows):
        ints = torch.randint(-2, 3, (rows, K), generator=g).float()
        return (ints * torch.exp2(torch.randint(-e, e + 1, (rows, 1), generator=g).float())).to(torch.bfloat16)
    return [one(M) for _ in range(N)], [one(Nb) for _ in range(N)]


def partials(a, b):
    """Every rank's fp32 partial ``a @ b.T``, flattened: computed in fp64 where ``a`` is (exact for these operands, Inf
    and NaN included), then cast."""
    return [(x.double() @ y.double().T).float().reshape(-1) for x, y in zip(a, b)]


def _plans(ctx, N, R, Nb=None, grid=0, signal_every=1, chunk=None):
    chunk = chunk or BM * Nb
    plans = [RS.RingReduceScatterFp8(ctx, R * chunk, chunk, q, N, grid=grid, timeout_ms=WAIT_MS,
                                     signal_every=signal_every, engine_ctas=ENGINE_CTAS) for q in range(N)]
    RS.link_in_process(plans)
    return plans


def _bf16_full(shape, value=7.0):
    return torch.full(shape, value, dtype=torch.bfloat16, device="cuda")


def _session(ctx, plans, runs):
    """``runs``: (kind, callable that runs every rank once), back to back in one engine session from poisoned landing
    regions.  Returns each run's results and each rank's send-queue WQE growth."""
    for p in plans:
        _poison(p.landing, p.chunk)
    wqe0 = [p.send_qp.counters()["n_wqe"] for p in plans]
    torch.cuda.synchronize()
    results = []
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        for _, run in runs:
            results.append(run())
    finally:
        ctx.engine_stop()
    return results, [p.send_qp.counters()["n_wqe"] - w for p, w in zip(plans, wqe0)]


def _flushes(kind, N):
    """Flushes a run adds to a rank's send queue: ``gemm_reduce_send``'s last CTA posts one; ``run``'s pack and its
    hops 0..N-3 post one each, and hop N-2 writes ``out`` without a queue pair."""
    return 1 if kind == GEMM else N - 1


def _check_runs(plans, results, growth, kinds):
    """Every launch OK, (N-1)R records received and posted a run, the send queue grown by exactly those records and
    the flushes, the words stamped, no guard word written, no work request in error."""
    N, R = plans[0].world, plans[0].R
    for kind, res in zip(kinds, results):
        for r in res:
            assert r.ok, (kind, r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
            assert all(l.status == "OK" for l in r.launches), (kind, r.rank, [(l.name, l.status) for l in r.launches])
            assert r.received == r.posted == (N - 1) * R, (kind, r.rank, r.received, r.posted)
    assert growth == [sum((N - 1) * R + _flushes(k, N) for k in kinds)] * N, growth
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0


def _mismatch(got, want):
    g, w = got.reshape(-1).view(torch.int16), want.reshape(-1).view(torch.int16)
    d = (g != w).nonzero()
    if d.numel() == 0:
        return ""
    i = int(d[0])
    return f"{d.numel()} elements differ, first at {i}: got {got.reshape(-1)[i].item()}, want {want.reshape(-1)[i].item()}"


def _check_outs(outs, want, label):
    """Every rank's ``out`` bit for bit against its shard of the reference."""
    for q, (o, w) in enumerate(zip(outs, want)):
        o, w = o.reshape(-1), w.reshape(-1).to(o.device)
        assert torch.equal(o.view(torch.int16), w.view(torch.int16)), f"{label}: rank {q}: {_mismatch(o, w)}"


def _check_outs_nan(outs, want, label):
    """As ``_check_outs``, with NaN at the same positions and of either sign."""
    for q, (o, w) in enumerate(zip(outs, want)):
        assert_bits_equal(o.reshape(-1).cpu(), w.reshape(-1).cpu().view(torch.int16).numpy().astype(np.uint16),
                          f"{label}: rank {q}")


# ------------------------------------------------------------------ 1. walk geometries
@pytest.mark.parametrize("case,walk_claims,reduce_claims", GEOMETRY_CASES, ids=GEOMETRY_IDS)
def test_reduce_scatter_geometry(ctx, case, walk_claims, reduce_claims):
    """``run_gemm`` on exact operands, then ``run`` on spread bf16 inputs, in one engine session: every rank's ``out``
    against the reference, bit for bit."""
    N, K, R, Nb, grid, sig = case
    assert case_facts(N, K, R, Nb, grid) == (walk_claims, reduce_claims)
    _sm_budget(N, grid)
    M = N * R * BM
    plans = _plans(ctx, N, R, Nb, grid, sig)
    assert plans[0].group_m == next(v for v in (4, 2, 1) if R % v == 0)
    g = torch.Generator().manual_seed(10_000 + 100 * N + R)
    a_cpu, b_cpu = exact_operands(N, M, Nb, K, g)
    a, b = [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    xs = _spread_gpu(N, N * R * BM * Nb, seed=10_500 + 100 * N + R)
    cg = [_bf16_full((M // N, Nb)) for _ in range(N)]
    cx = [_bf16_full((R * BM * Nb,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [(GEMM, lambda: RS.run_gemm_in_process(plans, a, b, cg)),
                                            (RUN, lambda: RS.run_in_process(plans, xs, cx))])
    _check_runs(plans, results, growth, [GEMM, RUN])
    _check_outs(cg, ops.ref_reduce_scatter_fp8(partials(a, b), BM * Nb), "run_gemm")
    _check_outs(cx, ops.ref_reduce_scatter_fp8(xs, BM * Nb), "run")


# ------------------------------------------------------------------ 2. the landed addend at every code under every scale
def test_fused_add_every_code_under_every_scale(ctx):
    """``gemm_reduce_send`` alone on a loopback QP, Nb = 512 so that a panel record is one sweep record: two landed
    sweep records (every e4m3 code under every scale byte, permuted differently), the walk [0, 1], add [0, 1], send
    [0, -1].  Panel 0 leaves as a record, panel 1 as bf16 rows.  The partial is zero in every other block, so the
    smallest decodes reach the sum unchanged, and spread over 2^-40..2^40 in the others.  Both outputs equal
    ``ref_reduce_fp8`` and the independent path (the bit-field decoder, one numpy fp32 add, then the bit-level bf16
    rounding for the rows and the block model's encoder for the record)."""
    Nb, K = 512, 64
    walk, add, send = [0, 1], [0, 1], [0, -1]
    o = _Op(ctx, 2 * BM, Nb, K, walk, add, send, 2, seed=11_000)
    g = torch.Generator().manual_seed(11_001)
    a = torch.randint(-2, 3, (2 * BM, K), generator=g).float()
    a = a * torch.exp2(torch.randint(-20, 21, (2 * BM, 1), generator=g).float())
    eb = torch.exp2(torch.randint(-20, 21, (Nb // 32, 1), generator=g).float()).repeat_interleave(32, 0)
    b = torch.randint(-2, 3, (Nb, K), generator=g).float() * eb
    b[(torch.arange(Nb) // 32) % 2 == 0] = 0
    o.a_cpu, o.b_cpu = a.to(torch.bfloat16), b.to(torch.bfloat16)
    o.a.copy_(o.a_cpu.cuda())
    o.b.copy_(o.b_cpu.cuda())
    o.c = partials([o.a_cpu], [o.b_cpu])[0].reshape(2 * BM, Nb)
    nz = o.c.reshape(-1, 32).abs().amax(1)
    assert bool((nz.reshape(2 * BM, -1)[:, 0::2] == 0).all()) and float(nz.max()) >= 2.0 ** 36
    o.land_cpu = sweep_records(2, seed=11_002)
    assert o.land_cpu.numel() == o.land.numel() == 2 * o.rec
    o.land.copy_(o.land_cpu.cuda())
    o.ready.fill_(1)
    torch.cuda.synchronize()
    r = o.launch(post_only=True)
    assert r.ok and r.records_posted == 1 and r.records_added == 2, r
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    recs, rows = _want(o.c, walk, add, send, o.land_cpu, Nb)
    st, ds, out = o.staging.cpu(), o.dst.cpu(), o.out.cpu().reshape(-1)
    records_equal_up_to_nan_sign(st, recs[0], SWEEP, "staging record against ref_reduce_fp8")
    records_equal_up_to_nan_sign(ds, recs[0], SWEEP, "destination record against ref_reduce_fp8")
    _assert_bf16_bits(out, rows.reshape(-1).view(torch.int16).numpy().astype(np.uint16), "bf16 rows against ref_reduce_fp8")
    d = decode_fp32(o.land_cpu, 2, SWEEP, SWEEP)
    c = o.c.numpy().reshape(2, -1)
    with np.errstate(over="ignore", invalid="ignore"):
        s0, s1 = c[0] + d[0], c[1] + d[1]
    records_equal_up_to_nan_sign(st, _records_of(*encode(s0.reshape(-1, 32)), SWEEP), SWEEP, "record against the model")
    _assert_bf16_bits(out, bf16_rne_bits(s1), "bf16 rows against the independent sum")
    sc = st[SWEEP:].reshape(-1)
    assert bool((sc == 0).any()) and bool(np.isnan(s1).any()) and bool(np.isinf(s1).any())
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 1 + 1, q


# ------------------------------------------------------------------ 3. the largest plans the receive queue allows
@pytest.mark.parametrize("N,R", [(2, 8192), (8, 1170)])
def test_reduce_scatter_largest_legal_plan(ctx, N, R):
    """R = max_records(N) with chunk 8192: the receive queue at 16384 entries.  In one session ``run_gemm`` with
    Nb = 64 (one panel a chunk) and K_l = 24, with group_m 4 at R = 8192 and 2 at R = 1170, then ``run`` on spread
    inputs; every element exact.  SMs: engine 16 + N x (default grid + 1) <= 132."""
    assert R == RS.max_records(N)
    _sm_budget(N, 0)
    Nb, K = 64, 24
    chunk, M = BM * Nb, N * R * BM
    assert chunk == 8192
    plans = _plans(ctx, N, R, Nb)
    assert plans[0].recv_qp.rq_depth == RS.MAX_QUEUE_DEPTH
    assert plans[0].group_m == (4 if N == 2 else 2)
    g = torch.Generator().manual_seed(12_000 + N)
    a_cpu, b_cpu = exact_operands(N, M, Nb, K, g)
    a, b = [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    del a_cpu
    xs = _spread_gpu(N, N * R * chunk, seed=12_100 + N)
    cg = [_bf16_full((M // N, Nb)) for _ in range(N)]
    cx = [_bf16_full((R * chunk,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [(GEMM, lambda: RS.run_gemm_in_process(plans, a, b, cg)),
                                            (RUN, lambda: RS.run_in_process(plans, xs, cx))])
    _check_runs(plans, results, growth, [GEMM, RUN])
    _check_outs(cg, ops.ref_reduce_scatter_fp8(partials(a, b), chunk), "run_gemm")
    _check_outs(cx, ops.ref_reduce_scatter_fp8(xs, chunk), "run")


# ------------------------------------------------------------------ 4. the benchmark's shapes
@pytest.mark.parametrize("N,Nb", [(2, 8192), (4, 4096), (4, 8192), (8, 8192)])
def test_reduce_scatter_at_the_benchmark_shape(ctx, N, Nb):
    """tools/reduce_scatter_bench.py's shapes and inputs: M = 8192, a total K of 8192, integers in [-2, 2], the
    default grid.  ``run_gemm``, then ``run`` over every rank's ``gemm_send`` bf16 C (the bench's unfused path), in
    one session: both against the reference, computed on the GPU, and C against its exact partial."""
    M, Kt = 8192, 8192
    K, R = Kt // N, M // (N * BM)
    _sm_budget(N, 0)
    plans = _plans(ctx, N, R, Nb)
    g = torch.Generator().manual_seed(13_000 + N + Nb)
    a = [torch.randint(-2, 3, (M, K), generator=g).to(torch.bfloat16).cuda() for _ in range(N)]
    b = [torch.randint(-2, 3, (Nb, K), generator=g).to(torch.bfloat16).cuda() for _ in range(N)]
    cs = [torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    for x, y, c in zip(a, b, cs):
        assert ops.gemm_send(ctx, x, y, c).ok
    cs_flat = [c.reshape(-1) for c in cs]
    outs_f = [_bf16_full((M // N, Nb)) for _ in range(N)]
    outs_u = [_bf16_full(((M // N) * Nb,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [(GEMM, lambda: RS.run_gemm_in_process(plans, a, b, outs_f)),
                                            (RUN, lambda: RS.run_in_process(plans, cs_flat, outs_u))])
    _check_runs(plans, results, growth, [GEMM, RUN])
    parts = partials(a, b)
    for q in range(N):
        assert torch.equal(cs_flat[q].view(torch.int16), parts[q].to(torch.bfloat16).view(torch.int16)), f"rank {q}'s C"
    _check_outs(outs_f, ops.ref_reduce_scatter_fp8(parts, BM * Nb), "run_gemm")
    del parts
    _check_outs(outs_u, ops.ref_reduce_scatter_fp8(cs_flat, BM * Nb), "gemm_send + run")


# ------------------------------------------------------------------ 5. the edge payload through run
def test_reference_on_the_gpu_equals_the_reference_on_the_cpu():
    """``ref_reduce_scatter_fp8`` gives the same bits on both devices, on bf16 inputs with the edge band and on fp32
    partials with the fp32 edge payload (NaN sign free)."""
    N = 4
    xs = _edge_band(_spread_gpu(N, N * 2 * CHUNK, seed=14_000), CHUNK, seed=14_001)
    _check_outs_nan(ops.ref_reduce_scatter_fp8(xs, CHUNK), ops.ref_reduce_scatter_fp8([x.cpu() for x in xs], CHUNK), "bf16")
    xf = edge_payload_fp32(N, seed=14_002)
    _check_outs_nan(ops.ref_reduce_scatter_fp8([x.cuda() for x in xf], BM * 64),
                    ops.ref_reduce_scatter_fp8(xf, BM * 64), "fp32")


@pytest.mark.parametrize("N", [3, 8])
def test_reduce_scatter_edge_payload(ctx, N):
    """``run`` on the edge payload of test_ring_fp8_references.py (every kind enters every shard at every hop, at the
    first and last blocks of records and tiles), then on spread inputs with the edge band in the first and last 8
    blocks of every record: every rank against the reference up to the sign of NaN, and the first run also against
    the independent block model."""
    xs_cpu, R = edge_payload(N, seed=15_000 + N)
    _sm_budget(N, 0)
    plans = _plans(ctx, N, R, chunk=CHUNK)
    xs = [x.cuda() for x in xs_cpu]
    xb = _edge_band(_spread_gpu(N, N * R * CHUNK, seed=15_100 + N), CHUNK, seed=15_200 + N)
    o1 = [_bf16_full((R * CHUNK,)) for _ in range(N)]
    o2 = [_bf16_full((R * CHUNK,)) for _ in range(N)]
    results, growth = _session(ctx, plans, [(RUN, lambda: RS.run_in_process(plans, xs, o1)),
                                            (RUN, lambda: RS.run_in_process(plans, xb, o2))])
    _check_runs(plans, results, growth, [RUN, RUN])
    want = ops.ref_reduce_scatter_fp8(xs_cpu, CHUNK)
    _check_outs_nan(o1, want, "edge payload")
    model = model_reduce_scatter(xs_cpu)
    for q in range(N):
        assert_bits_equal(o1[q].cpu(), model[q], f"rank {q} against the model")
    assert any(bool(torch.isnan(o).any()) for o in o1) and any(bool(torch.isinf(o).any()) for o in o1)
    _check_outs_nan(o2, ops.ref_reduce_scatter_fp8(xb, CHUNK), "edge band")


# ------------------------------------------------------------------ 6. the range of the fused add through run_gemm
TOP_E120 = (1.9375, -1.875, 1.75)       # x 2^127: block exponent 120; 1.9375 scales to 248 and saturates to 240


def range_operands(N, M, K, Nb, g):
    """``b``: row j selects column j mod (K - 1) of ``a`` (1 there, 0 elsewhere) and holds 1 in column K - 1, which
    ``a`` keeps 0 but in the Inf rows; so rank q's partial of row i, column j is ``a_q[i, j mod (K - 1)]``, exact.
    Rows of shard s take kind (row mod 128) mod 5 of what rank (s + 1 + d) mod N (hop d) holds:

    0. e120: hop 0 holds TOP_E120 x 2^127 in columns 0..2, small integers elsewhere; later hops add integers x 2^100.
       The sums stay finite with block exponent 120 (scale byte 247), and 248 x 2^120 saturates to 240.
    1. overflow: every hop holds 1.5 x 2^127 (one column -1.5 x 2^127) in columns 0..3: the first fused add
       overflows to +-Inf.
    2. scale0: every hop holds +-(1..3) x 2^-124: amax / 448 <= 2^-127 at every hop, scale byte 0.
    3. cancel: hop 0 holds +-(1..8) / 8, hop 1 the negation, later hops 0: the sum is exactly 0.
    4. spread: integers in [-2, 2] times 2^e, e uniform in [-20, 20] per row.

    Rank 0's row 5 holds +Inf and row 6 -Inf in column K - 1, so +-Inf enter through the tensor cores in every column;
    row 7 holds +Inf there and -Inf in column 0, so its partials are NaN (Inf x 0, and Inf - Inf).  Every finite
    partial is 0 or at least 2^-124 in magnitude."""
    i = torch.arange(M)[:, None]
    k = torch.arange(K)[None, :]
    kind = (i % BM) % 5
    sign = torch.where((i * 5 + k * 3) % 7 < 3, -1.0, 1.0)
    cancel = ((i * 7 + k * 3) % 8 + 1).float() / 8 * sign                       # the same on every rank
    rexp = torch.randint(-20, 21, (M, 1), generator=g).float()
    top = torch.zeros(1, K)
    top[0, :3] = torch.tensor(TOP_E120) * 2.0 ** 127
    ovf = torch.zeros(1, K)
    ovf[0, :4] = torch.tensor([1.5, -1.5, 1.5, 1.5]) * 2.0 ** 127
    a = []
    for q in range(N):
        d = (q - i // (M // N) - 1) % N
        ints = torch.randint(-2, 3, (M, K), generator=g).float()
        small = torch.randint(1, 4, (M, K), generator=g).float() * sign * 2.0 ** -124
        x = torch.where(d == 0, torch.where(k < 3, top, ints), ints * 2.0 ** 100)
        x = torch.where(kind == 1, ovf.expand(M, K), x)
        x = torch.where(kind == 2, small, x)
        x = torch.where(kind == 3, cancel * torch.where(d == 0, 1.0, torch.where(d == 1, -1.0, 0.0)), x)
        x = torch.where(kind == 4, ints * torch.exp2(rexp), x)
        x[:, K - 1] = 0
        if q == 0:
            x[5, K - 1], x[6, K - 1], x[7, K - 1], x[7, 0] = float("inf"), float("-inf"), float("inf"), float("-inf")
        a.append(x.to(torch.bfloat16))
    sel = torch.zeros(Nb, K)
    sel[torch.arange(Nb), torch.arange(Nb) % (K - 1)] = 1
    sel[:, K - 1] = 1
    return a, [sel.to(torch.bfloat16) for _ in range(N)]


def test_reduce_scatter_gemm_range(ctx):
    """``run_gemm`` at N = 3 on ``range_operands``: finite sums in the e = 120 band (with saturation), fused adds that
    overflow to Inf, blocks at scale byte 0, exact cancellation between two ranks and +-Inf and NaN from the tensor
    cores.  Every rank's ``out`` equals the reference of the fp64 partials, NaN at the same positions.  The reference
    partials are IEEE arithmetic (Inf x 0 is NaN); the tensor cores must give the same."""
    N, R, Nb, K = 3, 2, 256, 64
    M = N * R * BM
    _sm_budget(N, 0)
    plans = _plans(ctx, N, R, Nb)
    a_cpu, b_cpu = range_operands(N, M, K, Nb, torch.Generator().manual_seed(16_000))
    parts = partials(a_cpu, b_cpu)
    fin = torch.cat([p[torch.isfinite(p)] for p in parts])
    assert float(fin[fin != 0].abs().min()) >= 2.0 ** -124
    want = ops.ref_reduce_scatter_fp8(parts, BM * Nb)
    out = torch.cat(want).float()
    assert bool(torch.isnan(out).any()) and bool((out == float("inf")).any()) and bool((out == float("-inf")).any())
    assert bool((torch.isfinite(out) & (out.abs() > 1.75 * 2.0 ** 127)).any()), "no finite sum in the e = 120 band"
    assert bool((out == 0).any())
    m = parts[0].numel() // N
    scales = torch.cat([ops.ref_pack_fp8(parts[(s + 1) % N][s * m:(s + 1) * m], BM * Nb)
                        .reshape(-1, ops.record_bytes(BM * Nb))[:, BM * Nb:] for s in range(N)])
    assert bool((scales == 0).any()) and bool((scales == 247).any())
    a, b = [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    outs = [_bf16_full((M // N, Nb)) for _ in range(N)]
    results, growth = _session(ctx, plans, [(GEMM, lambda: RS.run_gemm_in_process(plans, a, b, outs))])
    _check_runs(plans, results, growth, [GEMM])
    _check_outs_nan(outs, want, "run_gemm")


# ------------------------------------------------------------------ 7. repeated runs in one engine session
def test_reduce_scatter_repeated_runs_one_engine_session(ctx):
    """N = 4, R = 4 (group_m 4), Nb = 320, grid 3, signal_every 3, with the engine started once: ``run``,
    ``run_gemm``, ``run``, ``run_gemm``, each on other inputs.  The four runs' receives pass the receive queue's
    depth, so its index wraps, and the reduce hops and the fused kernel share each rank's scratch slot."""
    N, K, R, Nb, grid = 4, 200, 4, 320, 3
    M = N * R * BM
    _sm_budget(N, grid)
    plans = _plans(ctx, N, R, Nb, grid, signal_every=3)
    assert 4 * plans[0].n_recv > plans[0].recv_qp.rq_depth
    g = torch.Generator().manual_seed(17_000)
    ops_ = [exact_operands(N, M, Nb, K, g) for _ in range(2)]
    ab = [([t.cuda() for t in a], [t.cuda() for t in b]) for a, b in ops_]
    xs = [_spread_gpu(N, N * R * BM * Nb, seed=17_100 + i) for i in range(2)]
    cx = [[_bf16_full((R * BM * Nb,)) for _ in range(N)] for _ in range(2)]
    cg = [[_bf16_full((M // N, Nb)) for _ in range(N)] for _ in range(2)]
    runs = [(RUN, lambda: RS.run_in_process(plans, xs[0], cx[0])),
            (GEMM, lambda: RS.run_gemm_in_process(plans, *ab[0], cg[0])),
            (RUN, lambda: RS.run_in_process(plans, xs[1], cx[1])),
            (GEMM, lambda: RS.run_gemm_in_process(plans, *ab[1], cg[1]))]
    results, growth = _session(ctx, plans, runs)
    _check_runs(plans, results, growth, [k for k, _ in runs])
    for i in range(2):
        _check_outs(cx[i], ops.ref_reduce_scatter_fp8(xs[i], BM * Nb), f"run {2 * i}")
        _check_outs(cg[i], ops.ref_reduce_scatter_fp8(partials(*ab[i]), BM * Nb), f"run_gemm {2 * i + 1}")
