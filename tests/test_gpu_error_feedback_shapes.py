"""Error feedback on the GPU at every record geometry, at the largest plans and the benchmark's shapes, across every
(e4m3 code, scale byte) pair, at the top of the fp32 range and on fp32-denormal residuals.

Every check is bit-exact against ``ops.ref_pack_fp8`` / ``ref_reduce_fp8`` / ``ref_allreduce_fp8`` with a residual:
records, delivered records, bf16 ``out`` and residuals; NaN is compared without its sign.  Every case threads its
residual through at least 2 calls or runs, so that nonzero residuals are read.

* K3 with a residual posts over a loopback QP with RDMA_WRITE_IMM at 1, 2, 3, 5, 8 and 128 tiles per record (2 tiles
  per step where a record holds an even number, else 1), on grids from 1 to more CTAs than groups.
* Both EF reduce variants (``ReduceSchedule`` with ``ef=True``: one tile per step) at 1, 3, 5 and 128 tiles per record,
  with arrival words, ``imm_base`` and ``signal_every = 3``; each case asserts the facts of its walk.
* The sweep holds every (code, scale byte) pair and is checked against an fp64-decoded numpy sum that uses the
  saturating add of test_error_feedback_references.py.
* The ring runs every geometry of test_gpu_ring_fp8_shapes.py, its largest plans and the benchmark's shape.
* Top of range: finite inputs near bf16 max stay finite over repeated calls and runs (every add of an EF kernel
  saturates at +-FLT_MAX).  Denormals: blocks at exponents -133..-120 leave fp32-denormal residuals, which must match
  bit for bit (no flush to zero).

The rules of test_gpu_ring_fp8.py hold: posting launches run ``post_only`` and a one-shot engine delivers afterwards,
so no kernel waits on another; the ring's kernels are resident with the engine (each case asserts its SM budget), every
wait is bounded by 5 s, nothing allocates or synchronises the device while the engine runs, and landing and staging
buffers start as poison.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import ring_fp8 as RF
from test_error_feedback_references import FLT_MAX, ef_add
from test_gpu_numerics import _gen, _records_equal_up_to_nan_sign
from test_gpu_receive_fusion import _arrival_words, _check_arrival_words
from test_gpu_reduce import CANARY, WAIT_MS, _bf16_equal_up_to_nan, _poison, _source_records
from test_gpu_reduce_schedule import (SWEEP, ReduceSchedule, _assert_bf16_bits, bf16_rne_bits, decode_fp32,
                                      sweep_addend, sweep_records)
from test_gpu_ring_fp8_shapes import ENGINE_CTAS, GEOMETRY_CASES, GEOMETRY_IDS, _edge_band, _run, _sm_budget
from test_ring_fp8_references import BF16_MAX, edge_payload

pytestmark = pytest.mark.gpu

TILE = P.TILE_ELEMS
R_MAX = FLT_MAX - 240 * 2.0 ** 120


def _f32_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32).cpu(), b.contiguous().view(torch.int32).cpu())


def _spread(n, seed, lo=-20, hi=20):
    g = _gen(seed)
    return (torch.randn(n, generator=g) *
            torch.exp2(torch.randint(lo, hi + 1, (n // 32,), generator=g).float()).repeat_interleave(32)).to(torch.bfloat16)


def _small_residual(n, seed):
    g = _gen(seed)
    return torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, -8, (n // 32,), generator=g).float()).repeat_interleave(32)


def _recv_imms(qp):
    wc = qp.rcq.poll(64)
    assert not any(w.is_error for w in wc), wc
    return sorted(w.imm for w in wc)


# ------------------------------------------------------------------ 1. K3 with a residual, posting
# (tiles per record, records, grid (0: default), signal_every)
PACK_CASES = [
    (1, 6, 0, 1),          # G 1, default grid clamped to the 6 tiles
    (2, 5, 1, 3),          # G 2, one CTA walks every group
    (3, 4, 5, 1),          # G 1, records shared by CTAs
    (5, 3, 0, 3),          # G 1
    (8, 2, 64, 1),         # G 2: 8 groups, 16 CTAs after the clamp, half of them idle
    (128, 2, 5, 3),        # G 2, 64 groups per record over 5 CTAs
    (128, 2, 0, 1),        # G 2, the default grid
]
PACK_IDS = [f"tpc{t}-rec{r}-grid{g or 'default'}-sig{s}" for t, r, g, s in PACK_CASES]


def _pack_calls(ctx, xs, chunk, grid=0, signal_every=1, res0=None):
    """K3 with a residual, one call per input in ``xs`` (CPU bf16), each posting every record with RDMA_WRITE_IMM over
    a loopback QP (``post_only``) and delivered by a one-shot engine run afterwards.  Checks every call's records,
    delivered records, immediates and residual against ``ref_pack_fp8``; returns the final residual."""
    n = xs[0].numel()
    n_chunks = n // chunk
    nb = P.staging_bytes(n, chunk)
    stg = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    smr, dmr = ctx.reg_mr(stg[:nb]), ctx.reg_mr(dst[:nb])
    qp = ctx.loopback_qp(depth=64)
    ref = torch.zeros(n) if res0 is None else res0.clone()
    res = ref.cuda()
    for call, x in enumerate(xs):
        want, ref = P.ref_pack_fp8(x, chunk, residual=ref)
        stg.fill_(CANARY)
        dst.fill_(CANARY)
        _poison(stg[:nb], chunk)
        _poison(dst[:nb], chunk)
        for _ in range(n_chunks):
            qp.post_recv(dmr, 0)
        torch.cuda.synchronize()
        r = ops.pack_fp8_write(ctx, x.cuda(), smr, qp=qp, dst_mr=dmr, chunk_elems=chunk, with_imm=True,
                               signal_every=signal_every, grid=grid, post_only=True, timeout_ms=WAIT_MS, residual=res)
        assert r.ok and r.wqes == n_chunks, r
        ctx.engine_run_oneshot(ctas=8)
        assert ctx.last_engine_fatal == 0
        torch.cuda.synchronize()
        _records_equal_up_to_nan_sign(stg[:nb].cpu(), want, chunk)
        _records_equal_up_to_nan_sign(dst[:nb].cpu(), want, chunk)
        assert bool((stg[nb:] == CANARY).all()) and bool((dst[nb:] == CANARY).all()), f"call {call}: stored past the records"
        assert _f32_equal(res, ref), f"call {call}: residual"
        assert _recv_imms(qp) == list(range(n_chunks)), f"call {call}: immediates"
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == len(xs) * (n_chunks + 1), c
    return ref


@pytest.mark.parametrize("case", PACK_CASES, ids=PACK_IDS)
def test_pack_with_residual_posts_every_record(ctx, case):
    tpc, n_rec, grid, sig = case
    chunk = tpc * TILE
    n = chunk * n_rec
    ref = _pack_calls(ctx, [_spread(n, 10 * tpc + c) for c in range(2)], chunk, grid, sig)
    assert bool((ref != 0).any())


# ------------------------------------------------------------------ 2. both EF reduce variants
# (P, addend, tiles per record, records, grid (0: default)) and the facts each case is there for
REDUCE_CASES = [
    ((1, False, 1, 7, 3), {"one_cta"}),
    ((1, False, 3, 2, 1), {"one_cta"}),
    ((1, False, 128, 1, 0), {"shared", "clamped"}),
    ((1, True, 5, 7, 3), {"shared"}),
    ((1, True, 1, 1, 0), {"one_cta", "clamped"}),
    ((1, True, 3, 2, 3), {"shared"}),
    ((2, True, 5, 2, 1), {"one_cta"}),
    ((2, True, 3, 7, 0), {"shared", "clamped"}),
    ((2, True, 128, 2, 3), {"shared"}),
]
SCHEDULE_FACTS = {"shared": "record_shared", "one_cta": "record_owned_by_one_cta"}
REDUCE_IDS = [f"P{p}{'-local' if l else ''}-tpc{t}-rec{r}-grid{g or 'default'}" for (p, l, t, r, g), _ in REDUCE_CASES]


def _reduce_calls(ctx, n_src, local, chunk, n_rec, grid, inputs, imm_base=5, signal_every=3, res0=None):
    """The EF reduce, once per (source records, addend) in ``inputs`` (CPU), with every arrival word set, bf16 ``out``
    and every record posted with WRITE_IMM (immediate ``imm_base + r``, ``post_only``) and delivered by a one-shot
    engine run afterwards.  Checks records, delivered records, bf16 out, immediates and residual against
    ``ref_reduce_fp8``; returns the final residual."""
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    rbuf = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    dbuf = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    y = torch.empty(n + 64, dtype=torch.bfloat16, device="cuda")
    smr, dmr = ctx.reg_mr(rbuf[:nb]), ctx.reg_mr(dbuf[:nb])
    qp = ctx.loopback_qp(depth=64)
    full, ready = _arrival_words(n_src * n_rec)
    ready.fill_(1)
    ref = torch.zeros(n) if res0 is None else res0.clone()
    res = ref.cuda()
    for call, (recs, loc) in enumerate(inputs):
        want_y, want_r, ref = P.ref_reduce_fp8(recs, n_src, n, chunk, local=loc, residual=ref)
        rbuf.fill_(CANARY)
        dbuf.fill_(CANARY)
        _poison(rbuf[:nb], chunk)
        _poison(dbuf[:nb], chunk)
        y.fill_(7.0)
        for _ in range(n_rec):
            qp.post_recv(dmr, 0)
        recs_d = recs.cuda()
        loc_d = None if loc is None else loc.cuda()
        torch.cuda.synchronize()
        r = ops.reduce_fp8(ctx, recs_d, n_src, n, chunk, local=loc_d, out=y[:n], out_mr=smr, qp=qp, dst_mr=dmr,
                           with_imm=True, signal_every=signal_every, post_only=True, ready=ready, grid=grid,
                           timeout_ms=WAIT_MS, imm_base=imm_base, residual=res)
        assert r.ok and r.records_posted == n_rec and r.records_reduced == n_rec, r
        ctx.engine_run_oneshot(ctas=8)
        assert ctx.last_engine_fatal == 0
        torch.cuda.synchronize()
        _records_equal_up_to_nan_sign(rbuf[:nb].cpu(), want_r, chunk)
        _records_equal_up_to_nan_sign(dbuf[:nb].cpu(), want_r, chunk)
        _bf16_equal_up_to_nan(y[:n].cpu(), want_y)
        assert bool((rbuf[nb:] == CANARY).all()) and bool((dbuf[nb:] == CANARY).all()), f"call {call}: stored past"
        assert bool((y[n:] == 7.0).all()), f"call {call}: stored past the bf16 output"
        assert _f32_equal(res, ref), f"call {call}: residual"
        assert _recv_imms(qp) == [imm_base + i for i in range(n_rec)], f"call {call}: immediates"
    _check_arrival_words(full, n_src * n_rec)
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == len(inputs) * (n_rec + 1), c
    return ref


@pytest.mark.parametrize("case,claims", REDUCE_CASES, ids=REDUCE_IDS)
def test_reduce_with_residual_every_geometry(ctx, case, claims):
    n_src, local, tpc, n_rec, grid = case
    chunk = tpc * TILE
    sch = ReduceSchedule(chunk, n_rec, n_src, local, grid, ready=True, ef=True)
    assert sch.G == 1 and sch.pmax == (2 if local else 1)
    f = sch.facts()
    have = {k for k, fact in SCHEDULE_FACTS.items() if f[fact]} | ({"clamped"} if sch.requested > sch.grid else set())
    assert have == claims, (claims, have)
    n = chunk * n_rec
    inputs = [(_source_records(n_src, n, chunk, seed=100 * call + tpc + n_rec, edges=True),
               _spread(n, 50 + call) if local else None) for call in range(2)]
    ref = _reduce_calls(ctx, n_src, local, chunk, n_rec, grid, inputs)
    assert bool((ref != 0).any())


# ------------------------------------------------------------------ 3. every code under every scale byte
@pytest.mark.parametrize("n_src,local", [(1, False), (1, True), (2, True)], ids=["P1", "P1-local", "P2-local"])
def test_reduce_with_residual_every_code_under_every_scale(ctx, n_src, local):
    """All 65536 (e4m3 code, scale byte) pairs in every source, a small random residual: the bf16 out equals an
    fp64-decoded numpy sum with the saturating add, the records and the residual equal ``ref_reduce_fp8``.  Scale bytes
    254 and 255 decode past fp32 max: the sum takes Inf there, and a finite overflow saturates."""
    recs = sweep_records(n_src, seed=700 + 2 * n_src + local)
    loc = sweep_addend(710 + n_src) if local else None
    r0 = _small_residual(SWEEP, 720 + n_src)
    d = decode_fp32(recs, n_src, SWEEP, SWEEP)
    if local:
        v, first = (loc.view(torch.int16).numpy().astype(np.uint16).astype(np.uint32) << 16).view(np.float32), 0
    else:
        v, first = d[0], 1
    for s in range(first, n_src):
        v = ef_add(v, d[s])
    v = ef_add(v, r0.numpy())
    want_y, _, _ = P.ref_reduce_fp8(recs, n_src, SWEEP, SWEEP, local=loc, residual=r0)
    _assert_bf16_bits(want_y, bf16_rne_bits(v), "the reference against the independent sum")
    # the kernel, held to the reference bit for bit: two calls, the second reading the first's residual
    _reduce_calls(ctx, n_src, local, SWEEP, 1, 0, [(recs, loc), (recs, loc)], imm_base=0, signal_every=1, res0=r0)


# ------------------------------------------------------------------ 4/5. the ring
def _ef_plans(ctx, N, chunk, R, grid=0, signal_every=1):
    plans = [RF.RingAllreduceFp8(ctx, N * R * chunk, chunk, q, N, grid=grid, timeout_ms=WAIT_MS,
                                 signal_every=signal_every, engine_ctas=ENGINE_CTAS, error_feedback=True)
             for q in range(N)]
    RF.link_in_process(plans)
    return plans


def _ef_ring_runs(ctx, plans, inputs):
    """One run per entry of ``inputs`` (the N ranks' bf16 tensors on the GPU), back to back in one engine session,
    each into its own outputs.  Every rank holds the same bits, every output equals ``ref_allreduce_fp8(residuals=)``
    (computed on the GPU before the engine starts), every rank posts and receives 2(N-1)R records per run, and each
    rank's residual after the last run equals the reference's."""
    N, R = plans[0].world, plans[0].R
    chunk = plans[0].chunk
    n = N * R * chunk
    ref = [torch.zeros(n, device="cuda") for _ in range(N)]
    runs, wants = [], []
    for xs in inputs:
        want, ref = ops.ref_allreduce_fp8(xs, chunk, residuals=ref)
        wants.append(want)
        runs.append((xs, [torch.full_like(x, 7.0) for x in xs]))
    results, growth = _run(ctx, plans, runs)
    for res in results:
        for r in res:
            assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
            assert r.posted == r.received == 2 * (N - 1) * R, (r.rank, r.posted, r.received)
    assert growth == [len(runs) * (2 * (N - 1) * R + 2 * N - 2)] * N, growth
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0
    for i, ((_, outs), want) in enumerate(zip(runs, wants)):
        first = outs[0].view(torch.int16)
        for q in range(N):
            assert torch.equal(outs[q].view(torch.int16), first), f"run {i}: rank {q} differs from rank 0"
        _bf16_equal_up_to_nan(outs[0], want)
    for q, p in enumerate(plans):
        assert _f32_equal(p.residual, ref[q]), f"rank {q}: residual differs from the reference"
    return [outs for _, outs in runs], ref


def _spread_gpu(N, n, seed, lo=-20, hi=20):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(n, generator=g, device="cuda") *
             torch.exp2(torch.randint(lo, hi + 1, (n // 32,), generator=g, device="cuda").float()).repeat_interleave(32)
             ).to(torch.bfloat16) for _ in range(N)]


@pytest.mark.parametrize("case,unpack_claims,reduce_claims", GEOMETRY_CASES, ids=GEOMETRY_IDS)
def test_ef_ring_geometry(ctx, case, unpack_claims, reduce_claims):
    """The record geometries of test_gpu_ring_fp8_shapes.py, 2 runs each.  The forwarding unpacks walk as there; the
    EF hops take one tile per step (``ReduceSchedule(ef=True)``) where the plain hops take two."""
    N, tpc, R, grid, sig = case
    _sm_budget(N, grid)
    chunk = tpc * TILE
    plans = _ef_plans(ctx, N, chunk, R, grid, sig)
    n = N * R * chunk
    _, ref = _ef_ring_runs(ctx, plans, [_spread_gpu(N, n, seed=8000 + 10 * N + tpc + run) for run in range(2)])
    assert any(bool((r != 0).any()) for r in ref)


@pytest.mark.parametrize("N,R", [(2, 4096), (8, 585)])
def test_ef_ring_largest_legal_plan(ctx, N, R):
    assert R == RF.max_records(N)
    _sm_budget(N, 0)
    chunk = 8192
    plans = _ef_plans(ctx, N, chunk, R)
    _ef_ring_runs(ctx, plans, [_spread_gpu(N, N * R * chunk, seed=8100 + 10 * N + run) for run in range(2)])


@pytest.mark.parametrize("N", [2, 4, 8])
def test_ef_ring_at_the_benchmark_shape(ctx, N):
    """2^26 elements, chunk 2^20, the default grid, spread exponents with the edge band, 2 runs."""
    n, chunk = 1 << 26, 1 << 20
    _sm_budget(N, 0)
    plans = _ef_plans(ctx, N, chunk, n // (N * chunk))
    inputs = [_edge_band(_spread_gpu(N, n, seed=8200 + 10 * N + run), chunk, seed=8300 + 10 * N + run)
              for run in range(2)]
    _ef_ring_runs(ctx, plans, inputs)


def test_ef_reference_on_the_gpu_equals_the_reference_on_the_cpu():
    """Outputs and residuals over 2 runs, on the edge band and near the top of the range."""
    N, chunk = 4, 1 << 16
    n = N * 2 * chunk
    xs = _edge_band(_spread_gpu(N, n, seed=8400, lo=-133, hi=120), chunk, seed=8401)
    xs[0].view(-1, 32)[::5] = BF16_MAX / 2
    xs[1].view(-1, 32)[::5] = BF16_MAX / 3
    xs_cpu = [x.cpu() for x in xs]
    rg = [torch.zeros(n, device="cuda") for _ in range(N)]
    rc = [torch.zeros(n) for _ in range(N)]
    for run in range(2):
        og, rg = ops.ref_allreduce_fp8(xs, chunk, residuals=rg)
        oc, rc = ops.ref_allreduce_fp8(xs_cpu, chunk, residuals=rc)
        _bf16_equal_up_to_nan(og.cpu(), oc)
        for q in range(N):
            assert _f32_equal(rg[q], rc[q]), f"run {run}: residual of rank {q}"


# ------------------------------------------------------------------ 6. top of range and the edge payload
def test_pack_bf16_max_stays_finite_over_calls(ctx):
    """bf16 max packed three times with its own residual: every call decodes to 240 * 2^120 (the second used to
    decode to NaN), the residual stays at most FLT_MAX - 240 * 2^120."""
    chunk = 8192
    x = torch.full((2 * chunk,), BF16_MAX, dtype=torch.bfloat16)
    ref = _pack_calls(ctx, [x, x, x], chunk, grid=1)
    assert float(ref.max()) > 0 and float(ref.abs().max()) <= R_MAX


def test_ef_ring_near_the_top_stays_finite_over_runs(ctx):
    """N = 2: 2.5e38 on rank 0 and 0.8e38 on rank 1, the same every run, 4 runs: every output finite."""
    N, chunk, R = 2, 8192, 2
    _sm_budget(N, 0)
    n = N * R * chunk
    xs = [torch.full((n,), 2.5e38, device="cuda").to(torch.bfloat16),
          torch.full((n,), 0.8e38, device="cuda").to(torch.bfloat16)]
    plans = _ef_plans(ctx, N, chunk, R)
    outs, ref = _ef_ring_runs(ctx, plans, [xs] * 4)
    for o in outs:
        assert bool(torch.isfinite(o[0].float()).all())
    assert all(float(r.abs().max()) <= R_MAX for r in ref)


def test_pack_edge_payload_with_residual(ctx):
    """The edge payload through EF K3 for 2 calls, with residuals that push top-of-range values over fp32 max: the
    residual is +0 at every NaN and Inf input."""
    xs, _ = edge_payload(3, seed=8500, chunk=16384)
    x = xs[0]
    r0 = _small_residual(x.numel(), 8501)
    xf = x.float()
    top = torch.isfinite(xf) & (xf.abs() >= 1e38)
    r0[top] = torch.copysign(torch.tensor(3.0e38), xf[top])
    assert bool(top.any())
    ref = _pack_calls(ctx, [x, xs[1]], 16384, res0=r0)
    assert bool((ref != 0).any())


def test_pack_edge_payload_residual_is_zero_at_non_finite_inputs(ctx):
    xs, _ = edge_payload(2, seed=8510, chunk=16384)
    x = xs[0]
    ref = _pack_calls(ctx, [x, x], 16384)
    bad = ~torch.isfinite(x.float())
    assert bool(bad.any()) and bool((ref[bad].view(torch.int32) == 0).all())


def test_reduce_edge_payload_with_residual(ctx):
    """The edge payload's records through the P = 2 EF variant with its addend, 2 calls."""
    chunk = 16384
    xs, _ = edge_payload(3, seed=8520, chunk=chunk)
    n = xs[0].numel()
    n_rec = n // chunk
    recs = torch.cat([P.ref_pack_fp8(xs[s], chunk) for s in range(2)])
    inputs = [(recs, xs[2]), (recs, xs[2])]
    _reduce_calls(ctx, 2, True, chunk, n_rec, 0, inputs)


@pytest.mark.parametrize("N", [3, 8])
def test_ef_ring_edge_payload(ctx, N):
    """Every edge kind enters every shard at every hop, 2 runs of the same inputs."""
    xs_cpu, R = edge_payload(N, seed=8600 + N)
    chunk = 16384
    _sm_budget(N, 0)
    plans = _ef_plans(ctx, N, chunk, R)
    xs = [x.cuda() for x in xs_cpu]
    _ef_ring_runs(ctx, plans, [xs, xs])


# ------------------------------------------------------------------ 7. fp32-denormal residuals
def _denormal_payload(n, seed):
    """Blocks at exponents -133..-120: under e = -127 their codes are e4m3 subnormals, and what they lose is an fp32
    denormal."""
    return _spread(n, seed, lo=-133, hi=-120)


def _denormals(r):
    a = r.abs()
    return int(((a > 0) & (a < 2.0 ** -126)).sum())


def test_pack_denormal_residuals(ctx):
    chunk = 16384
    n = 4 * chunk
    ref = _pack_calls(ctx, [_denormal_payload(n, 8700 + c) for c in range(2)], chunk, grid=3)
    assert _denormals(ref) > n // 8, "the residuals are not fp32 denormals: the check is vacuous"


@pytest.mark.parametrize("n_src,local", [(1, False), (2, True)], ids=["P1", "P2-local"])
def test_reduce_denormal_residuals(ctx, n_src, local):
    chunk, n_rec = 3 * TILE, 3
    n = chunk * n_rec
    inputs = [(torch.cat([P.ref_pack_fp8(_denormal_payload(n, 8800 + 10 * c + s), chunk) for s in range(n_src)]),
               _denormal_payload(n, 8850 + c) if local else None) for c in range(2)]
    # a denormal residual to start from: P = 1 without the addend re-quantises decoded records, which lose nothing
    g = _gen(8860)
    r0 = torch.randn(n, generator=g) * torch.exp2(torch.randint(-140, -127, (n // 32,), generator=g).float()).repeat_interleave(32)
    assert _denormals(r0) > n // 2
    ref = _reduce_calls(ctx, n_src, local, chunk, n_rec, 3, inputs, res0=r0)
    assert _denormals(ref) > n // 8, "the residuals are not fp32 denormals: the check is vacuous"


def test_ef_ring_denormal_residuals(ctx):
    N, chunk, R = 3, 8192, 2
    _sm_budget(N, 0)
    n = N * R * chunk
    plans = _ef_plans(ctx, N, chunk, R)
    _, ref = _ef_ring_runs(ctx, plans, [[x.cuda() for x in (_denormal_payload(n, 8900 + 10 * run + q) for q in range(N))]
                                        for run in range(2)])
    assert sum(_denormals(r) for r in ref) > n // 8
