"""The scatter pack and the fp8 all-to-all (collective and fused with K7) on one GPU, N ranks simulated in one context.

The rules of test_gpu_ring_fp8.py hold: every kernel that waits is resident with what it waits for, every wait is
bounded, nothing allocates or synchronises the device while the engine runs, arrival words are the head of a zeroed
tensor whose guard words must stay zero, and landing regions start as poison before every session, so a record read
before it has landed changes the result.  Shards for the GEMM are test_allgather_fp8_references.py's exact shards, so
every rank's C must equal ``ops.ref_gemm_mxfp8`` of its landed records bit for bit.
"""
import os
import subprocess
import sys
import time

import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import gemm_mx as MX, pack as P
from rocnrdma_b200.parallel import alltoall_fp8 as A2A
from test_allgather_fp8_references import exact_shard, record_fields
from test_gpu_numerics import _mx_exact_operand
from test_gpu_receive_fusion import _check_arrival_words
from test_gpu_ring_fp8 import WAIT_MS, _poison

pytestmark = pytest.mark.gpu

ENGINE_CTAS = 16


def _bf16_full(shape, value=7.0):
    return torch.full(shape, value, dtype=torch.bfloat16, device="cuda")


# ------------------------------------------------------------------ 1. the scatter pack alone
def test_scatter_pack_posts_every_shard_to_its_rank(ctx):
    """Rank 1 of 3, three records per shard, loopback queue pairs: shards 2 and 0 land in slot 1 of their ranks' landing
    regions, shard 1 in the own slot with its three words stamped, and the second result record counts 3 per peer."""
    N, rank, chunk, R = 3, 1, 8192, 3
    rec = P.record_bytes(chunk)
    x = (torch.randn(N * R * chunk, generator=torch.Generator().manual_seed(5)) * 8).to(torch.bfloat16).cuda()
    staging = torch.zeros(N * R * rec, dtype=torch.uint8, device="cuda")
    lands = [torch.zeros(N * R * rec, dtype=torch.uint8, device="cuda") for _ in range(N)]
    words_full = torch.zeros(R + 8, dtype=torch.int64, device="cuda")
    smr, lmrs = ctx.reg_mr(staging), [ctx.reg_mr(t) for t in lands]
    qps = [ctx.loopback_qp(depth=64) if d != rank else None for d in range(N)]
    for d in range(N):
        _poison(lands[d], chunk)
    torch.cuda.synchronize()
    own = lands[rank][rank * R * rec:(rank + 1) * R * rec]
    r, counts = ops.pack_fp8_scatter(ctx, x, rank, N, smr, own, words_full[:R], qps, lmrs, chunk, with_imm=False,
                                     signal_every=2, post_only=True)
    assert r.ok and r.wqes == (N - 1) * R, r
    assert counts == [R, 0, R] + [0] * 5, counts
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    n = R * chunk
    for d in range(N):
        want = ops.ref_pack_fp8(x[d * n:(d + 1) * n].cpu(), chunk)
        assert torch.equal(lands[d][rank * R * rec:(rank + 1) * R * rec].cpu(), want), f"shard {d}"
    _check_arrival_words(words_full, R)
    for d in (0, 2):
        c = qps[d].counters()
        assert c["n_err"] == 0 and c["n_wqe"] == R + 1, c


def test_scatter_pack_and_consumer_refusals(ctx):
    N, chunk = 2, 8192
    rec = P.record_bytes(chunk)
    x = torch.zeros(N * chunk, dtype=torch.bfloat16, device="cuda")
    staging = torch.zeros(N * rec, dtype=torch.uint8, device="cuda")
    land = torch.zeros(N * rec, dtype=torch.uint8, device="cuda")
    words = torch.zeros(1, dtype=torch.int64, device="cuda")
    smr, lmr = ctx.reg_mr(staging), ctx.reg_mr(land)
    qp = ctx.loopback_qp(depth=64)
    own = land[:rec]
    ok = dict(ctx=ctx, x=x, rank=0, world=N, staging_mr=smr, own=own, own_words=words, qps=[None, qp], dst_mrs=[None, lmr],
              chunk_elems=chunk)
    bad = [(dict(residual=torch.zeros(N * chunk, device="cuda")), "no error feedback"),
           (dict(world=9, qps=[qp] * 9, dst_mrs=[lmr] * 9), "2..8"),
           (dict(rank=2), "2..8"),
           (dict(x=x[:8192 * 3 // 2]), "shards"),
           (dict(own=land), "own"),
           (dict(own_words=torch.zeros(2, dtype=torch.int64, device="cuda")), "own_words"),
           (dict(qps=[None, None]), "queue pair"),
           (dict(qps=[qp]), "one entry per rank")]
    for kw, what in bad:
        args = dict(ok, **kw)
        with pytest.raises(ValueError, match=what):
            ops.pack_fp8_scatter(**args)
    a, b = ctx.loopback_qp(depth=16), ctx.loopback_qp(depth=16)
    with pytest.raises(ValueError, match="share one receive CQ"):
        ops.recv_consume_qps([a, b], 1, [1, 0], lmr)
    with pytest.raises(ValueError, match="1..7"):
        ops.recv_consume_qps([a] * 8, 1, [0] * 8, lmr)
    with pytest.raises(ValueError, match="prepost"):
        ops.recv_consume_qps([a], 1, [a.rq_depth + 1], lmr)


# ------------------------------------------------------------------ 2. the all-to-all, N simulated ranks
def _plans(ctx, N, chunk, R, grid=0, signal_every=1, timeout_ms=WAIT_MS):
    plans = [A2A.AllToAllFp8(ctx, R * chunk, chunk, q, N, grid=grid, timeout_ms=timeout_ms, signal_every=signal_every,
                             engine_ctas=ENGINE_CTAS) for q in range(N)]
    A2A.link_in_process(plans)
    return plans


def _session(ctx, plans, runs):
    """``runs`` back to back in one engine session, from poisoned landing regions."""
    for p in plans:
        _poison(p.landing, p.chunk)
    torch.cuda.synchronize()
    results = []
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        for run in runs:
            results.append(run())
    finally:
        ctx.engine_stop()
    return results


def _check_runs(plans, results):
    """Every launch OK, R records posted to every peer and (N-1)R received a run, the words stamped, no guard word
    written, no work request in error."""
    N, R = plans[0].world, plans[0].R
    for res in results:
        for r in res:
            assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
            assert r.received == r.posted == (N - 1) * R, (r.rank, r.received, r.posted)
            assert r.posted_to == [0 if d == r.rank else R for d in range(N)], (r.rank, r.posted_to)
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert all(p.send_qps[d].counters()["n_err"] == 0 for d in range(N) if d != p.rank)


def _check_outs(plans, outs, xs):
    want, want_rec = ops.ref_alltoall_fp8([x.reshape(-1) for x in xs], plans[0].chunk)
    for q, p in enumerate(plans):
        assert torch.equal(outs[q].view(torch.int16), want[q].view(torch.int16)), f"rank {q}'s out differs"
        assert torch.equal(p.records(), want_rec[q]), f"rank {q}'s landed records"


def _check_c(plans, cs, xs, bs, K):
    """Every rank's landed records are the reference's, and its C equals ref_gemm_mxfp8 of them bit for bit."""
    _, want_rec = ops.ref_alltoall_fp8([x.reshape(-1) for x in xs], plans[0].chunk)
    for q, p in enumerate(plans):
        assert torch.equal(p.records(), want_rec[q]), f"rank {q}'s landed records"
        aq, as_ = record_fields(p.records(), p.chunk, K)
        ref = MX.ref_gemm_mxfp8(aq.contiguous(), as_.contiguous(), *bs[q])
        assert torch.equal(cs[q].view(torch.int16), ref.view(torch.int16)), f"rank {q}'s C"


# (N, K, rows per record, R, Nb, grid, signal_every): R = 1, R odd, records of 1, 2 and 4 tiles, small and default grids
GEOMETRIES = [(2, 64, 128, 1, 128, 0, 1), (3, 64, 128, 3, 136, 0, 1), (4, 256, 128, 5, 200, 3, 3),
              (8, 64, 256, 2, 128, 0, 2), (8, 64, 128, 1, 64, 0, 1), (4, 128, 128, 7, 64, 0, 1)]


@pytest.mark.parametrize("case", GEOMETRIES, ids=["-".join(map(str, c)) for c in GEOMETRIES])
def test_alltoall_geometry(ctx, case):
    """``run_gemm`` on exact shards, then ``run`` on other exact shards, in one engine session."""
    N, K, rows_per_rec, R, Nb, grid, sig = case
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    plans = _plans(ctx, N, chunk, R, grid, sig)
    g = torch.Generator().manual_seed(9500 + 10 * N + R)
    xg = [exact_shard(N * rows, K, g).cuda() for _ in range(N)]
    xr = [exact_shard(N * rows, K, g).reshape(-1).cuda() for _ in range(N)]
    bs = [_mx_exact_operand(Nb, K, g) for _ in range(N)]
    cs = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    outs = [_bf16_full((N * rows * K,)) for _ in range(N)]
    results = _session(ctx, plans, [
        lambda: A2A.run_gemm_in_process(plans, xg, [MX.MxOperand.from_tensors(*b) for b in bs], cs),
        lambda: A2A.run_in_process(plans, xr, outs)])
    _check_runs(plans, results)
    _check_outs(plans, outs, xr)
    # run_gemm's landed records were overwritten by run: check its C against the reference of its own inputs
    _, rec_g = ops.ref_alltoall_fp8([x.reshape(-1) for x in xg], chunk)
    for q in range(N):
        aq, as_ = record_fields(rec_g[q].cuda(), chunk, K)
        ref = MX.ref_gemm_mxfp8(aq.contiguous(), as_.contiguous(), *bs[q])
        assert torch.equal(cs[q].view(torch.int16), ref.view(torch.int16)), f"rank {q}'s C"


@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_alltoall_largest_plan(ctx, N):
    """R = max_records(N): the shared receive CQ takes 2(N-1)R entries, up to 16384.  ``run``, then ``run_gemm``."""
    K, rows_per_rec, Nb = 64, 128, 64
    R = A2A.max_records(N)
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    plans = _plans(ctx, N, chunk, R)
    assert plans[0].recv_qp.rcq.depth == A2A._pow2(2 * plans[0].n_recv) == A2A._pow2(2 * (N - 1) * R)
    g = torch.Generator().manual_seed(9600 + N)
    xr = [(torch.randn(N * rows * K, generator=g) * 8).to(torch.bfloat16).cuda() for _ in range(N)]
    xg = [exact_shard(N * rows, K, g).cuda() for _ in range(N)]
    bs = [_mx_exact_operand(Nb, K, g) for _ in range(N)]
    outs = [_bf16_full((N * rows * K,)) for _ in range(N)]
    cs = [_bf16_full((N * rows, Nb)) for _ in range(N)]
    results = _session(ctx, plans, [lambda: A2A.run_in_process(plans, xr, outs)])
    _check_runs(plans, results)
    _check_outs(plans, outs, xr)
    results = _session(ctx, plans, [
        lambda: A2A.run_gemm_in_process(plans, xg, [MX.MxOperand.from_tensors(*b) for b in bs], cs)])
    _check_runs(plans, results)
    _check_c(plans, cs, xg, bs, K)


def test_alltoall_repeated_runs_one_engine_session(ctx):
    """N = 4, grid 3, signal_every 3, the engine started once: ``run``, ``run_gemm``, ``run``, ``run_gemm`` with other
    inputs and weights.  The four runs' receives pass the shared receive CQ's depth, so its index wraps."""
    N, K, rows_per_rec, R, Nb, grid = 4, 64, 128, 3, 72, 3
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    plans = _plans(ctx, N, chunk, R, grid, signal_every=3)
    assert 4 * plans[0].n_recv > plans[0].recv_qp.rcq.depth
    g = torch.Generator().manual_seed(9700)
    x1, x2, x3, x4 = ([exact_shard(N * rows, K, g).cuda() for _ in range(N)] for _ in range(4))
    b2, b4 = ([_mx_exact_operand(Nb, K, g) for _ in range(N)] for _ in range(2))
    o1, o3 = ([_bf16_full((N * rows * K,)) for _ in range(N)] for _ in range(2))
    c2, c4 = ([_bf16_full((N * rows, Nb)) for _ in range(N)] for _ in range(2))
    flat = lambda xs: [x.reshape(-1) for x in xs]  # noqa: E731
    ops_ = lambda bs: [MX.MxOperand.from_tensors(*b) for b in bs]  # noqa: E731
    results = _session(ctx, plans, [lambda: A2A.run_in_process(plans, flat(x1), o1),
                                    lambda: A2A.run_gemm_in_process(plans, x2, ops_(b2), c2),
                                    lambda: A2A.run_in_process(plans, flat(x3), o3),
                                    lambda: A2A.run_gemm_in_process(plans, x4, ops_(b4), c4)])
    _check_runs(plans, results)
    want1, want3 = ops.ref_alltoall_fp8(flat(x1), chunk)[0], ops.ref_alltoall_fp8(flat(x3), chunk)[0]
    for q in range(N):
        assert torch.equal(o1[q].view(torch.int16), want1[q].view(torch.int16)), f"rank {q}'s first out"
        assert torch.equal(o3[q].view(torch.int16), want3[q].view(torch.int16)), f"rank {q}'s third out"
    _, rec2 = ops.ref_alltoall_fp8(flat(x2), chunk)
    for q in range(N):
        aq, as_ = record_fields(rec2[q].cuda(), chunk, K)
        ref = MX.ref_gemm_mxfp8(aq.contiguous(), as_.contiguous(), *b2[q])
        assert torch.equal(c2[q].view(torch.int16), ref.view(torch.int16)), f"rank {q}'s second C"
    _check_c(plans, c4, x4, b4, K)


def test_alltoall_rank_that_never_contributes(ctx):
    """Rank 1 posts its receives but never runs its main and compute streams: the ranks that wait for its shard end
    TIMEOUT, no wait is longer than timeout_ms and the run ends within 2N x timeout_ms.  The next ``run_gemm`` and
    ``run``, with all ranks in the same process, are OK and exact: each rank's receive queue pair from rank 1 still holds
    the R receives the failed run left, and they take rank 1's records."""
    N, K, rows_per_rec, R, Nb, tmo = 3, 64, 128, 2, 136, 300
    chunk, rows = rows_per_rec * K, R * rows_per_rec
    plans = _plans(ctx, N, chunk, R, timeout_ms=tmo)
    g = torch.Generator().manual_seed(9800)
    x1, x2, x3 = ([exact_shard(N * rows, K, g).cuda() for _ in range(N)] for _ in range(3))
    bs = [_mx_exact_operand(Nb, K, g) for _ in range(N)]
    b = [MX.MxOperand.from_tensors(*v) for v in bs]
    c1, c2 = ([_bf16_full((N * rows, Nb)) for _ in range(N)] for _ in range(2))
    outs = [_bf16_full((N * rows * K,)) for _ in range(N)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        res = A2A.run_gemm_in_process(plans, x1, b, c1, skip={1})
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    for q in (0, 2):
        assert res[q].status == "TIMEOUT", (q, res[q].status, res[q].failed)
        assert [l.status for l in res[q].launches if l.name == "gemm"] == ["TIMEOUT"], res[q].launches
        assert plans[q]._backlogs == [0, R, 0] and plans[q]._stale_cqes == 0
    for r in res:
        for l in r.launches:
            assert l.status in ("OK", "TIMEOUT"), (r.rank, l)
    assert dt < 2 * N * tmo / 1000 + 1.0, f"the failed run took {dt:.2f} s"
    results = _session(ctx, plans, [lambda: A2A.run_gemm_in_process(plans, x2, b, c2),
                                    lambda: A2A.run_in_process(plans, [x.reshape(-1) for x in x3], outs)])
    _check_runs(plans, results)
    _check_outs(plans, outs, x3)
    _, rec2 = ops.ref_alltoall_fp8([x.reshape(-1) for x in x2], chunk)
    for q in range(N):
        aq, as_ = record_fields(rec2[q].cuda(), chunk, K)
        ref = MX.ref_gemm_mxfp8(aq.contiguous(), as_.contiguous(), *bs[q])
        assert torch.equal(c2[q].view(torch.int16), ref.view(torch.int16)), f"rank {q}'s C"


def test_alltoall_rejections(ctx):
    with pytest.raises(ValueError, match="SM budget"):
        A2A.link_in_process([A2A.AllToAllFp8(ctx, 8192, 8192, q, 2, grid=58) for q in range(2)])
    A2A.link_in_process([A2A.AllToAllFp8(ctx, 8192, 8192, q, 2, grid=57) for q in range(2)])   # 16 + 2 x 58 fits
    with pytest.raises(ValueError, match="all-to-all plans"):
        A2A.link_in_process([A2A.AllToAllFp8(ctx, 8192, 8192, 0, 2), A2A.AllToAllFp8(ctx, 16384, 8192, 1, 2)])
    plans = _plans(ctx, 2, 8192, 1)
    x = torch.zeros(2 * 8192, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="overlap"):
        plans[0].run(x, x)
    with pytest.raises(ValueError, match="out"):
        plans[0].run(x, torch.zeros(8192, dtype=torch.bfloat16, device="cuda"))
    b = MX.MxOperand.from_tensors(torch.zeros(128, 128, dtype=torch.uint8, device="cuda"),
                                  torch.zeros(128, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="128 \\* K"):
        plans[0].run_gemm(x.view(128, 128), b, torch.zeros(128, 128, dtype=torch.bfloat16, device="cuda"))


# ------------------------------------------------------------------ 3. the first run of a fresh process
_FIRST_RUN = """
import sys
import torch
sys.path.insert(0, {root!r})
import rocnrdma_b200 as rn
from rocnrdma_b200 import ops
from rocnrdma_b200.parallel import alltoall_fp8 as A2A
ctx = rn.Context(device=0)
N, R, chunk = {N}, {R}, 8192
plans = [A2A.AllToAllFp8(ctx, R * chunk, chunk, q, N, timeout_ms=2000) for q in range(N)]
A2A.link_in_process(plans)
xs = [torch.randn(N * R * chunk, device="cuda").to(torch.bfloat16) for _ in range(N)]
outs = [torch.zeros(N * R * chunk, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
torch.cuda.synchronize()
ctx.engine_start(ctas=16, idle_timeout_ms=5000)
try:
    res = A2A.run_in_process(plans, xs, outs)
finally:
    ctx.engine_stop()
want = ops.ref_alltoall_fp8(xs, chunk)[0]
print("statuses", *[r.status for r in res])
print("exact", all(torch.equal(o.view(torch.int16), w.view(torch.int16)) for o, w in zip(outs, want)))
ctx.close()
"""


@pytest.mark.parametrize("N,R", [(2, 3), (3, 5)])
def test_alltoall_first_run_of_a_fresh_process(N, R):
    """The first run in a new process: every kernel a run uses is loaded before the engine starts (a first load waits
    for the resident engine, DESIGN.md 3.2).  A process of its own, because a kernel loaded by an earlier test would
    hide a missing load."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", _FIRST_RUN.format(root=root, N=N, R=R)], capture_output=True, text=True,
                       timeout=300, cwd=root)
    assert p.returncode == 0, p.stderr[-3000:]
    assert f"statuses {' '.join(['OK'] * N)}" in p.stdout and "exact True" in p.stdout, p.stdout
