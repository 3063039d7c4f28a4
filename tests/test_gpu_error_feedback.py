"""Error feedback on the GPU: K3 and the reduce with a residual, and the fp8 ring with ``error_feedback=True``.

Every launch threads its residual into the next one, and records, delivered records, bf16 output and residual must equal
``ops.ref_pack_fp8`` / ``ref_reduce_fp8`` / ``ref_allreduce_fp8`` with ``residual(s)=`` bit for bit.  The rules of
test_gpu_ring_fp8.py hold: every kernel that waits is resident with what it waits for, every wait is bounded, and
landing buffers start as poison.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import _native as NAT
from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import ring_fp8 as RF
from test_gpu_numerics import _bits_equal, _gen
from test_gpu_ring_fp8 import WAIT_MS, _inputs, _poison
from test_gpu_receive_fusion import _check_arrival_words

pytestmark = pytest.mark.gpu


def _f32_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32).cpu(), b.contiguous().view(torch.int32).cpu())


def _spread(n, seed):
    g = _gen(seed)
    return (torch.randn(n, generator=g) *
            torch.exp2(torch.randint(-20, 21, (n // 32,), generator=g).float()).repeat_interleave(32)).to(torch.bfloat16)


# ------------------------------------------------------------------ K3 and the reduce
@pytest.mark.parametrize("chunk", [8192, 16384], ids=["G1", "G2"])
def test_pack_with_residual_matches_reference_over_three_calls(ctx, chunk):
    """One tile per record (a step of one tile) and two (a step of two); partial and full grids."""
    n = 6 * chunk
    stg = torch.zeros(P.staging_bytes(n, chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(stg)
    res = torch.zeros(n, dtype=torch.float32, device="cuda")
    ref = torch.zeros(n)
    for call, grid in enumerate((0, 1, 5)):
        x = _spread(n, seed=10 + call)
        _poison(stg, chunk)
        ops.pack_fp8_write(ctx, x.cuda(), smr, chunk_elems=chunk, grid=grid, residual=res)
        want, ref = P.ref_pack_fp8(x, chunk, residual=ref)
        assert torch.equal(stg.cpu(), want), f"call {call}: records"
        assert _f32_equal(res, ref), f"call {call}: residual"
    assert bool((ref != 0).any())


def _reduce_case(ctx, n_src, with_local, grid, ready, with_out, chunk=16384, n_rec=3):
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nb, dtype=torch.uint8, device="cuda")
    smr, dmr = ctx.reg_mr(stg), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    words = torch.ones(n_src * n_rec, dtype=torch.int64, device="cuda") if ready else None   # every record has landed
    res = torch.zeros(n, dtype=torch.float32, device="cuda")
    ref = torch.zeros(n)
    y = torch.full((n,), 7.0, dtype=torch.bfloat16, device="cuda") if with_out else None
    torch.cuda.synchronize()
    for call in range(3):
        recs = torch.cat([P.ref_pack_fp8(_spread(n, 100 * call + s), chunk) for s in range(n_src)])
        loc = _spread(n, 100 * call + 50) if with_local else None
        _poison(stg, chunk)
        _poison(dst, chunk)
        torch.cuda.synchronize()
        r = ops.reduce_fp8(ctx, recs.cuda(), n_src, n, chunk, local=None if loc is None else loc.cuda(), out=y,
                           out_mr=smr, qp=qp, dst_mr=dmr, post_only=True, ready=words, grid=grid, timeout_ms=WAIT_MS,
                           residual=res)
        assert r.ok and r.records_posted == n_rec and r.records_reduced == n_rec, r
        ctx.engine_run_oneshot(ctas=8)
        assert ctx.last_engine_fatal == 0
        torch.cuda.synchronize()
        want_y, want_r, ref = P.ref_reduce_fp8(recs, n_src, n, chunk, local=loc, residual=ref)
        assert torch.equal(stg.cpu(), want_r), f"call {call}: records"
        assert torch.equal(dst.cpu(), want_r), f"call {call}: delivered records"
        assert _f32_equal(res, ref), f"call {call}: residual"
        if with_out:
            assert _bits_equal(y.cpu(), want_y), f"call {call}: bf16 out"
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == 3 * (n_rec + 1), c


@pytest.mark.parametrize("ready", [False, True], ids=["no_words", "words"])
@pytest.mark.parametrize("grid", [0, 2], ids=["full_grid", "grid2"])
@pytest.mark.parametrize("n_src,with_local", [(1, False), (1, True), (2, True)], ids=["P1", "P1_addend", "P2_addend"])
def test_reduce_with_residual_matches_reference_over_three_calls(ctx, n_src, with_local, grid, ready):
    """Both EF variants (P = 1 without the addend; P <= 2 with it) at a full and a partial grid, with and without
    arrival words, posting every record; bf16 ``out`` beside the records on the addend cases."""
    _reduce_case(ctx, n_src, with_local, grid, ready, with_out=with_local)


# ------------------------------------------------------------------ the ring
def _ef_ring(ctx, N, chunk, R, signal_every, timeout_ms=WAIT_MS):
    plans = [RF.RingAllreduceFp8(ctx, N * R * chunk, chunk, q, N, timeout_ms=timeout_ms, signal_every=signal_every,
                                 error_feedback=True) for q in range(N)]
    RF.link_in_process(plans)
    return plans


def _ef_run(ctx, plans, xs_cpu, ref_res, in_place):
    """One run from poisoned landing buffers; every output and every residual against the reference.  Returns the
    reference's new residuals."""
    N = len(plans)
    chunk = plans[0].chunk
    xs_dev = [x.cuda() for x in xs_cpu]
    want, ref_res = ops.ref_allreduce_fp8(xs_dev, chunk, residuals=ref_res)
    xs = [x.clone() for x in xs_dev]
    outs = None if in_place else [torch.full_like(x, 7.0) for x in xs]
    for p in plans:
        _poison(p.landing, chunk)
        _poison(p.staging, chunk)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = RF.run_in_process(plans, xs, outs)
    finally:
        ctx.engine_stop()
    for r in res:
        assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
        assert r.received == plans[0].n_ids and r.posted == plans[0].n_ids
    got = xs if in_place else outs
    for q in range(N):
        assert _bits_equal(got[q], want), f"rank {q} differs from the reference"
        assert _f32_equal(plans[q].residual, ref_res[q]), f"rank {q}: residual differs from the reference"
        _check_arrival_words(plans[q].words_full, plans[q].n_ids)
        assert plans[q].send_qp.counters()["n_err"] == 0
    return ref_res, got[0]


@pytest.mark.parametrize("signal_every", [1, 4])
@pytest.mark.parametrize("chunk", [8192, 1 << 20], ids=["8192", "1M"])
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_ef_allreduce_matches_reference_over_three_runs(ctx, N, chunk, signal_every):
    """In place, into ``out``, in place again: each run's outputs and residuals bit-identical to the reference."""
    R = 3 if chunk == 8192 else 1
    plans = _ef_ring(ctx, N, chunk, R, signal_every)
    n = N * R * chunk
    ref_res = [torch.zeros(n, device="cuda") for _ in range(N)]
    for run, in_place in enumerate((True, False, True)):
        ref_res, _ = _ef_run(ctx, plans, _inputs(N, n, seed=1000 * N + 10 * run + signal_every), ref_res, in_place)
    assert any(bool((r != 0).any()) for r in ref_res)


def test_ef_allreduce_removes_the_bias_of_a_fixed_input(ctx):
    """The same inputs for T = 16 runs: the mean output's error against the exact sum is at most 1/8 of the error of
    one run without feedback (which every run would repeat)."""
    N, chunk, R, T = 4, 8192, 1, 16
    n = N * R * chunk
    xs = [_spread(n, seed=700 + q) for q in range(N)]
    exact = np.sum([x.double().numpy() for x in xs], axis=0)
    plain = np.linalg.norm(ops.ref_allreduce_fp8(xs, chunk).double().numpy() - exact)
    plans = _ef_ring(ctx, N, chunk, R, 1)
    ref_res = [torch.zeros(n, device="cuda") for _ in range(N)]
    total = np.zeros(n)
    for t in range(T):
        ref_res, out = _ef_run(ctx, plans, xs, ref_res, in_place=False)
        total += out.double().cpu().numpy()
    err = np.linalg.norm(total / T - exact)
    assert err <= plain / 8, (err, plain)


def test_ef_allreduce_failed_run_then_reset(ctx):
    """Rank 1 never contributes: every rank ends TIMEOUT and the residuals are undefined.  After reset_residual() a
    clean run matches the reference from zero residuals."""
    N, chunk, R, tmo = 3, 8192, 2, 300
    plans = _ef_ring(ctx, N, chunk, R, 1, timeout_ms=tmo)
    n = N * R * chunk
    xs = [x.cuda() for x in _inputs(N, n, seed=77)]
    outs = [torch.zeros_like(x) for x in xs]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = RF.run_in_process(plans, xs, outs, skip={1})
    finally:
        ctx.engine_stop()
    assert all(r.status == "TIMEOUT" for r in res), [(r.rank, r.status) for r in res]
    for p in plans:
        p.reset_residual()
        p.main_stream.synchronize()
        assert not bool(p.residual.any())
    _ef_run(ctx, plans, _inputs(N, n, seed=78), [torch.zeros(n, device="cuda") for _ in range(N)], in_place=False)


def test_ef_residual_checkpoint_round_trip(ctx):
    """``residual`` can be saved after a run and restored before another: restoring it repeats that run exactly."""
    N, chunk, R = 2, 8192, 2
    plans = _ef_ring(ctx, N, chunk, R, 1)
    n = N * R * chunk
    ref_res = [torch.zeros(n, device="cuda") for _ in range(N)]
    ref_res, _ = _ef_run(ctx, plans, _inputs(N, n, seed=5), ref_res, in_place=False)
    saved = [p.residual.clone() for p in plans]
    xs = _inputs(N, n, seed=6)
    _, first = _ef_run(ctx, plans, xs, [r.clone() for r in ref_res], in_place=False)
    for p, s in zip(plans, saved):
        p.residual.copy_(s)
    _, again = _ef_run(ctx, plans, xs, ref_res, in_place=False)
    assert _bits_equal(first, again)


# ------------------------------------------------------------------ rejections
def test_residual_host_rejections(ctx):
    chunk, n = 8192, 2 * 8192
    x = _spread(n, 1).cuda()
    stg = torch.zeros(P.staging_bytes(n, chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(stg)
    recs = P.ref_pack_fp8(_spread(2 * n, 2), chunk).cuda()
    loc = _spread(n, 3).cuda()
    good = torch.zeros(n, dtype=torch.float32, device="cuda")
    big = torch.zeros(n + 8, dtype=torch.float32, device="cuda")
    bad = [
        (torch.zeros(n, dtype=torch.bfloat16, device="cuda"), "float32"),
        (torch.zeros(n + 8, dtype=torch.float32, device="cuda"), "elements"),
        (torch.zeros(n, dtype=torch.float32), "cuda:0"),
        (big[1:n + 1], "aligned"),
        (big[:2 * n:2], "contiguous"),
    ]
    for r, what in bad:
        with pytest.raises(ValueError, match=what):
            ops.pack_fp8_write(ctx, x, smr, chunk_elems=chunk, residual=r)
        with pytest.raises(ValueError, match=what):
            ops.reduce_fp8(ctx, recs, 1, n, chunk, local=loc, out_mr=smr, residual=r)
    y = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="needs out_mr"):
        ops.reduce_fp8(ctx, recs, 1, n, chunk, local=loc, out=y, residual=good)
    with pytest.raises(ValueError, match="n_src=2"):
        ops.reduce_fp8(ctx, recs, 2, n, chunk, out_mr=smr, residual=good)
    # the C entry points refuse a misaligned residual and an unsupported reduce themselves (-22, nothing launched)
    lib = NAT.load()
    mis = good.data_ptr() + 4
    assert lib.rn_k_pack_fp8_write(0, 1, x.data_ptr(), smr.addr, n, chunk, 0, smr.addr, smr.lkey, 0, 0, 0, 1, 0, 0,
                                   0, mis) == -22
    common = (0, 1, recs.data_ptr())
    assert lib.rn_k_reduce_fp8(*common, 1, loc.data_ptr(), 0, smr.addr, n, chunk, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0,
                               mis) == -22
    assert lib.rn_k_reduce_fp8(*common, 1, loc.data_ptr(), y.data_ptr(), 0, n, chunk, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0,
                               0, good.data_ptr()) == -22                      # no records out
    assert lib.rn_k_reduce_fp8(*common, 2, 0, 0, smr.addr, n, chunk, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0,
                               good.data_ptr()) == -22                         # P = 2 without the addend
    plain = RF.RingAllreduceFp8(ctx, 2 * chunk, chunk, 0, 2)
    assert plain.residual is None and not plain.error_feedback
    with pytest.raises(RuntimeError, match="error_feedback=True"):
        plain.reset_residual()
