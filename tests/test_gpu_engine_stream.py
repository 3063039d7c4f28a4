"""GPU tests of the engine's streaming copy path: the mover keeps one TMA pipeline running over a queue of chunks, so
chunk k + 1 is loading while chunk k's stores are still in flight.  Every test checks the bytes exactly, checks that
completions arrive in order, and checks that the engine left cleanly (no fatal fault, no CTA still running)."""
import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W
from rc_model import BULK_MIN, _chunks

pytestmark = pytest.mark.gpu


def _left_cleanly(ctx):
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    return st


@pytest.mark.parametrize("ctas", [1, 4, 32])
def test_chunk_boundaries_multi_chunk_writes(ctx, ctas):
    """Many multi-chunk WQEs whose last 16 KiB step is short, to distinct destinations, on a QP with small chunks.  On
    one CTA the queue holds chunk k + 1 while chunk k completes, which is the case the streaming mover must get right."""
    chunk_bytes, nbytes, n = 64 << 10, (5 << 20) + 48, 12
    slot = nbytes + 16
    src = torch.empty(n * slot, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(n * slot, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=ctas)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64, chunk_bytes=chunk_bytes)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=3000)
    try:
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, nbytes, iters=n, window=8, slot_stride=slot, nslots=n, timeout_ms=5000)
    finally:
        ctx.engine_stop()
    st = _left_cleanly(ctx)
    assert r.ok and r.done == [n], r.status
    for i in range(n):
        assert torch.equal(src[i * slot:i * slot + nbytes], dst[i * slot:i * slot + nbytes]), f"slot {i}"
        assert int(dst[i * slot + nbytes:(i + 1) * slot].sum()) == 0, f"engine wrote past slot {i}"
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_db_order_violations"] == 0 and c["n_wqe"] == n and c["retire_head"] == n
    chunks = _chunks(nbytes, ctas, chunk_bytes)
    assert len(chunks) > 1
    assert st["n_bulk_chunks"] == n * sum(1 for b in chunks if b >= BULK_MIN)


def test_bulk_and_generic_interleaved(ctx):
    """Unaligned and small WQEs between large aligned ones, on one QP and across two QPs served at the same time."""
    big, n = 3 << 20, 4
    src = torch.empty(32 << 20, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(32 << 20, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=99)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qps = [ctx.loopback_qp(depth=64, mem=W.MEM_HOST_PINNED, chunk_bytes=64 << 10) for _ in range(2)]
    torch.cuda.synchronize()
    # per QP: (src offset, dst offset, bytes), alternating bulk-eligible and generic-only WQEs
    plans = []
    for q in range(2):
        base, plan = q * (16 << 20), []
        for i in range(n):
            off = base + i * (big + (64 << 10))
            plan.append((off, off, big))                                       # aligned, multi-chunk
            plan.append((off + big + 3, off + big + 5, 1000 + 17 * i))         # unaligned, small
        plans.append(plan)
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        for k in range(2 * n):
            for q, qp in enumerate(qps):
                so, do, nb = plans[q][k]
                qp.post_write(ms, md, nb, src_off=so, dst_off=do)
        wcs = [qp.scq.wait(2 * n, timeout_s=10.0) for qp in qps]
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    for q, qp in enumerate(qps):
        assert [w.wqe_counter for w in wcs[q]] == list(range(2 * n)), "completions out of order"
        assert not any(w.is_error for w in wcs[q])
        assert [w.byte_cnt for w in wcs[q]] == [nb for _, _, nb in plans[q]]
        for so, do, nb in plans[q]:
            assert torch.equal(src[so:so + nb], dst[do:do + nb]), (q, so, nb)
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == 2 * n


@pytest.mark.parametrize("ctas", [1, 32])
def test_put_with_signal_under_streaming(ctx, ctas):
    """Large puts cut into many chunks, each followed by FA(+1) on a signal word; the receiver compares slot k with its
    source the moment the signal reaches k + 1.  A chunk counted before its bytes landed shows up as mismatches."""
    nslots, slot = 32, 4 << 20
    src = torch.empty(nslots * slot, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(nslots * slot, dtype=torch.uint8, device="cuda:0")
    sig = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    fetch = torch.zeros(nslots, dtype=torch.int64, device="cuda:0")
    ops.fill_random(src, seed=4243 + ctas)
    ms, md, msig, mf = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(sig), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=256, chunk_bytes=64 << 10)
    assert len(_chunks(slot, ctas, 64 << 10)) >= 8
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=3000)
    try:
        wview, wst = ops.signal_wait(ctx, sig, nslots, timeout_ms=8000, stream=ctx.aux_stream, sync=False,
                                     check=(dst, src, slot, slot))
        r = ops.put_signal(qp, ms, md, slot, msig, fetch_mr=mf, iters=nslots, slot_stride=slot, nslots=nslots, timeout_ms=8000)
        wst.synchronize()
        w = ops.parse_signal_wait(wview)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r.ok and r.done == [nslots], r.status
    assert w["status"] == "OK" and w["seen"] == nslots, w
    assert w["mismatches"] == 0, f"{w['mismatches']} 16-byte words read before their WRITE landed"
    assert int(sig.item()) == nslots and fetch.tolist() == list(range(nslots))
    assert ops.compare(src, dst) == 0


@pytest.mark.parametrize("nbytes", [4096, 64 << 10])
def test_lone_small_write_is_not_held_back(ctx, nbytes):
    """A single bulk WQE with nothing queued behind it: the mover must finish it at once, not wait for more work."""
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(nbytes, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=5)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=16)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, nbytes, iters=1, timeout_ms=2000)
    finally:
        ctx.engine_stop()
    st = _left_cleanly(ctx)
    assert r.ok and r.done == [1], r.status
    assert r.device_ns < 20_000_000, f"lone {nbytes} B write took {r.device_ns / 1e6:.1f} ms (poster timeout 2000 ms)"
    assert torch.equal(src, dst)
    assert st["n_bulk_chunks"] == 1
