"""GPU tests of the engine's mover: its stall profile (RN_ENGINE_PROFILE=1, Context.engine_mover_profile) and the
visibility of what it writes.  The mover reports a written chunk to its control warp with a CTA-scope mbarrier arrive
and no fence of its own; control's gpu-scope fence carries the bytes to the CQE and to a put-with-signal's atomic
(DESIGN.md 3.1).  The visibility tests check that at bench.py's shape (256 MiB WRITEs, window 8, 32 engine CTAs): a
consumer kernel on another SM compares each message the moment its completion is announced, for device, host-pinned
and peer-GPU destinations.  Every test checks that the engine left cleanly (no fatal fault, no CTA still running)."""
import time

import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W

pytestmark = pytest.mark.gpu

MSG, KSUB, CTAS = 256 << 20, 16384, 32


def _granule(nbytes, ctas, chunk_bytes=512 << 10):
    """The engine's work granule for one WQE (write_resolved's policy)."""
    want = -(-nbytes // (8 * ctas))
    return max(chunk_bytes, -(-want // KSUB) * KSUB)


def _left_cleanly(ctx):
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    return st


def _stream_with_profile(ctx, monkeypatch, profile):
    n = 24
    src = torch.empty(MSG * 4, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(MSG * 4, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=31)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    monkeypatch.setenv("RN_ENGINE_PROFILE", "1" if profile else "0")
    t0 = time.perf_counter_ns()
    ctx.engine_start(ctas=CTAS, idle_timeout_ms=5000)
    try:
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, MSG, iters=n, window=8, slot_stride=MSG, nslots=4, timeout_ms=10000)
    finally:
        ctx.engine_stop()
    wall_ns = time.perf_counter_ns() - t0
    st = _left_cleanly(ctx)
    assert r.ok and r.done == [n], r.status
    assert ops.compare(src, dst) == 0
    return st, wall_ns


def test_mover_profile_accounts_for_every_chunk(ctx, monkeypatch):
    st, wall_ns = _stream_with_profile(ctx, monkeypatch, profile=True)
    rows = ctx.engine_mover_profile()
    assert len(rows) == CTAS
    assert sum(r["chunks"] for r in rows) == st["n_bulk_chunks"] > 0
    for r in rows:
        assert 0 < r["total_ns"] <= wall_ns, (r, wall_ns)
        for k in rn.api.MOVER_PROFILE_FIELDS:
            if k.endswith("_ns"):
                assert r[k] <= r["total_ns"], (k, r)
        assert sum(r[k] for k in rn.api.MOVER_PROFILE_FIELDS if k.endswith("_ns") and k != "total_ns") <= r["total_ns"], r


def test_mover_profile_is_empty_when_off(ctx, monkeypatch):
    _stream_with_profile(ctx, monkeypatch, profile=False)
    assert ctx.engine_mover_profile() == []


def _watch_cq(ctx, qp, src, dst, n, nbytes, src_mr, dst_mr, ctas=CTAS):
    """Post n WRITEs of nbytes (slot k to slot k) while cq_watch checks each one as soon as its CQE is visible."""
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        view, ws = ops.cq_watch(qp.scq, n, dst, src, nbytes, n, nbytes, _granule(nbytes, ctas), timeout_ms=10000,
                                stream=ctx.aux_stream, sync=False)
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, src_mr, dst_mr, nbytes, iters=n, window=8, slot_stride=nbytes, nslots=n,
                            timeout_ms=10000)
        ws.synchronize()
        w = ops.parse_cq_watch(view)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r.ok and r.done == [n], r.status
    assert w["status"] == "OK" and w["seen"] == n and w["error_cqes"] == 0, w
    assert w["mismatches"] == 0, f"{w['mismatches']} 16-byte words read before their WRITE landed"
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_db_order_violations"] == 0 and c["n_wqe"] == n


def test_cq_announces_only_landed_bytes_device(ctx):
    n = 16
    src = torch.empty(n * MSG, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(n * MSG, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=77)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    _watch_cq(ctx, qp, src, dst, n, MSG, ms, md)
    assert ops.compare(src, dst) == 0


def test_cq_announces_only_landed_bytes_host_pinned(ctx):
    n, nbytes = 8, 32 << 20
    src = torch.empty(n * nbytes, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=78)
    dst = torch.zeros(n * nbytes, dtype=torch.uint8).pin_memory()
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    _watch_cq(ctx, qp, src, dst, n, nbytes, ms, md)
    assert torch.equal(src.cpu(), dst)


@pytest.mark.multigpu
def test_cq_announces_only_landed_bytes_peer_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n, nbytes = 8, 64 << 20
    ctx0, ctx1 = rn.Context(0), rn.Context(1)
    try:
        ctx0.enable_peer(1)                                     # also lets the watcher on GPU 0 read GPU 1's buffer
        src = torch.empty(n * nbytes, dtype=torch.uint8, device="cuda:0")
        ops.fill_random(src, seed=79)
        dst = torch.zeros(n * nbytes, dtype=torch.uint8, device="cuda:1")
        ms, md = ctx0.reg_mr(src), ctx0.reg_mr(dst)           # peer HBM: registration maps it over NVLink
        qp = ctx0.loopback_qp(depth=64)
        qp.set_flags(sys_scope=True)
        torch.cuda.synchronize(1)
        _watch_cq(ctx0, qp, src, dst, n, nbytes, ms, md)
        assert torch.equal(src.cpu(), dst.cpu())
    finally:
        ctx0.close()
        ctx1.close()


def test_signal_announces_only_landed_bytes(ctx):
    """Put-with-signal at bench's message size: the receiver compares slot k the moment the signal reaches k + 1."""
    n = 16
    src = torch.empty(n * MSG, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(n * MSG, dtype=torch.uint8, device="cuda:0")
    sig = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    fetch = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    ops.fill_random(src, seed=80)
    ms, md, msig, mf = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(sig), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=CTAS, idle_timeout_ms=5000)
    try:
        wview, wst = ops.signal_wait(ctx, sig, n, timeout_ms=10000, stream=ctx.aux_stream, sync=False, check=(dst, src, MSG, MSG))
        r = ops.put_signal(qp, ms, md, MSG, msig, fetch_mr=mf, iters=n, window=8, slot_stride=MSG, nslots=n, timeout_ms=10000)
        wst.synchronize()
        w = ops.parse_signal_wait(wview)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r.ok and r.done == [n], r.status
    assert w["status"] == "OK" and w["seen"] == n, w
    assert w["mismatches"] == 0, f"{w['mismatches']} 16-byte words read before their WRITE landed"
    assert int(sig.item()) == n and fetch.tolist() == list(range(n))
    assert ops.compare(src, dst) == 0
