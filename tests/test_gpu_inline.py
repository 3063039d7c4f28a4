"""GPU tier: inline work requests through the software HCA (and the mock ConnectX) on an H100 -- host-posted inline
WRITE / WRITE_IMM / SEND / SEND_IMM, device-posted inline puts with and without a signal, the error paths, and a put
into a peer GPU.  Every softhca test also checks that the engine left cleanly (no fatal fault, no CTA still running)."""
import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W

pytestmark = pytest.mark.gpu
H = W.MEM_HOST_PINNED


def _left_cleanly(ctx):
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    return st


def _values(rows, nbytes, seed, dev="cuda:0"):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (rows, nbytes), dtype=torch.uint8, generator=g).to(dev)


def test_host_posted_inline_write_every_length(ctx):
    """Lengths 1..28 at odd destination offsets, one 64-byte cell each; the bytes around every payload stay zero."""
    dst = torch.zeros(28 * 64, dtype=torch.uint8, device="cuda:0")
    md = ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64, mem=H)
    g = torch.Generator().manual_seed(7)
    payloads = {n: torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g) for n in range(1, 29)}
    offs = {n: 64 * (n - 1) + 1 + 2 * (n % 7) for n in payloads}
    want = torch.zeros(28 * 64, dtype=torch.uint8)
    for n, p in payloads.items():
        want[offs[n]:offs[n] + n] = p
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        for n, p in payloads.items():
            qp.post_write_inline(md, p if n % 2 else bytes(p.tolist()), dst_off=offs[n])
        wcs = qp.scq.wait(28)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert [w.status for w in wcs] == ["OK"] * 28
    assert [w.byte_cnt for w in wcs] == list(range(1, 29))
    assert all(w.wqe_opcode == W.OP_RDMA_WRITE and w.opcode == W.CQE_REQ for w in wcs)
    assert torch.equal(dst.cpu(), want)
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == 28 and c["n_bytes"] == sum(range(1, 29))


def test_host_posted_inline_send_send_imm_and_write_imm(ctx):
    rbuf = torch.zeros(3 * 32, dtype=torch.uint8, device="cuda:0")
    wbuf = torch.zeros(16, dtype=torch.uint8, device="cuda:0")
    mr, mw = ctx.reg_mr(rbuf), ctx.reg_mr(wbuf)
    cq_a, cq_b = ctx.create_cq(64, H), ctx.create_cq(64, H)
    qa = ctx.create_qp(cq_a, cq_a, 16, 16, H)
    qb = ctx.create_qp(cq_b, cq_b, 16, 16, H)
    qa.connect(qb)
    s13, s28 = bytes(range(100, 113)), bytes(range(200, 228))
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        for i in range(3):
            qb.post_recv(mr, 32, off=32 * i)
        qa.post_send_inline(s13)
        qa.post_send_inline(s28, imm=0x1234ABCD)
        qa.post_write_inline(mw, b"\x5a" * 5, dst_off=3, imm=0x99)
        ws = cq_a.wait(3)
        wr = cq_b.wait(3)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert [w.status for w in ws] == ["OK"] * 3
    assert [w.wqe_opcode for w in ws] == [W.OP_SEND, W.OP_SEND_IMM, W.OP_RDMA_WRITE_IMM]
    assert [w.opcode for w in wr] == [W.CQE_RESP_SEND, W.CQE_RESP_SEND_IMM, W.CQE_RESP_WR_IMM]
    assert [w.byte_cnt for w in wr[:2]] == [13, 28]
    assert (wr[1].imm, wr[2].imm) == (0x1234ABCD, 0x99)
    got = bytes(rbuf.cpu().tolist())
    assert got[:13] == s13 and got[13:32] == bytes(19)
    assert got[32:60] == s28 and got[60:] == bytes(36)
    assert bytes(wbuf.cpu().tolist()) == bytes(3) + b"\x5a" * 5 + bytes(8)


@pytest.mark.parametrize("nbytes", [8, 28])
def test_device_posted_inline_puts_32_qps(ctx, nbytes):
    nq, iters = 32, 1024
    values = _values(nq * iters, nbytes, seed=nbytes)          # unregistered: read by the poster into registers
    dst = torch.zeros(nq * iters * nbytes, dtype=torch.uint8, device="cuda:0")
    md = ctx.reg_mr(dst)
    qps = [ctx.loopback_qp(depth=64) for _ in range(nq)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.put_inline(qps, values, md, nbytes, iters=iters, nslots=nq * iters, window=16, burst=8, timeout_ms=5000)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r.ok and r.done == [iters] * nq, r.status
    assert torch.equal(dst.view(-1, nbytes), values), "a slot differs from its values row"
    for qp in qps[:4]:
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == iters and c["n_db_order_violations"] == 0, c


def test_device_posted_inline_puts_window_and_burst(ctx):
    n, nbytes = 2048, 8
    values = _values(256, nbytes, seed=3)                      # fewer rows than messages: row m % 256
    dst = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0")
    md = ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=32, idle_timeout_ms=3000)
    try:
        r = ops.put_inline(qp, values, md, nbytes, iters=n, window=16, burst=8, slot_stride=16, nslots=n, timeout_ms=5000)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r.ok and r.done == [n], r.status
    cells = dst.view(n, 16)
    assert torch.equal(cells[:, :nbytes], values.repeat(n // 256, 1))
    assert int(cells[:, nbytes:].sum()) == 0, "an inline put wrote past its payload"


def test_inline_put_with_signal(ctx):
    """p_signal: 256 inline WRITEs of 16 bytes, each followed by FA(+1) on the signal word.  The receiver compares slot k
    with its values row the moment the signal reaches k + 1.  A second run of 28-byte messages, on a second signal
    word, is compared in full once its signal reaches 256."""
    n = 256
    v16, v28 = _values(n, 16, seed=16), _values(n, 28, seed=28)
    d16 = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0")
    d28 = torch.zeros(n * 28, dtype=torch.uint8, device="cuda:0")
    sig = torch.zeros(2, dtype=torch.int64, device="cuda:0")
    fetch = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    m16, m28, msig, mf = ctx.reg_mr(d16), ctx.reg_mr(d28), ctx.reg_mr(sig), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=128)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=32, idle_timeout_ms=3000)
    try:
        wview, wst = ops.signal_wait(ctx, sig, n, timeout_ms=4000, stream=ctx.aux_stream, sync=False, check=(d16, v16, 16, 16))
        r16 = ops.put_inline(qp, v16, m16, 16, iters=n, nslots=n, sig_mr=msig, fetch_mr=mf, window=16, burst=4, timeout_ms=5000)
        wst.synchronize()
        w16 = ops.parse_signal_wait(wview)
        wview, wst = ops.signal_wait(ctx, (sig.data_ptr() + 8, 8), n, timeout_ms=4000, stream=ctx.aux_stream, sync=False)
        r28 = ops.put_inline(qp, v28, m28, 28, iters=n, nslots=n, sig_mr=msig, sig_off=8, fetch_mr=mf, timeout_ms=5000)
        wst.synchronize()
        w28 = ops.parse_signal_wait(wview)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert r16.ok and r16.done == [n] and r28.ok and r28.done == [n], (r16.status, r28.status)
    assert w16["status"] == "OK" and w16["seen"] == n and w16["mismatches"] == 0, w16
    assert w28["status"] == "OK" and w28["seen"] == n, w28
    assert sig.tolist() == [n, n]
    assert fetch.tolist() == list(range(n))                    # the second run's fetched values overwrite the first's
    assert torch.equal(d16.view(n, 16), v16) and torch.equal(d28.view(n, 28), v28)


def test_inline_write_without_remote_write_access(ctx):
    dst = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    md = ctx.reg_mr(dst, access=W.ACC_LOCAL_WRITE)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=2, idle_timeout_ms=3000)
    try:
        qp.post_write_inline(md, b"\x01" * 8)
        qp.post_write_inline(md, b"\x02" * 8, dst_off=16)
        wcs = qp.scq.wait(2)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wcs[0].is_error and wcs[0].status == "REMOTE_ACCESS_ERR"
    assert wcs[1].is_error and wcs[1].status == "WR_FLUSH_ERR"
    assert qp.state == "ERR" and int(dst.sum()) == 0


def test_inline_write_out_of_bounds(ctx):
    dst = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    md = ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=2, idle_timeout_ms=3000)
    try:
        qp.post_write_inline(md, b"\x03" * 28, dst_off=50)     # 14 bytes past the end of the region
        wc = qp.scq.wait(1)[0]
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wc.is_error and wc.status == "REMOTE_ACCESS_ERR"
    assert int(dst.sum()) == 0


def test_inline_write_behind_a_failing_write_is_flushed(ctx):
    """The inline WQE is parsed (possibly in the same batch) before the failing WRITE ahead of it commits; it must still
    complete with WR_FLUSH_ERR and write nothing."""
    src = torch.full((4096,), 9, dtype=torch.uint8, device="cuda:0")
    bad = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    good = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    ms, mbad, mgood = ctx.reg_mr(src), ctx.reg_mr(bad, access=W.ACC_LOCAL_WRITE), ctx.reg_mr(good)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        qp.post_write(ms, mbad, 4096)
        for k in range(4):
            qp.post_write_inline(mgood, bytes([0x40 + k]) * 20, dst_off=k)
        wcs = qp.scq.wait(5)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wcs[0].status == "REMOTE_ACCESS_ERR"
    assert [w.status for w in wcs[1:]] == ["WR_FLUSH_ERR"] * 4
    assert int(good.sum()) == 0 and int(bad.sum()) == 0


def test_device_posted_inline_puts_into_mock_connectx_queues():
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        n, nbytes = 64, 13
        values = _values(n, nbytes, seed=13)
        dst = torch.zeros(n * 16, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        md = vctx.reg_mr(dst)
        qp = vctx.loopback_qp(depth=16)
        assert qp.on_gpu
        r = ops.put_inline(qp, values, md, nbytes, iters=n, slot_stride=16, nslots=n, window=8, burst=4, timeout_ms=5000)
        assert r.ok and r.done == [n], r.status
        cells = dst.view(n, 16)
        assert torch.equal(cells[:, :nbytes], values) and int(cells[:, nbytes:].sum()) == 0
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == n and c["n_bytes"] == n * nbytes and c["n_db_order_violations"] == 0, c
    finally:
        vctx.close()


@pytest.mark.multigpu
def test_inline_put_into_peer_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n, nbytes = 512, 24
    ctx0, ctx1 = rn.Context(0), rn.Context(1)
    try:
        values = _values(n, nbytes, seed=24)
        dst = torch.zeros(n * nbytes, dtype=torch.uint8, device="cuda:1")
        md = ctx0.reg_mr(dst)                                   # peer HBM: registration maps it over NVLink
        qp = ctx0.loopback_qp(depth=64)
        qp.set_flags(sys_scope=True)
        torch.cuda.synchronize(0); torch.cuda.synchronize(1)
        ctx0.engine_start(ctas=16, idle_timeout_ms=3000)
        try:
            r = ops.put_inline(qp, values, md, nbytes, iters=n, nslots=n, window=16, burst=8, timeout_ms=5000)
        finally:
            ctx0.engine_stop()
        _left_cleanly(ctx0)
        assert r.ok and r.done == [n], r.status
        assert torch.equal(dst.view(n, nbytes).to("cuda:0"), values)
    finally:
        ctx0.close()
        ctx1.close()
