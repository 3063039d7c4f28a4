"""GPU tier: two-entry scatter-gather work requests on an H100 -- host-posted gather WRITE / WRITE_IMM / SEND and scatter
READ through the software HCA at entry lengths from 1 byte to 64 MiB, aligned and not (so both the TMA path and the
generic copy run), on 1, 3 and 32 engine CTAs, with guard bands around every destination; an entry in pinned host memory;
the error paths; a fenced scatter READ behind a gather WRITE; device-posted gathers (ops.gather_stream) through the
exclusive poster and the one-call verbs; the mock ConnectX executing GPU-written gathers; and a gather into a peer GPU.
Every softhca test also checks that the engine left cleanly (no fatal fault, no CTA still running)."""
import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W
from rocnrdma_b200.api import MemoryRegion

pytestmark = pytest.mark.gpu
H = W.MEM_HOST_PINNED
GUARD = 4096
MiB = 1 << 20
LENS = [1, 15, 16, 4096, MiB + 7, 64 * MiB]
# every length as entry 0 and as entry 1
PAIRS = [(1, 15), (15, 16), (16, 4096), (4096, 1), (MiB + 7, 16), (16, MiB + 7), (64 * MiB, 4096), (4096, 64 * MiB),
         (MiB + 7, 64 * MiB)]
# (entry 0 offset, entry 1 offset, remote offset): 16-byte aligned, and not
ALIGNS = {"aligned": (16, 32, GUARD), "misaligned": (3, 5, GUARD + 7)}


def _left_cleanly(ctx):
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    return st


def _random(n, seed, dev="cuda:0", pin=False):
    g = torch.Generator(device="cpu").manual_seed(seed)
    t = torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g)
    return t.pin_memory() if pin else t.to(dev)


def _zero_outside(buf, lo, hi):
    return int(buf[:lo].count_nonzero()) == 0 and int(buf[hi:].count_nonzero()) == 0


def _cases():
    return [(n0, n1, name, ALIGNS[name]) for n0, n1 in PAIRS for name in ALIGNS]


@pytest.mark.parametrize("ctas", [1, 3, 32])
@pytest.mark.parametrize("op", ["write", "write_imm", "send"])
def test_host_posted_gathers(ctx, op, ctas):
    """Each case gathers entry 0 of S0 and entry 1 of S1 into its own destination (a receive buffer for SEND), with a
    guard band before and after that must stay zero."""
    cases = _cases()
    top = 64 * MiB + 64
    s0, s1 = _random(top, 1), _random(top, 2)
    dsts = [torch.zeros(r + n0 + n1 + GUARD, dtype=torch.uint8, device="cuda:0") for n0, n1, _, (_, _, r) in cases]
    m0, m1 = ctx.reg_mr(s0), ctx.reg_mr(s1)
    mds = [ctx.reg_mr(d) for d in dsts]
    cq_a, cq_b = ctx.create_cq(256, H), ctx.create_cq(256, H)
    qa = ctx.create_qp(cq_a, cq_a, 64, 64, H)
    qb = ctx.create_qp(cq_b, cq_b, 64, 64, H)
    qa.connect(qb)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        for k, (n0, n1, _, (o0, o1, r)) in enumerate(cases):
            sg = [(m0, o0, n0), (m1, o1, n1)]
            if op == "send":
                qb.post_recv(mds[k], off=r)
                qa.post_send_sg(sg, imm=k if k % 2 else None)
            elif op == "write_imm":
                qb.post_recv(mds[k], 0, off=0)
                qa.post_write_sg(sg, mds[k], dst_off=r, imm=0x100 + k)
            else:
                qa.post_write_sg(sg, mds[k], dst_off=r, signaled=k % 3 != 1 or k == len(cases) - 1)
        nsig = len(cases) if op != "write" else sum(1 for k in range(len(cases)) if k % 3 != 1 or k == len(cases) - 1)
        wcs = cq_a.wait(nsig, timeout_s=20)
        rwcs = cq_b.wait(len(cases), timeout_s=20) if op != "write" else []
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert [w.status for w in wcs] == ["OK"] * nsig
    if op != "write":
        assert [w.byte_cnt for w in wcs] == [n0 + n1 for n0, n1, _, _ in cases]
        assert [w.status for w in rwcs] == ["OK"] * len(cases)
        assert [w.byte_cnt for w in rwcs] == [n0 + n1 for n0, n1, _, _ in cases]
    for k, (n0, n1, name, (o0, o1, r)) in enumerate(cases):
        d = dsts[k]
        assert torch.equal(d[r:r + n0], s0[o0:o0 + n0]), (n0, n1, name, "entry 0")
        assert torch.equal(d[r + n0:r + n0 + n1], s1[o1:o1 + n1]), (n0, n1, name, "entry 1")
        assert _zero_outside(d, r, r + n0 + n1), (n0, n1, name, "guard band")
    c = qa.counters()
    assert c["n_err"] == 0 and c["n_bytes"] == sum(n0 + n1 for n0, n1, _, _ in cases), c


@pytest.mark.parametrize("ctas", [1, 3, 32])
def test_host_posted_scatter_reads(ctx, ctas):
    """Each case reads n0 + n1 remote bytes of S and scatters them into two fresh local buffers."""
    cases = _cases()
    s = _random(128 * MiB + 2 * GUARD, 3)
    locs = [(torch.zeros(o0 + n0 + GUARD, dtype=torch.uint8, device="cuda:0"),
             torch.zeros(o1 + n1 + GUARD, dtype=torch.uint8, device="cuda:0")) for n0, n1, _, (o0, o1, _) in cases]
    ms = ctx.reg_mr(s)
    mls = [(ctx.reg_mr(a), ctx.reg_mr(b)) for a, b in locs]
    qp = ctx.loopback_qp(depth=64, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        for k, (n0, n1, _, (o0, o1, r)) in enumerate(cases):
            qp.post_read_sg([(mls[k][0], o0, n0), (mls[k][1], o1, n1)], ms, remote_off=r)
        wcs = qp.scq.wait(len(cases), timeout_s=20)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert [w.status for w in wcs] == ["OK"] * len(cases)
    assert [w.byte_cnt for w in wcs] == [n0 + n1 for n0, n1, _, _ in cases]
    for k, (n0, n1, name, (o0, o1, r)) in enumerate(cases):
        a, b = locs[k]
        assert torch.equal(a[o0:o0 + n0], s[r:r + n0]), (n0, n1, name, "entry 0")
        assert torch.equal(b[o1:o1 + n1], s[r + n0:r + n0 + n1]), (n0, n1, name, "entry 1")
        assert _zero_outside(a, o0, o0 + n0) and _zero_outside(b, o1, o1 + n1), (n0, n1, name, "guard band")


def test_entry_in_pinned_host_memory(ctx):
    """Entry 1 of a gather WRITE, and of a scatter READ, lives in pinned host memory."""
    n0, n1 = 3 * MiB + 5, 2 * MiB + 16
    s0, h = _random(n0, 4), _random(n1 + 64, 5, pin=True)
    dst = torch.zeros(n0 + n1 + 2 * GUARD, dtype=torch.uint8, device="cuda:0")
    back0 = torch.zeros(n0, dtype=torch.uint8, device="cuda:0")
    back1 = torch.zeros(n1 + 64, dtype=torch.uint8).pin_memory()
    m0, mh, md, mb0, mb1 = ctx.reg_mr(s0), ctx.reg_mr(h), ctx.reg_mr(dst), ctx.reg_mr(back0), ctx.reg_mr(back1)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=5000)
    try:
        qp.post_write_sg([(m0, 0, n0), (mh, 7, n1)], md, dst_off=GUARD)
        qp.post_read_sg([(mb0, 0, n0), (mb1, 32, n1)], md, remote_off=GUARD, fence=True)
        wcs = qp.scq.wait(2, timeout_s=20)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert [w.status for w in wcs] == ["OK", "OK"] and [w.byte_cnt for w in wcs] == [n0 + n1] * 2
    assert torch.equal(dst[GUARD:GUARD + n0], s0) and torch.equal(dst[GUARD + n0:GUARD + n0 + n1].cpu(), h[7:7 + n1])
    assert _zero_outside(dst, GUARD, GUARD + n0 + n1)
    assert torch.equal(back0, s0) and torch.equal(back1[32:32 + n1], h[7:7 + n1])
    assert int(back1[:32].count_nonzero()) == 0 and int(back1[32 + n1:].count_nonzero()) == 0


def test_errors_in_entry_one(ctx):
    """Entry 1 under a key nobody registered: LOCAL_PROT_ERR; a READ into an entry 1 registered without local write:
    LOCAL_ACCESS_ERR.  Each fails its QP and moves nothing."""
    src = _random(8192, 6)
    dst = torch.zeros(16384, dtype=torch.uint8, device="cuda:0")
    ro = torch.zeros(8192, dtype=torch.uint8, device="cuda:0")
    ms, md, mro = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(ro, access=W.ACC_REMOTE_READ)
    bad = MemoryRegion(ctx, ms.addr, ms.length, ms.lkey ^ 0x100, W.ACC_ALL)
    qa, qb = ctx.loopback_qp(depth=16, mem=H), ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        qa.post_write_sg([(ms, 0, 4096), (bad, 0, 4096)], md)
        wa = qa.scq.wait(1)[0]
        qb.post_read_sg([(md, 0, 4096), (mro, 0, 4096)], ms)
        wb = qb.scq.wait(1)[0]
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wa.is_error and wa.status == "LOCAL_PROT_ERR" and qa.state == "ERR"
    assert wb.is_error and wb.status == "LOCAL_ACCESS_ERR" and qb.state == "ERR"
    assert int(dst.count_nonzero()) == 0 and int(ro.count_nonzero()) == 0


@pytest.mark.parametrize("op", ["send", "write_imm"])
def test_total_over_the_message_limit(ctx, op):
    """Two entries that each fit but sum past 2^30: LOCAL_LENGTH_ERR before any key, nothing moved, no receive taken."""
    src = _random(4096, 7)
    dst = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    rbuf = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    ms, md, mr = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(rbuf)
    cq_a, cq_b = ctx.create_cq(64, H), ctx.create_cq(64, H)
    qa = ctx.create_qp(cq_a, cq_a, 16, 16, H)
    qb = ctx.create_qp(cq_b, cq_b, 16, 16, H)
    qa.connect(qb)
    sg = [(ms, 0, (1 << 29) + 8), (ms, 16, 1 << 29)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        qb.post_recv(mr)
        if op == "send":
            qa.post_send_sg(sg)
        else:
            qa.post_write_sg(sg, md, imm=5)
        wc = cq_a.wait(1)[0]
        rest = cq_b.poll(4)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wc.is_error and wc.status == "LOCAL_LENGTH_ERR"
    assert rest == [], "a receive was consumed"
    assert int(dst.count_nonzero()) == 0 and int(rbuf.count_nonzero()) == 0
    assert qa.counters()["n_bytes"] == 0


def test_gather_flushed_behind_a_fault_writes_nothing(ctx):
    src = _random(2 * MiB, 8)
    bad = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    good = torch.zeros(4 * MiB, dtype=torch.uint8, device="cuda:0")
    ms, mbad, mgood = ctx.reg_mr(src), ctx.reg_mr(bad, access=W.ACC_LOCAL_WRITE), ctx.reg_mr(good)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    try:
        qp.post_write(ms, mbad, 4096)
        for k in range(4):
            qp.post_write_sg([(ms, k, MiB + k), (ms, MiB, 4096 + 3 * k)], mgood, dst_off=k * MiB // 2)
        qp.post_read_sg([(mgood, 0, 4096), (mgood, 8192, MiB)], ms)
        wcs = qp.scq.wait(6)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert wcs[0].status == "REMOTE_ACCESS_ERR"
    assert [w.status for w in wcs[1:]] == ["WR_FLUSH_ERR"] * 5
    assert int(good.count_nonzero()) == 0 and int(bad.count_nonzero()) == 0


@pytest.mark.parametrize("ctas", [3, 32])
def test_fenced_scatter_read_after_gather_write(ctx, ctas):
    """A gather WRITE of 2 x 4 MiB to R, then, under the same doorbells, a fenced scatter READ of R into two other
    buffers cut at a different point: the READ returns the written bytes.  Twenty rounds over fresh contents."""
    n0, n1, cut = 4 * MiB, 4 * MiB + 48, 3 * MiB + 16
    rounds = 20
    s0 = [_random(n0, 100 + i) for i in range(rounds)]
    s1 = [_random(n1, 200 + i) for i in range(rounds)]
    r = torch.zeros(n0 + n1, dtype=torch.uint8, device="cuda:0")
    backs = [(torch.zeros(cut, dtype=torch.uint8, device="cuda:0"), torch.zeros(n0 + n1 - cut, dtype=torch.uint8, device="cuda:0"))
             for _ in range(rounds)]
    m0, m1 = [ctx.reg_mr(t) for t in s0], [ctx.reg_mr(t) for t in s1]
    mr = ctx.reg_mr(r)
    mbs = [(ctx.reg_mr(x), ctx.reg_mr(y)) for x, y in backs]
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        statuses = []
        for i in range(rounds):
            qp.post_write_sg([(m0[i], 0, n0), (m1[i], 0, n1)], mr, signaled=False)
            qp.post_read_sg([(mbs[i][0], 0, cut), (mbs[i][1], 0, n0 + n1 - cut)], mr, fence=True)
            statuses.append(qp.scq.wait(1, timeout_s=10)[0].status)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert statuses == ["OK"] * rounds
    bad = [i for i in range(rounds) if not torch.equal(torch.cat(backs[i]), torch.cat([s0[i], s1[i]]))]
    assert bad == [], "a fenced READ returned bytes the WRITE before it had not written yet"


@pytest.mark.parametrize("via", ["poster", "one_call"])
@pytest.mark.parametrize("op", ["write", "read"])
def test_device_posted_gathers_32_qps(ctx, op, via):
    """32 QPs x 1,024 two-entry messages of 4 KiB + 48 cut at 1,040 bytes (entry 1's remote side is 16-byte aligned) and
    at 1,001 (it is not), window 16, bursts of 8; every destination byte compared."""
    nq, iters, nbytes = 32, 1024, 4096 + 48
    for split in (1040, 1001):
        slot = nbytes + 16
        total = nq * iters * slot
        a, b = _random(total, 11 + split), _random(total, 12 + split)
        remote = _random(total, 13 + split) if op == "read" else torch.zeros(total, dtype=torch.uint8, device="cuda:0")
        if op == "read":
            a.zero_(); b.zero_()
        ma, mb, mr = ctx.reg_mr(a), ctx.reg_mr(b), ctx.reg_mr(remote)
        qps = [ctx.loopback_qp(depth=64) for _ in range(nq)]
        torch.cuda.synchronize()
        ctx.engine_start(ctas=16, idle_timeout_ms=3000)
        try:
            res = ops.gather_stream(qps, W.OP_RDMA_WRITE if op == "write" else W.OP_RDMA_READ, ma, mb, mr, nbytes, split,
                                    iters=iters, window=16, burst=8, stride=iters * slot, slot_stride=slot, nslots=iters,
                                    via=via, timeout_ms=5000)
        finally:
            ctx.engine_stop()
        _left_cleanly(ctx)
        assert res.ok and res.done == [iters] * nq, (split, res.status)
        A, B, R = a.view(-1, slot), b.view(-1, slot), remote.view(-1, slot)
        assert torch.equal(R[:, :split], A[:, :split]), split
        assert torch.equal(R[:, split:nbytes], B[:, :nbytes - split]), split
        if op == "write":
            assert int(R[:, nbytes:].count_nonzero()) == 0, "a gather wrote past its message"
        else:
            assert int(A[:, split:].count_nonzero()) == 0 and int(B[:, nbytes - split:].count_nonzero()) == 0, \
                "a scatter wrote past its entry"
        for qp in qps[:4]:
            c = qp.counters()
            assert c["n_err"] == 0 and c["n_wqe"] == iters and c["n_bytes"] == iters * nbytes, c
        del qps


@pytest.mark.parametrize("via", ["poster", "one_call"])
def test_device_posted_gather_sends(ctx, via):
    n, nbytes, split = 256, 3000, 1111
    a, b = _random(n * 4096, 21), _random(n * 4096, 22)
    rbuf = torch.zeros(n * 4096, dtype=torch.uint8, device="cuda:0")
    ma, mb, mr = ctx.reg_mr(a), ctx.reg_mr(b), ctx.reg_mr(rbuf)
    cq_a, cq_b = ctx.create_cq(512), ctx.create_cq(512, H)
    qa = ctx.create_qp(cq_a, cq_a, 64, 512)
    qb = ctx.create_qp(cq_b, cq_b, 64, 512, H)
    qa.connect(qb)
    for i in range(n):
        qb.post_recv(mr, 4096, off=i * 4096)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    try:
        res = ops.gather_stream(qa, W.OP_SEND, ma, mb, None, nbytes, split, iters=n, window=16, burst=8, slot_stride=4096,
                                nslots=n, via=via, timeout_ms=5000)
        rw = cq_b.wait(n, timeout_s=10)
    finally:
        ctx.engine_stop()
    _left_cleanly(ctx)
    assert res.ok and res.done == [n], res.status
    assert [w.byte_cnt for w in rw] == [nbytes] * n and all(not w.is_error for w in rw)
    A, B, R = a.view(n, 4096), b.view(n, 4096), rbuf.view(n, 4096)
    assert torch.equal(R[:, :split], A[:, :split]) and torch.equal(R[:, split:nbytes], B[:, :nbytes - split])
    assert int(R[:, nbytes:].count_nonzero()) == 0


def test_mock_connectx_executes_gpu_written_gathers():
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        n, nbytes, split = 64, 200, 77
        a, b = _random(n * 256, 31), _random(n * 256, 32)
        dst = torch.zeros(n * 256, dtype=torch.uint8, device="cuda:0")
        back0, back1 = torch.zeros(n * 256, dtype=torch.uint8, device="cuda:0"), torch.zeros(n * 256, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        ma, mb, md, m0, m1 = vctx.reg_mr(a), vctx.reg_mr(b), vctx.reg_mr(dst), vctx.reg_mr(back0), vctx.reg_mr(back1)
        qp = vctx.loopback_qp(depth=16)
        assert qp.on_gpu
        r = ops.gather_stream(qp, W.OP_RDMA_WRITE, ma, mb, md, nbytes, split, iters=n, window=8, burst=4, slot_stride=256,
                              nslots=n, timeout_ms=5000)
        assert r.ok and r.done == [n], r.status
        r = ops.gather_stream(qp, W.OP_RDMA_READ, m0, m1, md, nbytes, split, iters=n, window=8, burst=4, slot_stride=256,
                              nslots=n, timeout_ms=5000)
        assert r.ok and r.done == [n], r.status
        A, B, D = a.view(n, 256), b.view(n, 256), dst.view(n, 256)
        assert torch.equal(D[:, :split], A[:, :split]) and torch.equal(D[:, split:nbytes], B[:, :nbytes - split])
        assert int(D[:, nbytes:].count_nonzero()) == 0
        assert torch.equal(back0.view(n, 256)[:, :split], A[:, :split])
        assert torch.equal(back1.view(n, 256)[:, :nbytes - split], B[:, :nbytes - split])
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == 2 * n and c["n_bytes"] == 2 * n * nbytes, c
    finally:
        vctx.close()


@pytest.mark.multigpu
def test_gather_into_peer_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n0, n1 = 5 * MiB + 3, 7 * MiB
    ctx0, ctx1 = rn.Context(0), rn.Context(1)
    try:
        s0, s1 = _random(n0, 41), _random(n1, 42)
        dst = torch.zeros(n0 + n1 + 2 * GUARD, dtype=torch.uint8, device="cuda:1")
        m0, m1, md = ctx0.reg_mr(s0), ctx0.reg_mr(s1), ctx0.reg_mr(dst)
        qp = ctx0.loopback_qp(depth=16, mem=H)
        qp.set_flags(sys_scope=True)
        torch.cuda.synchronize(0); torch.cuda.synchronize(1)
        ctx0.engine_start(ctas=16, idle_timeout_ms=3000)
        try:
            qp.post_write_sg([(m0, 0, n0), (m1, 0, n1)], md, dst_off=GUARD)
            wc = qp.scq.wait(1, timeout_s=10)[0]
        finally:
            ctx0.engine_stop()
        _left_cleanly(ctx0)
        assert wc.status == "OK" and wc.byte_cnt == n0 + n1
        d = dst.to("cuda:0")
        assert torch.equal(d[GUARD:GUARD + n0], s0) and torch.equal(d[GUARD + n0:GUARD + n0 + n1], s1)
        assert _zero_outside(d, GUARD, GUARD + n0 + n1)
    finally:
        ctx0.close()
        ctx1.close()
