"""The forwarding unpack, ``reduce_fp8(imm_base=)`` and the fp8 ring all-reduce on one GPU.

The rules of test_gpu_reduce.py hold: every kernel that waits is resident with what it waits for, every wait is bounded
by 5 s or less, nothing allocates or synchronises the device while the engine runs, arrival words are the head of a
zeroed tensor whose guard words must stay zero, and landing buffers start as poison (e4m3 448 under scale 2^127), so a
record read or forwarded before it has landed changes the result.
"""
import time
import types

import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import ring_fp8 as RF
from test_gpu_numerics import _bits_equal, _gen
from test_gpu_receive_fusion import _arrival_words, _check_arrival_words

pytestmark = pytest.mark.gpu

WAIT_MS = 5000
POISON_Q, POISON_S = 0x7E, 0xFE


def _poison(buf, chunk):
    r = buf.view(-1, P.record_bytes(chunk))
    r.fill_(POISON_S)
    r[:, :chunk] = POISON_Q


def _records(n, chunk, seed):
    x = (torch.randn(n, generator=_gen(seed)) * 16).to(torch.bfloat16)
    return P.ref_pack_fp8(x, chunk)


class _Fwd:
    """A landing buffer of n_rec records with its words, forwarded over a loopback QP into a poisoned destination whose
    receive completions ``recv_consume`` turns into downstream words at ``imm_base + r``."""

    def __init__(self, ctx, chunk, n_rec, imm_base, seed):
        self.ctx, self.chunk, self.n_rec, self.imm_base = ctx, chunk, n_rec, imm_base
        self.n = chunk * n_rec
        self.nb = P.staging_bytes(self.n, chunk)
        self.want = _records(self.n, chunk, seed)
        self.src = self.want.cuda()
        self.land = torch.empty(self.nb + 256, dtype=torch.uint8, device="cuda")
        self.dst = torch.empty(self.nb + 256, dtype=torch.uint8, device="cuda")
        for b in (self.land, self.dst):
            _poison(b[:self.nb], chunk)
            b[self.nb:].fill_(0xC5)
        self.y = torch.full((self.n + 64,), 7.0, dtype=torch.bfloat16, device="cuda")
        self.lmr, self.dmr = ctx.reg_mr(self.land[:self.nb]), ctx.reg_mr(self.dst[:self.nb])
        self.full, self.ready = _arrival_words(n_rec)
        self.dfull, self.dready = _arrival_words(imm_base + n_rec)
        self.qp = ctx.loopback_qp(depth=64)

    def check_bytes(self, records):
        rec = P.record_bytes(self.chunk)
        d, w = self.dst[:self.nb].view(self.n_rec, rec).cpu(), self.want.view(self.n_rec, rec)
        for r in range(self.n_rec):
            if r in records:
                assert torch.equal(d[r], w[r]), f"record {r} at the destination"
            else:
                assert bool((d[r, :self.chunk] == POISON_Q).all()) and bool((d[r, self.chunk:] == POISON_S).all()), \
                    f"record {r} was forwarded"
        assert bool((self.dst[self.nb:] == 0xC5).all())


# ------------------------------------------------------------------ 1. the forwarding unpack
@pytest.mark.parametrize("signal_every", [1, 4])
def test_forwarding_unpack_words_set_out_of_order(ctx, signal_every):
    """The unpack is launched on poisoned records; another stream lands and stamps them in a shuffled order.  Each
    record is forwarded once, as WRITE_IMM with imm_base + r: the downstream words at [imm_base, imm_base + n_rec) are
    stamped and nothing below; both ends are bit-exact and n_wqe == n_rec + 1."""
    chunk, n_rec, imm_base = 16384, 6, 10
    f = _Fwd(ctx, chunk, n_rec, imm_base, seed=1)
    rec = P.record_bytes(chunk)
    order = torch.randperm(n_rec, generator=_gen(2)).tolist()
    s_set, s_c, s_u = ctx.streams(3)
    # the setter runs once before the unpack exists: a kernel's first load waits for every resident kernel (DESIGN.md
    # 3.2), so only these very calls load what the setter needs
    with torch.cuda.stream(s_set):
        for r in order:
            f.land[r * rec:(r + 1) * rec].copy_(f.src[r * rec:(r + 1) * rec])
            f.ready[r:r + 1].fill_(1)
    torch.cuda.synchronize()
    _poison(f.land[:f.nb], chunk)
    f.full.zero_()
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + unpack 8 = 17 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cv, _ = ops.recv_consume(f.qp, n_rec, imm_base + n_rec, f.dready, timeout_ms=WAIT_MS, sync=False, stream=s_c,
                                 prepost_mr=f.dmr, prepost_bytes=0)
        uv, _ = ops.unpack_fp8(ctx, f.land[:f.nb], f.y[:f.n], chunk, ready=f.ready, grid=8, timeout_ms=WAIT_MS,
                               stream=s_u, sync=False, fwd_qp=f.qp, fwd_src_mr=f.lmr, fwd_dst_mr=f.dmr, with_imm=True,
                               imm_base=imm_base, signal_every=signal_every)
        with torch.cuda.stream(s_set):
            for r in order:
                f.land[r * rec:(r + 1) * rec].copy_(f.src[r * rec:(r + 1) * rec])
                f.ready[r:r + 1].fill_(1)
        for s in (s_set, s_c, s_u):
            s.synchronize()
    finally:
        ctx.engine_stop()
    u = ops.parse_unpack(uv)
    assert u["status"] == "OK" and u["records_forwarded"] == n_rec and u["t_first_post_ns"] > 0, u
    c = ops.parse_recv(cv)
    assert c["status"] == "OK" and c["seen"] == n_rec, c
    assert bool((f.dfull[:imm_base] == 0).all()), "a word below imm_base was stamped"
    _check_arrival_words(f.dfull[imm_base:], n_rec)
    f.check_bytes(set(range(n_rec)))
    assert _bits_equal(f.y[:f.n].cpu(), P.ref_unpack_fp8(f.want, f.n, chunk))
    assert bool((f.y[f.n:] == 7.0).all())
    q = f.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == n_rec + 1, q


def test_forwarding_unpack_without_words_post_only(ctx):
    """No words at all (the records are in place) and post_only: the kernel ends on its own and the one-shot engine
    then delivers every record once."""
    chunk, n_rec = 8192, 5
    f = _Fwd(ctx, chunk, n_rec, 0, seed=3)
    f.land[:f.nb].copy_(f.src)
    for _ in range(n_rec):
        f.qp.post_recv(f.dmr, 0)
    torch.cuda.synchronize()
    u = ops.unpack_fp8(ctx, f.land[:f.nb], f.y[:f.n], chunk, grid=3, timeout_ms=WAIT_MS, fwd_qp=f.qp, fwd_src_mr=f.lmr,
                       fwd_dst_mr=f.dmr, post_only=True)
    assert u["status"] == "OK" and u["records_forwarded"] == n_rec, u
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    f.check_bytes(set(range(n_rec)))
    q = f.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == n_rec + 1, q


def test_forwarding_unpack_withheld_word_times_out(ctx):
    """Word 2 never comes: TIMEOUT within the bound, record 2 is never forwarded, every other record once."""
    chunk, n_rec = 8192, 4
    f = _Fwd(ctx, chunk, n_rec, 0, seed=4)
    f.land[:f.nb].copy_(f.src)
    f.ready.fill_(1)
    f.ready[2] = 0
    s_c, s_u = ctx.streams(2)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cv, _ = ops.recv_consume(f.qp, n_rec - 1, n_rec, f.dready, timeout_ms=WAIT_MS, sync=False, stream=s_c,
                                 prepost_mr=f.dmr, prepost_bytes=0)
        t0 = time.monotonic()
        u = ops.unpack_fp8(ctx, f.land[:f.nb], f.y[:f.n], chunk, ready=f.ready, grid=4, timeout_ms=300, stream=s_u,
                           fwd_qp=f.qp, fwd_src_mr=f.lmr, fwd_dst_mr=f.dmr, with_imm=True)
        dt = time.monotonic() - t0
        s_c.synchronize()
    finally:
        ctx.engine_stop()
    assert u["status"] == "TIMEOUT" and u["records_forwarded"] == n_rec - 1, u
    assert dt < 3.0, f"the timeout took {dt:.2f} s"
    st = f.dfull.tolist()
    assert st[2] == 0 and all(st[i] != 0 for i in (0, 1, 3)), st
    f.check_bytes({0, 1, 3})
    q = f.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == n_rec, q                  # three records and the flush


def test_forwarding_unpack_bad_rkey(ctx):
    """A destination region with a bad rkey: the first WRITE fails and puts the QP in error, the records posted after
    it complete flushed (or are refused, which ``post_record`` reports as TIMEOUT), the status is not OK, the kernel
    ends without waiting out its timeout, and nothing lands at the real destination."""
    chunk, n_rec = 8192, 4
    f = _Fwd(ctx, chunk, n_rec, 0, seed=5)
    f.land[:f.nb].copy_(f.src)
    # an MKey index far past the table: it translates nowhere
    bad = types.SimpleNamespace(addr=f.dmr.addr, length=f.dmr.length, rkey=(f.dmr.rkey & 0xFF) | 0xFFFF00)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        u = ops.unpack_fp8(ctx, f.land[:f.nb], f.y[:f.n], chunk, grid=1, timeout_ms=WAIT_MS, fwd_qp=f.qp,
                           fwd_src_mr=f.lmr, fwd_dst_mr=bad)
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    assert u["status"] != "OK" and u["records_forwarded"] < n_rec, u
    assert dt < WAIT_MS / 1000, f"the failed forward took {dt:.2f} s"
    f.check_bytes(set())
    q = f.qp.counters()
    assert q["n_err"] >= 1, q


def test_forwarding_unpack_through_the_mock_connectx():
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        chunk, n_rec = 1 << 16, 4
        f = _Fwd(vctx, chunk, n_rec, 0, seed=6)
        f.land[:f.nb].copy_(f.src)
        assert f.qp.on_gpu
        torch.cuda.synchronize()
        u = ops.unpack_fp8(vctx, f.land[:f.nb], f.y[:f.n], chunk, timeout_ms=WAIT_MS, fwd_qp=f.qp, fwd_src_mr=f.lmr,
                           fwd_dst_mr=f.dmr, signal_every=2)
        assert u["status"] == "OK" and u["records_forwarded"] == n_rec, u
        f.check_bytes(set(range(n_rec)))
        assert _bits_equal(f.y[:f.n].cpu(), P.ref_unpack_fp8(f.want, f.n, chunk))
        q = f.qp.counters()
        assert q["n_err"] == 0 and q["n_db_order_violations"] == 0, q
    finally:
        vctx.close()


def test_forwarding_unpack_host_rejections(ctx):
    chunk, n_rec = 8192, 2
    f = _Fwd(ctx, chunk, n_rec, 0, seed=7)
    small = ctx.reg_mr(f.dst[:f.nb - 64])
    other = ctx.reg_mr(f.dst[:f.nb])
    base = dict(fwd_qp=f.qp, fwd_src_mr=f.lmr, fwd_dst_mr=f.dmr)
    bad = [
        (dict(fwd_dst_mr=small), "do not"),
        (dict(fwd_dst_off=64), "do not"),
        (dict(fwd_src_mr=other), "inside fwd_src_mr"),
        (dict(qp=f.qp), "not both|CQ poller"),
        (dict(imm_base=(1 << 32) - 1), "32 bits"),
        (dict(fwd_dst_mr=None), "together"),
    ]
    torch.cuda.synchronize()
    for kw, what in bad:
        args = dict(base)
        args.update(kw)
        with pytest.raises(ValueError, match=what):
            ops.unpack_fp8(ctx, f.land[:f.nb], f.y[:f.n], chunk, **args)
    assert f.qp.counters()["n_wqe"] == 0


# ------------------------------------------------------------------ 2. reduce_fp8(imm_base=)
def test_reduce_imm_base_lands_in_the_offset_words(ctx):
    chunk, n_rec, imm_base = 8192, 4, 9
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    recs = _records(n, chunk, seed=8).cuda()
    loc = (torch.randn(n, generator=_gen(9)) * 4).to(torch.bfloat16).cuda()
    _, want_r = P.ref_reduce_fp8(recs.cpu(), 1, n, chunk, local=loc.cpu())
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nb, dtype=torch.uint8, device="cuda")
    _poison(dst, chunk)
    smr, dmr = ctx.reg_mr(stg), ctx.reg_mr(dst)
    full, ready = _arrival_words(imm_base + n_rec)
    qp = ctx.loopback_qp(depth=64)
    s_c, s_r = ctx.streams(2)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cv, _ = ops.recv_consume(qp, n_rec, imm_base + n_rec, ready, timeout_ms=WAIT_MS, sync=False, stream=s_c,
                                 prepost_mr=dmr, prepost_bytes=0)
        r = ops.reduce_fp8(ctx, recs, 1, n, chunk, local=loc, out_mr=smr, qp=qp, dst_mr=dmr, with_imm=True, grid=4,
                           timeout_ms=WAIT_MS, stream=s_r, imm_base=imm_base)
        s_c.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.records_posted == n_rec, r
    assert ops.parse_recv(cv)["seen"] == n_rec
    assert bool((full[:imm_base] == 0).all())
    _check_arrival_words(full[imm_base:], n_rec)
    assert torch.equal(dst.cpu(), want_r)


# ------------------------------------------------------------------ 3. the ring all-reduce, N simulated ranks
def _ring(ctx, N, chunk, R, signal_every, timeout_ms=WAIT_MS):
    plans = [RF.RingAllreduceFp8(ctx, N * R * chunk, chunk, q, N, timeout_ms=timeout_ms, signal_every=signal_every)
             for q in range(N)]
    RF.link_in_process(plans)
    return plans


def _inputs(N, n, seed):
    g = _gen(seed)
    return [(torch.randn(n, generator=g) * 4).to(torch.bfloat16) for _ in range(N)]


def _run_checked(ctx, plans, xs_cpu, in_place):
    """One run from poisoned landing buffers; every output against the reference and against rank 0's."""
    N = len(plans)
    chunk = plans[0].chunk
    want = ops.ref_allreduce_fp8(xs_cpu, chunk)
    xs = [x.cuda() for x in xs_cpu]
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
        assert _bits_equal(got[q].cpu(), want), f"rank {q} differs from the reference"
        assert torch.equal(got[q].view(torch.int16), got[0].view(torch.int16))
        _check_arrival_words(plans[q].words_full, plans[q].n_ids)
        c = plans[q].send_qp.counters()
        assert c["n_err"] == 0, c
    return res


@pytest.mark.parametrize("signal_every", [1, 4])
@pytest.mark.parametrize("chunk", [8192, 1 << 20], ids=["8192", "1M"])
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_allreduce_matches_reference(ctx, N, chunk, signal_every):
    """In place, then into ``out`` with other inputs: every rank bit-identical to ``ref_allreduce_fp8``."""
    R = 3 if chunk == 8192 else 1
    plans = _ring(ctx, N, chunk, R, signal_every)
    n = N * R * chunk
    _run_checked(ctx, plans, _inputs(N, n, seed=N * 10 + signal_every), in_place=True)
    _run_checked(ctx, plans, _inputs(N, n, seed=N * 10 + signal_every + 5), in_place=False)


def test_allreduce_rank_that_never_contributes(ctx):
    """Rank 1 posts its receives but never runs its main stream: every other rank reports TIMEOUT, no wait is longer
    than timeout_ms and the run ends within 2N x timeout_ms.  The next run, with all ranks, is clean."""
    N, chunk, R, tmo = 3, 8192, 2, 300
    plans = _ring(ctx, N, chunk, R, 1, timeout_ms=tmo)
    n = N * R * chunk
    xs = [x.cuda() for x in _inputs(N, n, seed=77)]
    outs = [torch.zeros_like(x) for x in xs]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        res = RF.run_in_process(plans, xs, outs, skip={1})
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    for r in res:
        assert r.status == "TIMEOUT", (r.rank, r.status, r.failed)
        for l in r.launches:
            assert l.status in ("OK", "TIMEOUT"), (r.rank, l)
    assert dt < 2 * N * tmo / 1000 + 1.0, f"the failed run took {dt:.2f} s"
    for p in plans:
        assert p.send_qp.counters()["n_err"] == 0
    _run_checked(ctx, plans, _inputs(N, n, seed=78), in_place=False)


def test_allreduce_rejections(ctx):
    with pytest.raises(ValueError, match="at least 2"):
        RF.RingAllreduceFp8(ctx, 8192, 8192, 0, 1)
    with pytest.raises(ValueError, match="multiple of world"):
        RF.RingAllreduceFp8(ctx, 3 * 8192, 8192, 0, 2)
    plans = [RF.RingAllreduceFp8(ctx, 2 * 8192, 8192, q, 2) for q in range(2)]
    with pytest.raises(ValueError, match="must hold"):
        RF.link_in_process(plans, rq_depth=2)
    with pytest.raises(ValueError, match="SM budget"):
        RF.link_in_process([RF.RingAllreduceFp8(ctx, 2 * 8192, 8192, q, 2, grid=200) for q in range(2)])
    big = [RF.RingAllreduceFp8(ctx, 9 * 8192, 8192, q, 9) for q in range(9)]
    with pytest.raises(ValueError, match="scratch"):
        RF.link_in_process(big)
