"""The maximum message length (2^30 bytes, DESIGN.md section 3.1) on one H100, on both wires.

At the limit: 1 GiB WRITE, READ, WRITE_IMM and SEND_IMM (into a receive of exactly 2^30 bytes) at lengths L, L-1, L-15
and L-16, from source / destination residues (0,0), (8,8) and (1,15) mod 16 -- the bulk TMA path, the generic path's
16-byte body and its byte loop -- on 1, 32 and 128 engine CTAs and chunk_bytes of 16 KiB, 512 KiB and L, posted from the
host and from the device (rdma_stream, and put_signal checked by signal_wait).  Every case checks the bytes, 4 KiB
poisoned guards on both sides, byte_cnt, the number of bulk chunks rc_model predicts, and that the engine left cleanly.
The mock ConnectX runs the same at the limit with its data in HBM.

Past the limit, from the device on both wires: the WR completes with LOCAL_LENGTH_ERR, moves nothing, and fails the QP.
Byte counts of 2^31 and more reach the wire saturated, so they fail the same way instead of being truncated."""
import itertools
import types

import pytest
import torch

import rc_model as M
import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, ops, wire as W

pytestmark = pytest.mark.gpu

K = 1 << 10
L = W.MAX_MSG
G = 4 * K                         # poisoned guard on each side of a message
BUF = L + 128 * K                 # room for guards, residues and an MR of L + 64 KiB
POISON = 0xA5
H = W.MEM_HOST_PINNED
OPS4 = ("WRITE", "READ", "WRITE_IMM", "SEND_IMM")
LENS = (L, L - 1, L - 15, L - 16)
RES = ((0, 0), (8, 8), (1, 15))
CTAS = (1, 32, 128)
CHUNKS = (16 * K, 512 * K, L)
TIMEOUT_MS = 30000


def _layout(i):
    """Case i's (residues, engine CTAs, chunk_bytes): the first nine cover every residue x CTA pair and each of those
    with every chunk size once (a Latin square).  The byte loop of (1,15) is not run on one CTA: too slow there."""
    res, ctas = RES[i % 3], CTAS[(i // 3) % 3]
    if res == (1, 15) and ctas == 1:
        ctas = 128
    return res, ctas, CHUNKS[(i + i // 3) % 3]


HOST_CASES = [(op, n) + _layout(i) for i, (op, n) in enumerate(itertools.product(OPS4, LENS))]
DEV_CASES = [(op, n) + _layout(i + 1) for i, (op, n) in enumerate(itertools.product(OPS4[:3], LENS))]
SIGNAL_CASES = [(L, 128, 16 * K), (L - 16, 1, 512 * K), (L, 32, L)]     # signal_wait's check wants 16-byte alignment
OVER = (L + 16, 2**31, 2**31 + 4096, 2**32 - 16)
_OPC = {"WRITE": W.OP_RDMA_WRITE, "READ": W.OP_RDMA_READ, "WRITE_IMM": W.OP_RDMA_WRITE_IMM}


def _id(c):
    op, n, res, ctas, chunk = c
    return f"{op}-L{n - L:+d}-r{res[0]}.{res[1]}-c{ctas}-k{chunk // K}"


@pytest.fixture(scope="module")
def bufs():
    src = torch.empty(BUF, dtype=torch.uint8, device="cuda:0")
    dst = torch.empty(BUF, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=2024)
    torch.cuda.synchronize()
    yield src, dst
    del src, dst
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def hca(bufs):
    src, dst = bufs
    ctx = rn.Context(device=0, wire="softhca")
    sig, fetch = torch.zeros(64, dtype=torch.uint8, device="cuda:0"), torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    m = types.SimpleNamespace(ctx=ctx, src=ctx.reg_mr(src), dst=ctx.reg_mr(dst), sig=ctx.reg_mr(sig), fetch=ctx.reg_mr(fetch),
                              sig_t=sig)
    yield m
    ctx.close()


@pytest.fixture(scope="module")
def mock(bufs):
    src, dst = bufs
    ctx = rn.Context(device=0, wire="verbs", nic=0)
    assert ctx.nic_is_mock
    yield types.SimpleNamespace(ctx=ctx, src=ctx.reg_mr(src), dst=ctx.reg_mr(dst))
    ctx.close()


def _at(mr, off):
    """The MR's keys with its address moved by ``off`` (what the device posters take)."""
    return types.SimpleNamespace(addr=mr.addr + off, lkey=mr.lkey, rkey=mr.rkey, length=mr.length - off)


def _poison(dst):
    dst.fill_(POISON)
    torch.cuda.synchronize()


def _check_bytes(src, dst, s0, d0, n):
    assert ops.compare(dst[d0:d0 + n], src[s0:s0 + n], n) == 0
    assert int((dst[:d0] != POISON).sum()) == 0 and int((dst[d0 + n:] != POISON).sum()) == 0, "guard bytes changed"


def _host_post(qp, m, op, n, s0, d0):
    if op == "READ":
        qp.post_read(m.dst, m.src, n, local_off=d0, remote_off=s0)
    elif op.startswith("WRITE"):
        qp.post_write(m.src, m.dst, n, src_off=s0, dst_off=d0, imm=0x51 if op == "WRITE_IMM" else None)
    else:
        qp.post_send(m.src, n, src_off=s0, imm=0x52)


def _completions(qp, op, n):
    wc = qp.scq.wait(1)[0]
    assert (wc.status, wc.byte_cnt) == ("OK", n), wc
    if op in ("WRITE_IMM", "SEND_IMM"):
        r = qp.rcq.wait(1)[0]
        assert (r.status, r.byte_cnt) == ("OK", n), r


def _engine_left_cleanly(ctx, n, s0, d0, ctas, chunk):
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    assert st["n_bulk_chunks"] == M.bulk_chunks(n, s0, d0, ctas, chunk), st


# ---------------------------------------------------------------------------------------------------------------- at the limit
@pytest.mark.parametrize("case", HOST_CASES, ids=map(_id, HOST_CASES))
def test_softhca_host_posted_at_the_limit(bufs, hca, case):
    op, n, (rs, rd), ctas, chunk = case
    src, dst = bufs
    s0, d0 = G + rs, G + rd
    _poison(dst)
    qp = hca.ctx.loopback_qp(depth=16, mem=H, chunk_bytes=chunk)
    if op in ("WRITE_IMM", "SEND_IMM"):
        qp.post_recv(hca.dst, L, off=d0)            # a receive of exactly L bytes
    _host_post(qp, hca, op, n, s0, d0)
    hca.ctx.engine_run_oneshot(ctas=ctas)
    _engine_left_cleanly(hca.ctx, n, s0, d0, ctas, chunk)
    _completions(qp, op, n)
    assert qp.counters()["n_bytes"] == n
    _check_bytes(src, dst, s0, d0, n)


@pytest.mark.parametrize("case", DEV_CASES, ids=map(_id, DEV_CASES))
def test_softhca_device_posted_at_the_limit(bufs, hca, case):
    op, n, (rs, rd), ctas, chunk = case
    src, dst = bufs
    s0, d0 = G + rs, G + rd
    _poison(dst)
    qp = hca.ctx.loopback_qp(depth=16, chunk_bytes=chunk)
    if op == "WRITE_IMM":
        qp.post_recv(hca.dst, L, off=d0)
    local, remote = (_at(hca.dst, d0), _at(hca.src, s0)) if op == "READ" else (_at(hca.src, s0), _at(hca.dst, d0))
    r = ops.rdma_stream(qp, _OPC[op], local, remote, n, post_only=True, timeout_ms=TIMEOUT_MS)
    assert r.ok and r.done == [1], r.status
    hca.ctx.engine_run_oneshot(ctas=ctas)
    _engine_left_cleanly(hca.ctx, n, s0, d0, ctas, chunk)
    _completions(qp, op, n)
    assert qp.counters()["n_bytes"] == n
    _check_bytes(src, dst, s0, d0, n)


@pytest.mark.parametrize("n,ctas,chunk", SIGNAL_CASES, ids=[f"L{n - L:+d}-c{c}-k{k // K}" for n, c, k in SIGNAL_CASES])
def test_softhca_put_signal_at_the_limit(bufs, hca, n, ctas, chunk):
    """A 1 GiB put-with-signal: the receiver's signal_wait compares the message the moment the signal covers it."""
    src, dst = bufs
    _poison(dst)
    hca.sig_t.zero_()
    torch.cuda.synchronize()
    qp = hca.ctx.loopback_qp(depth=16, chunk_bytes=chunk)
    hca.ctx.engine_start(ctas=ctas, idle_timeout_ms=10000)
    try:
        r = ops.put_signal(qp, _at(hca.src, G), _at(hca.dst, G), n, hca.sig, fetch_mr=hca.fetch, timeout_ms=TIMEOUT_MS)
        assert r.ok and r.done == [1], r.status
        w = ops.signal_wait(hca.ctx, hca.sig, 1, check=(dst[G:], src[G:], n, n), timeout_ms=TIMEOUT_MS)
        assert w["status"] == "OK" and w["seen"] == 1 and w["mismatches"] == 0, w
    finally:
        hca.ctx.engine_stop()
    _engine_left_cleanly(hca.ctx, n, G, G, ctas, chunk)
    assert qp.counters()["n_bytes"] == n + 8       # the WRITE and the 8-byte fetch-and-add
    _check_bytes(src, dst, G, G, n)


MOCK_HOST = [(op, n, RES[i % 3]) for i, (op, n) in enumerate(itertools.product(OPS4, (L, L - 15)))]
MOCK_DEV = [(op, n, RES[(i + 1) % 3]) for i, (op, n) in enumerate(itertools.product(OPS4[:3], (L, L - 1)))]


@pytest.mark.parametrize("op,n,res", MOCK_HOST, ids=[f"{o}-L{n - L:+d}-r{r[0]}.{r[1]}" for o, n, r in MOCK_HOST])
def test_mock_host_posted_at_the_limit_on_hbm(bufs, mock, op, n, res):
    src, dst = bufs
    s0, d0 = G + res[0], G + res[1]
    _poison(dst)
    qp = mock.ctx.loopback_qp(depth=16, mem=H)
    if op in ("WRITE_IMM", "SEND_IMM"):
        qp.post_recv(mock.dst, L, off=d0)
    _host_post(qp, mock, op, n, s0, d0)
    _completions(qp, op, n)
    torch.cuda.synchronize()
    assert mock.ctx.max_msg_bytes == L and qp.counters()["n_bytes"] == n
    _check_bytes(src, dst, s0, d0, n)


@pytest.mark.parametrize("op,n,res", MOCK_DEV, ids=[f"{o}-L{n - L:+d}-r{r[0]}.{r[1]}" for o, n, r in MOCK_DEV])
def test_mock_device_posted_at_the_limit_on_hbm(bufs, mock, op, n, res):
    src, dst = bufs
    s0, d0 = G + res[0], G + res[1]
    _poison(dst)
    qp = mock.ctx.loopback_qp(depth=16)
    if op == "WRITE_IMM":
        qp.post_recv(mock.dst, L, off=d0)
    local, remote = (_at(mock.dst, d0), _at(mock.src, s0)) if op == "READ" else (_at(mock.src, s0), _at(mock.dst, d0))
    r = ops.rdma_stream(qp, _OPC[op], local, remote, n, timeout_ms=TIMEOUT_MS)
    assert r.ok and r.done == [1], r.status
    torch.cuda.synchronize()
    c = qp.counters()
    assert (c["n_bytes"], c["n_err"]) == (n, 0), c
    _check_bytes(src, dst, s0, d0, n)


# ---------------------------------------------------------------------------------------------------------------- past the limit
def _over_limit_outcome(qp, r, dst):
    assert r.status == ["CQE_ERROR"], r.status
    wc = qp.scq.poll(4)
    assert [w.status for w in wc] == ["LOCAL_LENGTH_ERR"], wc
    c = qp.counters()
    assert (c["n_err"], c["n_bytes"], c["state"]) == (1, 0, "ERR"), c
    assert int((dst != POISON).sum()) == 0


def test_softhca_device_posted_past_the_limit(bufs, hca):
    _, dst = bufs
    _poison(dst)
    qps = [hca.ctx.loopback_qp(depth=16) for _ in OVER]          # every QP exists before the engine is resident
    hca.ctx.engine_start(ctas=32, idle_timeout_ms=10000)
    try:
        results = [ops.rdma_stream(qp, W.OP_RDMA_WRITE, _at(hca.src, G), _at(hca.dst, G), n, timeout_ms=TIMEOUT_MS)
                   for qp, n in zip(qps, OVER)]
    finally:
        hca.ctx.engine_stop()
    st = hca.ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0 and st["n_bulk_chunks"] == 0, st
    for qp, r in zip(qps, results):
        _over_limit_outcome(qp, r, dst)
    with pytest.raises(ValueError):
        ops.rdma_stream(qps[0], W.OP_RDMA_WRITE, hca.src, hca.dst, 2**32 + 64)


def test_mock_device_posted_past_the_limit(bufs, mock):
    _, dst = bufs
    _poison(dst)
    for n in OVER:
        qp = mock.ctx.loopback_qp(depth=16)
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, _at(mock.src, G), _at(mock.dst, G), n, timeout_ms=TIMEOUT_MS)
        torch.cuda.synchronize()
        _over_limit_outcome(qp, r, dst)
    with pytest.raises(ValueError):
        ops.rdma_stream(qp, W.OP_RDMA_WRITE, mock.src, mock.dst, 2**32 + 64)


def test_default_length_on_an_mr_past_the_limit(bufs, hca):
    """post_write(src_mr, dst_mr) sends the whole source MR: at L + 64 KiB that is one message too long."""
    src, dst = bufs
    _poison(dst)
    ms, md = hca.ctx.reg_mr(src, nbytes=L + 64 * K), hca.ctx.reg_mr(dst, nbytes=L + 64 * K)
    qp = hca.ctx.loopback_qp(depth=16, mem=H)
    qp.post_write(ms, md)
    qp.post_write(ms, md, 64)
    hca.ctx.engine_run_oneshot(ctas=32)
    assert [w.status for w in qp.scq.wait(2)] == ["LOCAL_LENGTH_ERR", "WR_FLUSH_ERR"]
    assert hca.ctx.engine_stats()["fatal"] == 0
    assert int((dst != POISON).sum()) == 0
    ms.dereg(); md.dereg()


def test_chunk_bytes_and_host_byte_counts_are_bounded(hca):
    assert hca.ctx.max_msg_bytes == L
    hca.ctx.loopback_qp(depth=16, mem=H, chunk_bytes=L)
    with pytest.raises(N.NativeError, match="chunk_bytes"):
        hca.ctx.loopback_qp(depth=16, mem=H, chunk_bytes=L + 16)
    with pytest.raises(ValueError):
        hca.ctx.loopback_qp(depth=16, mem=H, chunk_bytes=2**32 + 64)
    qp = hca.ctx.loopback_qp(depth=16, mem=H)
    for call in (lambda: qp.post_write(hca.src, hca.dst, 2**32 + 64), lambda: qp.post_read(hca.dst, hca.src, 2**32 + 64),
                 lambda: qp.post_send(hca.src, 2**32 + 64, imm=1), lambda: qp.post_recv(hca.dst, 2**32 + 64)):
        with pytest.raises(ValueError):
            call()
    assert qp.counters()["n_wqe"] == 0


def test_a_send_lands_in_a_receive_buffer_past_2_31_bytes(bufs, hca):
    """A receive of 2^31 + 64 KiB (more than a data segment says) takes a 1 MiB SEND; it used to read as 64 KiB."""
    src, _ = bufs
    big = torch.full((2**31 + 64 * K,), POISON, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    mbig = hca.ctx.reg_mr(big)
    qp = hca.ctx.loopback_qp(depth=16, mem=H)
    qp.post_recv(mbig)
    qp.post_send(hca.src, 1 << 20, src_off=G, imm=9)
    hca.ctx.engine_run_oneshot(ctas=32)
    assert qp.scq.wait(1)[0].status == "OK"
    r = qp.rcq.wait(1)[0]
    assert (r.status, r.byte_cnt, r.imm) == ("OK", 1 << 20, 9)
    assert ops.compare(big[:1 << 20], src[G:G + (1 << 20)]) == 0 and int((big[1 << 20:] != POISON).sum()) == 0
    mbig.dereg()
    del big
    torch.cuda.empty_cache()
