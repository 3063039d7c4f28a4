"""The maximum message length on the mock ConnectX, CPU only (DESIGN.md section 3.1).

A WRITE, WRITE_IMM, READ, SEND or SEND_IMM longer than 2^30 bytes completes with LOCAL_LENGTH_ERR before any key is
looked at: it moves nothing, consumes no receive, and the QP flushes what follows.  A byte count of 2^31 or more is
posted as the saturated 2^31 - 1, so it fails the same way instead of arriving as its low 31 bits (2^31 + 64 would
otherwise be a valid 64-byte WRITE).  Lengths that do not fit 32 bits are refused with ValueError before they are
posted.  Every buffer here is 64 KiB: an over-long WR is far longer than its MRs, which the length-first rule makes
harmless."""
import numpy as np
import pytest

import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, ops, wire as W

H = W.MEM_HOST_PINNED
L = W.MAX_MSG
BUF = 1 << 16
OFF, SPAN = 16 << 10, 16 << 10          # the WR's region inside the destination buffer; the rest are guards
POISON = 0xA5
OPS = ("WRITE", "WRITE_IMM", "READ", "SEND", "SEND_IMM")
TOO_LONG = [L + 1, L + 16, 2**31 - 1, 2**31, 2**31 + 64, 2**32 - 16]


@pytest.fixture(scope="module")
def lib():
    l = N.load()
    assert l.rn_verbs_available() >= 2 and l.rn_verbs_is_mock() == 1, l.rn_verbs_why()
    return l


@pytest.fixture
def pair(lib):
    """Two host-only contexts on two mock HCAs, one connected QP each: q0 requests, q1 responds."""
    c0, c1 = rn.Context(device=None, wire="verbs", nic=0), rn.Context(device=None, wire="verbs", nic=1)
    q0 = c0.create_qp(c0.create_cq(64, H), c0.create_cq(64, H), 16, 16, H)
    q1 = c1.create_qp(c1.create_cq(64, H), c1.create_cq(64, H), 16, 16, H)
    q0.connect(q1)
    yield c0, c1, q0, q1
    c0.close()
    c1.close()


def _post(q, op, src, dst, n):
    if op in ("WRITE", "WRITE_IMM"):
        return q.post_write(src, dst, n, src_off=OFF, dst_off=OFF, imm=7 if op == "WRITE_IMM" else None)
    if op == "READ":
        return q.post_read(dst, src, n, local_off=OFF, remote_off=OFF)
    return q.post_send(src, n, src_off=OFF, imm=7 if op == "SEND_IMM" else None)


def test_the_context_reports_the_limit(pair):
    c0, _, _, _ = pair
    assert c0.max_msg_bytes == L == 1 << 30          # the mock port's max_msg_sz


@pytest.mark.parametrize("n", TOO_LONG)
@pytest.mark.parametrize("op", OPS)
def test_over_long_fails_with_local_length_err(pair, op, n):
    c0, c1, q0, q1 = pair
    src = np.random.default_rng(n % 9973).integers(0, 256, BUF, dtype=np.uint8)
    dst = np.full(BUF, POISON, np.uint8)
    # the destination is the responder's for WRITE / SEND and the requester's own for READ
    if op == "READ":
        md, ms = c0.reg_mr(dst), c1.reg_mr(src)
    else:
        ms, md = c0.reg_mr(src), c1.reg_mr(dst)
    rcv = np.full(BUF, POISON, np.uint8)
    mr_rcv = c1.reg_mr(rcv)
    q1.post_recv(mr_rcv, SPAN, off=OFF)              # what a SEND or WRITE_IMM would take
    _post(q0, op, ms, md, n)
    q0.post_write(ms, md, 64) if op != "READ" else q0.post_read(md, ms, 64)
    wcs = q0.scq.wait(2)
    assert [w.status for w in wcs] == ["LOCAL_LENGTH_ERR", "WR_FLUSH_ERR"], (op, n, wcs)
    assert wcs[0].is_error and wcs[0].opcode == W.CQE_REQ_ERR
    assert (dst == POISON).all() and (rcv == POISON).all()
    assert q1.rcq.poll() == []                       # no receive was consumed
    c = q0.counters()
    assert (c["state"], c["n_wqe"], c["n_err"], c["n_bytes"]) == ("ERR", 2, 2, 0)


@pytest.mark.parametrize("op", OPS)
def test_the_limit_itself_is_a_legal_length(pair, op):
    """At exactly 2^30 the length check passes and the (64 KiB) MR check is what fails."""
    c0, c1, q0, q1 = pair
    src, dst = np.zeros(BUF, np.uint8), np.full(BUF, POISON, np.uint8)
    ms, md = (c1.reg_mr(src), c0.reg_mr(dst)) if op == "READ" else (c0.reg_mr(src), c1.reg_mr(dst))
    q1.post_recv(c1.reg_mr(np.zeros(BUF, np.uint8)), SPAN)
    _post(q0, op, ms, md, L)
    st = q0.scq.wait(1)[0].status
    assert st in ("LOCAL_PROT_ERR", "REMOTE_ACCESS_ERR", "REMOTE_INVAL_REQ_ERR") and (dst == POISON).all(), st


@pytest.mark.parametrize("rbytes", [2**31 + 4096, 2**32 - 1])
def test_an_oversized_receive_buffer_takes_a_send(pair, rbytes):
    """A receive buffer longer than the data segment can say holds any message (it used to be masked to 4096 bytes)."""
    c0, c1, q0, q1 = pair
    src = np.random.default_rng(3).integers(0, 256, BUF, dtype=np.uint8)
    dst = np.full(BUF, POISON, np.uint8)
    ms, md = c0.reg_mr(src), c1.reg_mr(dst)
    q1.post_recv(md, rbytes)
    q0.post_send(ms, 8192, imm=0x1234)
    assert q0.scq.wait(1)[0].status == "OK"
    r = q1.rcq.wait(1)[0]
    assert (r.status, r.byte_cnt, r.imm) == ("OK", 8192, 0x1234)
    assert (dst[:8192] == src[:8192]).all() and (dst[8192:] == POISON).all()


@pytest.mark.parametrize("n", [2**32 + 64, 2**33, -1])
def test_lengths_outside_32_bits_are_refused(pair, n):
    """Every host entry point that takes a byte count refuses one ctypes would wrap, and posts nothing."""
    c0, c1, q0, q1 = pair
    a, b = np.zeros(BUF, np.uint8), np.zeros(BUF, np.uint8)
    ma, mb = c0.reg_mr(a), c1.reg_mr(b)
    calls = [lambda: q0.post_write(ma, mb, n), lambda: q0.post_write(ma, mb, n, imm=1), lambda: q0.post_read(ma, mb, n),
             lambda: q0.post_send(ma, n), lambda: q0.post_send(ma, n, imm=1), lambda: q1.post_recv(mb, n),
             lambda: ops.rdma_stream(None, W.OP_RDMA_WRITE, None, None, n),
             lambda: ops.put_signal(None, None, None, n, None),
             lambda: ops.write_read(None, None, None, None, n)]
    for call in calls:
        with pytest.raises(ValueError, match="2\\*\\*32"):
            call()
    assert q0.counters()["n_wqe"] == 0 and q0.state == "RTS"
    assert q0.post_write(ma, mb, 16) is not None and q0.scq.wait(1)[0].status == "OK"


def test_write_resolved_granule_arithmetic_cannot_wrap():
    """The engine cuts a WQE into (bytes + chunk - 1) / chunk granules in uint32_t.  An unbounded chunk_bytes wraps that
    sum: chunk 0xFFFFFFF0 and a 100-byte WRITE give zero chunks.  With chunk_bytes and bytes both at most 2^30 -- what
    create_qp and the length check now guarantee -- the sum stays below 2^31 and the count is exact."""
    u32 = np.uint32
    with np.errstate(over="ignore"):
        assert int((u32(100) + u32(0xFFFFFFF0) - u32(1)) // u32(0xFFFFFFF0)) == 0
    for nbytes in (1, 16, L - 1, L):
        for chunk in (16, 16 << 10, 512 << 10, L):
            s = u32(nbytes) + u32(chunk) - u32(1)
            assert int(s) == nbytes + chunk - 1 < 2**31
            assert int(s // u32(chunk)) == -(-nbytes // chunk)
