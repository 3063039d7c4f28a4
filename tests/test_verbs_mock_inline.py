"""Inline work requests on the verbs wire, against the in-tree mock ConnectX (two ports, host memory, CPU only): the
payload is taken into the WQE when it is posted, SEND and WRITE_WITH_IMM deliver into posted receive buffers, and the
provider refuses what cannot be inline."""
import ctypes as C

import numpy as np
import pytest

import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, wire as W

H = W.MEM_HOST_PINNED
EINVAL = 22


@pytest.fixture
def pair():
    lib = N.load()
    if lib.rn_verbs_available() < 2 or lib.rn_verbs_is_mock() != 1:
        pytest.skip("needs the mock verbs provider with two ports")
    c0, c1 = rn.Context(device=None, wire="verbs", nic=0), rn.Context(device=None, wire="verbs", nic=1)
    q0 = c0.create_qp(c0.create_cq(64, H), c0.create_cq(64, H), 16, 16, H)
    q1 = c1.create_qp(c1.create_cq(64, H), c1.create_cq(64, H), 16, 16, H)
    q0.connect(q1)
    yield c0, c1, q0, q1
    c0.close()
    c1.close()


def test_inline_write_lands_and_the_source_may_change_after_the_post(pair):
    c0, c1, q0, _ = pair
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    src = bytearray(range(1, 29))
    q0.post_write_inline(md, src, dst_off=3)
    src[:] = bytes(28)                                   # the provider copied the bytes at post time
    q0.post_write_inline(md, np.array([0xAB, 0xCD], dtype=np.uint8), dst_off=40, signaled=False)
    q0.post_write_inline(md, b"\x11" * 12, dst_off=50)
    wcs = q0.scq.wait(2)
    assert [w.status for w in wcs] == ["OK", "OK"] and [w.byte_cnt for w in wcs] == [28, 12]
    assert bytes(dst[3:31]) == bytes(range(1, 29))
    assert bytes(dst[40:42]) == b"\xab\xcd" and bytes(dst[50:62]) == b"\x11" * 12
    assert not dst[:3].any() and not dst[31:40].any() and not dst[42:50].any() and not dst[62:].any()


def test_inline_send_lands_in_the_posted_receive_buffer(pair):
    c0, c1, q0, q1 = pair
    rbuf = np.zeros(32, dtype=np.uint8)
    q1.post_recv(c1.reg_mr(rbuf))
    q0.post_send_inline(b"0123456789abcdefghi", imm=0x5150)
    assert q0.scq.wait(1)[0].status == "OK"
    rwc = q1.rcq.wait(1)[0]
    assert rwc.status == "OK" and rwc.byte_cnt == 19 and rwc.imm == 0x5150
    assert bytes(rbuf[:19]) == b"0123456789abcdefghi" and not rbuf[19:].any()


def test_inline_write_with_imm_delivers_its_immediate(pair):
    c0, c1, q0, q1 = pair
    dst, rbuf = np.zeros(16, dtype=np.uint8), np.zeros(16, dtype=np.uint8)
    md = c1.reg_mr(dst)
    q1.post_recv(c1.reg_mr(rbuf))
    q0.post_write_inline(md, b"\x07" * 5, dst_off=1, imm=0xFEED)
    assert q0.scq.wait(1)[0].status == "OK"
    rwc = q1.rcq.wait(1)[0]
    assert rwc.status == "OK" and rwc.imm == 0xFEED
    assert bytes(dst[1:6]) == b"\x07" * 5 and dst[0] == 0 and not dst[6:].any()


def test_provider_refuses_what_cannot_be_inline(pair):
    c0, c1, q0, _ = pair
    lib = c0._lib
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    buf = C.create_string_buffer(29)
    wr = C.c_uint64()
    # the provider itself (ibv_post_send with IBV_SEND_INLINE) refuses these
    assert lib.rn_verbs_post_inline(q0._vq, W.OP_RDMA_WRITE, md.addr, md.rkey, buf, 29, 1, 0, C.byref(wr)) == -EINVAL
    assert lib.rn_verbs_post_inline(q0._vq, W.OP_RDMA_READ, md.addr, md.rkey, buf, 8, 1, 0, C.byref(wr)) == -EINVAL
    with pytest.raises(ValueError):
        q0.post_write_inline(md, bytes(29))
    with pytest.raises(ValueError):
        q0.post_send_inline(b"")
    q0.post_write_inline(md, b"ok")                       # nothing was queued by the refused posts
    wc = q0.scq.wait(1)[0]
    assert wc.status == "OK" and bytes(dst[:2]) == b"ok"


def test_inline_capacity(pair):
    c0, _, q0, _ = pair
    assert c0._lib.rn_verbs_qp_max_inline(q0._vq) == 28
    assert q0.max_inline == 28
