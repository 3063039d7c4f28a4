"""Tier-0 (no GPU, no NIC): byte-exact mlx5 WQE / CQE layouts, native vs Python mirror."""
import ctypes as C
import struct

import pytest

from rocnrdma_b200 import wire as W


def test_segment_sizes_and_wqebb():
    assert len(W.ctrl_seg(W.OP_RDMA_WRITE, 1, 2, 3)) == 16
    assert len(W.raddr_seg(0, 0)) == 16
    assert len(W.data_seg(0, 0, 0)) == 16
    assert len(W.rdma_wqe(W.OP_RDMA_WRITE, 0, 0, 0, 0, 0, 0, 0)) == 64
    assert len(W.send_wqe(W.OP_SEND, 0, 0, 0, 0, 0)) == 64
    assert len(W.cqe(W.CQE_REQ, 0, 0, 0)) == 64


def test_ctrl_segment_bytes_are_big_endian():
    b = W.ctrl_seg(W.OP_RDMA_WRITE, wqe_idx=0x1234, qpn=0xABCDEF, ds=3, fm_ce_se=W.CTRL_CQ_UPDATE, imm=0xDEADBEEF)
    # opmod | idx hi | idx lo | opcode ; qpn[23:0] | ds ; sig rsvd rsvd fm_ce_se ; imm
    assert b == bytes([0x00, 0x12, 0x34, 0x08, 0xAB, 0xCD, 0xEF, 0x03, 0, 0, 0, 0x08, 0xDE, 0xAD, 0xBE, 0xEF])


def test_rdma_wqe_field_offsets():
    w = W.rdma_wqe(W.OP_RDMA_READ, 7, 0x100, laddr=0x1122334455667788, lkey=0xA1A2A3A4,
                   raddr=0x99AABBCCDDEEFF00, rkey=0xB1B2B3B4, nbytes=0x01020304)
    assert w[16:24] == bytes.fromhex("99aabbccddeeff00")     # raddr be64
    assert w[24:28] == bytes.fromhex("b1b2b3b4")             # rkey
    assert w[32:36] == bytes.fromhex("01020304")             # byte_count
    assert w[36:40] == bytes.fromhex("a1a2a3a4")             # lkey
    assert w[40:48] == bytes.fromhex("1122334455667788")     # laddr be64
    assert w[48:] == bytes(16)
    v = W.decode_wqe(w)
    assert (v.opcode, v.wqe_idx, v.qpn, v.ds) == (W.OP_RDMA_READ, 7, 0x100, 3)
    assert (v.laddr, v.lkey, v.raddr, v.rkey, v.nbytes) == (0x1122334455667788, 0xA1A2A3A4, 0x99AABBCCDDEEFF00,
                                                            0xB1B2B3B4, 0x01020304)


def test_send_wqe_has_two_segments():
    w = W.send_wqe(W.OP_SEND_IMM, 0xFFFF, 5, laddr=0x10, lkey=0x20, nbytes=0x30, imm=0x55)
    v = W.decode_wqe(w)
    assert v.ds == 2 and v.wqe_idx == 0xFFFF and v.imm == 0x55 and (v.laddr, v.lkey, v.nbytes) == (0x10, 0x20, 0x30)


def test_cqe_layout_and_owner_bit():
    c = W.cqe(W.CQE_REQ, owner=1, wqe_counter=0xBEEF, qpn=0x123456, wqe_opcode=W.OP_RDMA_WRITE, byte_cnt=4096, imm=9)
    assert c[63] == 0x01 and c[60:62] == b"\xbe\xef"
    assert c[56:60] == bytes([W.OP_RDMA_WRITE, 0x12, 0x34, 0x56])
    assert struct.unpack_from(">I", c, 44)[0] == 4096
    v = W.decode_cqe(c)
    assert not v.is_error and v.wqe_counter == 0xBEEF and v.qpn == 0x123456 and v.byte_cnt == 4096 and v.imm == 9
    e = W.cqe(W.CQE_REQ_ERR, owner=0, wqe_counter=3, qpn=1, syndrome=W.SYN["REMOTE_ACCESS_ERR"])
    ve = W.decode_cqe(e)
    assert ve.is_error and ve.syndrome == 0x13 and e[55] == 0x13 and e[63] == 0xD0


@pytest.mark.parametrize("log_n", [1, 4, 10])
def test_cqe_validity_across_passes(log_n):
    n = 1 << log_n
    invalid = (W.CQE_INVALID << 4) | 1
    for ci in (0, n - 1, n, 2 * n - 1, 2 * n, 5 * n + 1):
        parity = (ci >> log_n) & 1
        assert not W.cqe_valid(invalid, ci, log_n)
        assert W.cqe_valid((W.CQE_REQ << 4) | parity, ci, log_n)
        assert not W.cqe_valid((W.CQE_REQ << 4) | (parity ^ 1), ci, log_n)


def test_doorbell_value_and_counter_expansion():
    v = W.doorbell_value(0x0102, 0x000100)
    assert v.to_bytes(8, "little") == bytes([0x00, 0x01, 0x02, 0x00, 0x00, 0x01, 0x00, 0x00])
    assert W.expand16(0x0005, near=0x1FFFE) == 0x20005
    assert W.expand16(0xFFFF, near=0xFFFF) == 0xFFFF
    assert W.expand16(0x0000, near=0xFFFF) == 0x10000


def test_native_struct_sizes_match():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    out = (C.c_uint32 * 8)()
    n = lib.rn_abi_sizes(out, 8)
    assert n == 8
    wqe, cqe, mkey, resolved = out[0], out[1], out[2], out[3]
    assert (wqe, cqe, mkey, resolved) == (64, 64, 48, 64)


def test_native_encoder_matches_python_mirror():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    if not hasattr(lib, "rn_wire_build_wqe"):
        pytest.skip("wire test hooks not built")
    buf = (C.c_uint8 * 64)()
    for (op, idx, qpn, la, lk, ra, rk, nb, fl, imm) in [
        (W.OP_RDMA_WRITE, 0, 0x100, 0x7F0000001000, 0x101, 0x7F0000002000, 0x201, 4096, W.CTRL_CQ_UPDATE, 0),
        (W.OP_RDMA_READ, 0xFFFF, 0xFFFFFF, 2 ** 63 + 5, 0xFFFFFFFF, 2 ** 64 - 1, 1, 0x7FFFFFFF, 0, 0),
        (W.OP_RDMA_WRITE_IMM, 77, 9, 16, 2, 32, 3, 0, W.CTRL_CQ_UPDATE | W.CTRL_FENCE, 0xCAFEF00D),
    ]:
        lib.rn_wire_build_wqe(buf, op, idx, qpn, la, lk, ra, rk, nb, fl, imm)
        assert bytes(buf) == W.rdma_wqe(op, idx, qpn, la, lk, ra, rk, nb, fl, imm)
    lib.rn_wire_build_wqe(buf, W.OP_SEND, 3, 0x100, 0x1000, 0x5, 0, 0, 100, W.CTRL_CQ_UPDATE, 0)
    assert bytes(buf) == W.send_wqe(W.OP_SEND, 3, 0x100, 0x1000, 0x5, 100)


@pytest.mark.parametrize("nb", [W.MAX_MSG, W.MAX_MSG + 1, 2**31 - 1, 2**31, 2**31 + 64, 2**32 - 16, 2**32 - 1])
@pytest.mark.parametrize("op", [W.OP_RDMA_WRITE, W.OP_RDMA_READ, W.OP_SEND])
def test_byte_counts_past_31_bits_saturate(op, nb):
    """A byte count the data segment cannot carry is posted as 2^31 - 1 -- longer than any message, so it fails at the
    HCA -- never as its low 31 bits (2^31 + 64 would be a valid 64-byte message, 2^31 an empty one).  Both encoders."""
    from rocnrdma_b200 import _native as N
    lib = N.load()
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_wqe(buf, op, 1, 0x100, 0x1000, 0x5, 0x2000, 0x6, nb, W.CTRL_CQ_UPDATE, 0)
    want = (W.send_wqe(op, 1, 0x100, 0x1000, 0x5, nb) if op == W.OP_SEND else
            W.rdma_wqe(op, 1, 0x100, 0x1000, 0x5, 0x2000, 0x6, nb))
    assert bytes(buf) == want
    sent = W.decode_wqe(bytes(buf)).nbytes
    assert sent == min(nb, W.MAX_BYTE_COUNT) and (sent > W.MAX_MSG) == (nb > W.MAX_MSG)


@pytest.mark.parametrize("op", [W.CQE_REQ, W.CQE_RESP_WR_IMM, W.CQE_RESP_SEND, W.CQE_RESP_SEND_IMM, W.CQE_REQ_ERR,
                                W.CQE_RESP_ERR])
def test_native_cqe_encoder_matches_python_mirror(op):
    """The CQE encoder the engine and the mock ConnectX share writes wire.cqe()'s bytes.  An error CQE keeps only the
    syndromes where a good one has imm, byte_cnt and the timestamp: every other byte of it is reserved and zero."""
    from rocnrdma_b200 import _native as N
    lib = N.load()
    buf = (C.c_uint8 * 64)()
    err = op in (W.CQE_REQ_ERR, W.CQE_RESP_ERR)
    for owner, ctr, qpn, wop, bc, imm, syn, ts in [
        (0, 0, 0, 0, 0, 0, 0, 0),
        (1, 0xBEEF, 0x123456, W.OP_RDMA_WRITE, 4096, 9, W.SYN["REMOTE_ACCESS_ERR"], 0x0102030405060708),
        (1, 0xFFFF, 0xFFFFFF, 0xFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFF, 2 ** 64 - 1),
    ]:
        lib.rn_wire_build_cqe(buf, op, owner, ctr, qpn, wop, bc, imm, syn, 0, ts)
        assert bytes(buf) == W.cqe(op, owner, ctr, qpn, wop, bc, imm, syn, ts)
        lib.rn_wire_build_cqe(buf, op, owner, ctr, qpn, wop, bc, imm, syn, 0x5A, ts)
        if err:    # the vendor syndrome is byte 54; every byte before it stays zero
            assert bytes(buf)[:56] == bytes(54) + bytes([0x5A, syn])
        else:      # a good CQE carries no syndrome
            assert bytes(buf) == W.cqe(op, owner, ctr, qpn, wop, bc, imm, syn, ts)
