"""Property tests (hypothesis): the C encoders / decoders the engine and the posters use (csrc/wire/mlx5_wire.h,
reached through the CPU test hooks) agree with the Python mirror on EVERY field value, not just on hand-picked ones.
Byte counts range over all 32 bits: one the data segment cannot carry saturates at 2^31 - 1 in both encoders."""
import ctypes as C

import pytest
from hypothesis import given, settings, strategies as st

from rocnrdma_b200 import _native as N, wire as W

u8, u16, u24, u31, u32, u64 = (st.integers(0, (1 << b) - 1) for b in (8, 16, 24, 31, 32, 64))
rdma_ops = st.sampled_from([W.OP_RDMA_WRITE, W.OP_RDMA_WRITE_IMM, W.OP_RDMA_READ])
send_ops = st.sampled_from([W.OP_SEND, W.OP_SEND_IMM])
flags = st.sampled_from([0, W.CTRL_CQ_UPDATE, W.CTRL_FENCE, W.CTRL_CQ_UPDATE | W.CTRL_FENCE])


@pytest.fixture(scope="module")
def lib():
    lib = N.load()
    if not hasattr(lib, "rn_wire_build_wqe"):
        pytest.skip("wire test hooks not built")
    return lib


@settings(max_examples=300, deadline=None)
@given(op=rdma_ops, idx=u16, qpn=u24, la=u64, lk=u32, ra=u64, rk=u32, nb=st.one_of(u31, u32), fl=flags, imm=u32)
def test_rdma_wqe_bytes_and_roundtrip(lib, op, idx, qpn, la, lk, ra, rk, nb, fl, imm):
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_wqe(buf, op, idx, qpn, la, lk, ra, rk, nb, fl, imm)
    raw = bytes(buf)
    assert raw == W.rdma_wqe(op, idx, qpn, la, lk, ra, rk, nb, fl, imm)
    v = W.decode_wqe(raw)
    assert (v.opcode, v.wqe_idx, v.qpn, v.laddr, v.lkey, v.raddr, v.rkey, v.fm_ce_se) == (op, idx, qpn, la, lk, ra, rk, fl)
    assert v.nbytes == min(nb, W.MAX_BYTE_COUNT)
    assert v.ds == 3
    if op == W.OP_RDMA_WRITE_IMM:
        assert v.imm == imm


@settings(max_examples=200, deadline=None)
@given(op=send_ops, idx=u16, qpn=u24, la=u64, lk=u32, nb=st.one_of(u31, u32), fl=flags, imm=u32)
def test_send_wqe_bytes_and_roundtrip(lib, op, idx, qpn, la, lk, nb, fl, imm):
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_wqe(buf, op, idx, qpn, la, lk, 0, 0, nb, fl, imm)
    raw = bytes(buf)
    assert raw == W.send_wqe(op, idx, qpn, la, lk, nb, fl, imm)
    v = W.decode_wqe(raw)
    assert (v.opcode, v.wqe_idx, v.qpn, v.laddr, v.lkey, v.nbytes, v.fm_ce_se, v.ds) == (op, idx, qpn, la, lk, min(nb, W.MAX_BYTE_COUNT),
                                                                                        fl, 2)


good_cqe_ops = st.sampled_from([W.CQE_REQ, W.CQE_RESP_WR_IMM, W.CQE_RESP_SEND, W.CQE_RESP_SEND_IMM])
err_cqe_ops = st.sampled_from([W.CQE_REQ_ERR, W.CQE_RESP_ERR])


@settings(max_examples=300, deadline=None)
@given(op=st.one_of(good_cqe_ops, err_cqe_ops), owner=st.integers(0, 1), ctr=u16, qpn=u24, wop=u8, bc=u32, imm=u32, syn=u8, ts=u64,
       vendor=u8)
def test_cqe_decoders_agree(lib, op, owner, ctr, qpn, wop, bc, imm, syn, ts, vendor):
    """The native encoder writes wire.cqe()'s bytes, and both decoders read them back."""
    raw = W.cqe(op, owner, ctr, qpn, wop, bc, imm, syn, ts)
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_cqe(buf, op, owner, ctr, qpn, wop, bc, imm, syn, vendor, ts)
    # the vendor syndrome (byte 54, which wire.cqe leaves 0) is the only byte the Python mirror does not model
    want = raw[:54] + bytes([vendor]) + raw[55:] if op in (W.CQE_REQ_ERR, W.CQE_RESP_ERR) else raw
    assert bytes(buf) == want
    wc = N.RnWc()
    assert lib.rn_wire_decode_cqe((C.c_uint8 * 64)(*raw), C.byref(wc)) == 0
    py = W.decode_cqe(raw)
    assert (wc.qpn, wc.wqe_counter, wc.opcode, wc.wqe_opcode, bool(wc.is_error)) == (py.qpn, py.wqe_counter, py.opcode, py.wqe_opcode, py.is_error)
    assert (py.qpn, py.wqe_counter, py.opcode, py.owner, py.wqe_opcode) == (qpn, ctr, op, owner, wop)
    if py.is_error:
        assert wc.syndrome == py.syndrome == syn
    else:
        assert (wc.byte_cnt, wc.imm) == (py.byte_cnt, py.imm) == (bc, imm)


@settings(max_examples=300, deadline=None)
@given(log_n=st.integers(1, 16), ci=st.integers(0, (1 << 24) - 1), op=good_cqe_ops)
def test_owner_bit_tracks_the_pass_over_the_ring(log_n, ci, op):
    """A CQE written for consumer index ci is valid exactly for the pass it was produced in (mlx5 ownership rule)."""
    owner = (ci >> log_n) & 1
    op_own = (op << 4) | owner
    assert W.cqe_valid(op_own, ci, log_n)
    assert not W.cqe_valid(op_own, ci + (1 << log_n), log_n)        # next pass over the same slot: stale
    assert not W.cqe_valid((W.CQE_INVALID << 4) | owner, ci, log_n)


@settings(max_examples=300, deadline=None)
@given(near=st.integers(0, 1 << 48), ahead=st.integers(0, 0xFFFF))
def test_sixteen_bit_counters_expand_to_the_right_index(near, ahead):
    full = near + ahead
    assert W.expand16(full & 0xFFFF, near) == full
