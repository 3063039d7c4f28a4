"""8-byte RDMA atomics on the wire: exact WQE bytes from the Python mirror, decode round trips, and the native
encoder / decoder (csrc/wire/mlx5_wire.h) against the mirror byte for byte."""
import ctypes as C
import struct

import pytest

from rocnrdma_b200 import wire as W


def test_fetch_add_wqe_bytes():
    w = W.atomic_wqe(W.OP_ATOMIC_FA, 0x0102, 0x0A0B0C, laddr=0x1122334455667788, lkey=0x00000101,
                     raddr=0x7F0000001000, rkey=0x00000202, swap_add=5, compare=0xDEAD)
    assert len(w) == 64
    # ctrl: opmod | idx | opcode, qpn | ds = 4, sig/rsvd/fm_ce_se, imm
    assert w[0:16] == bytes([0x00, 0x01, 0x02, 0x12, 0x0A, 0x0B, 0x0C, 0x04, 0, 0, 0, 0x08, 0, 0, 0, 0])
    # raddr segment
    assert w[16:32] == bytes.fromhex("00007f0000001000" "00000202" "00000000")
    # atomic segment: addend in swap_add, compare written as zero for FA
    assert w[32:48] == bytes.fromhex("0000000000000005" "0000000000000000")
    # data segment: 8 bytes at laddr
    assert w[48:64] == bytes.fromhex("00000008" "00000101" "1122334455667788")


def test_compare_swap_wqe_bytes():
    w = W.atomic_wqe(W.OP_ATOMIC_CS, 7, 0x100, laddr=0x2000, lkey=3, raddr=0x3000, rkey=4, swap_add=0x0102030405060708,
                     compare=0x1112131415161718, fm_ce_se=0)
    assert w[3] == 0x11 and w[7] == 0x04 and w[11] == 0
    assert w[32:48] == bytes.fromhex("0102030405060708" "1112131415161718")
    assert struct.unpack(">I", w[48:52])[0] == 8


@pytest.mark.parametrize("op", [W.OP_ATOMIC_FA, W.OP_ATOMIC_CS])
def test_decode_round_trip(op):
    w = W.atomic_wqe(op, 0xFFFF, 0xFFFFFF, 2 ** 63 + 8, 0xFFFFFFFF, 2 ** 64 - 8, 1, 2 ** 64 - 1, 0x8000000000000001)
    v = W.decode_wqe(w)
    assert (v.opcode, v.wqe_idx, v.qpn, v.ds) == (op, 0xFFFF, 0xFFFFFF, 4)
    assert (v.laddr, v.lkey, v.raddr, v.rkey, v.nbytes) == (2 ** 63 + 8, 0xFFFFFFFF, 2 ** 64 - 8, 1, 8)
    assert v.swap_add == 2 ** 64 - 1
    assert v.compare == (0x8000000000000001 if op == W.OP_ATOMIC_CS else 0)


CASES = [
    (W.OP_ATOMIC_FA, 0, 0x100, 0x7F0000001000, 0x101, 0x7F0000002000, 0x201, 1, 0, W.CTRL_CQ_UPDATE),
    (W.OP_ATOMIC_FA, 0xFFFF, 0xFFFFFF, 2 ** 63 + 8, 0xFFFFFFFF, 2 ** 64 - 8, 1, 2 ** 64 - 1, 77, 0),
    (W.OP_ATOMIC_CS, 77, 9, 16, 2, 32, 3, 0x0102030405060708, 0xCAFEF00DDEADBEEF, W.CTRL_CQ_UPDATE | W.CTRL_FENCE),
    (W.OP_ATOMIC_CS, 1, 1, 8, 8, 8, 8, 0, 0, W.CTRL_CQ_UPDATE),
]


def test_native_encoder_matches_python_mirror():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    buf = (C.c_uint8 * 64)()
    for (op, idx, qpn, la, lk, ra, rk, sa, cmp, fl) in CASES:
        lib.rn_wire_build_atomic_wqe(buf, op, idx, qpn, la, lk, ra, rk, sa, cmp, fl)
        assert bytes(buf) == W.atomic_wqe(op, idx, qpn, la, lk, ra, rk, sa, cmp, fl)


def test_native_decoder_reads_the_mirror():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    out = (C.c_uint64 * 13)()
    for (op, idx, qpn, la, lk, ra, rk, sa, cmp, fl) in CASES:
        b = (C.c_uint8 * 64)(*W.atomic_wqe(op, idx, qpn, la, lk, ra, rk, sa, cmp, fl))
        assert lib.rn_wire_decode_wqe(b, out) == 1
        assert list(out) == [op, idx, qpn, 4, fl, 0, ra, rk, la, lk, 8, sa, cmp if op == W.OP_ATOMIC_CS else 0]
    # an atomic must span four segments: ds = 3 is malformed (the engine completes it with LOCAL_QP_OP_ERR)
    bad = bytearray(W.atomic_wqe(W.OP_ATOMIC_FA, 0, 1, 8, 1, 8, 1, 1))
    bad[7] = 3
    assert lib.rn_wire_decode_wqe((C.c_uint8 * 64)(*bad), out) == 0
