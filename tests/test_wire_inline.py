"""Inline WQEs on the wire: exact bytes from the Python mirror, the native encoder against the mirror, decode round trips
through both decoders, and the malformed inline WQEs the decoders refuse (csrc/wire/mlx5_wire.h)."""
import ctypes as C
import struct

import pytest

from rocnrdma_b200 import wire as W

PAYLOAD = bytes(range(0xA0, 0xA0 + 28))


@pytest.mark.parametrize("n,ds", [(1, 3), (8, 3), (12, 3), (13, 4), (28, 4)])
def test_write_inline_wqe_bytes(n, ds):
    data = PAYLOAD[:n]
    w = W.inline_wqe(W.OP_RDMA_WRITE, 0x0102, 0x0A0B0C, data, raddr=0x7F0000001003, rkey=0x00000202)
    assert len(w) == 64
    assert w[0:16] == bytes([0x00, 0x01, 0x02, 0x08, 0x0A, 0x0B, 0x0C, ds, 0, 0, 0, 0x08, 0, 0, 0, 0])
    assert w[16:32] == bytes.fromhex("00007f0000001003" "00000202" "00000000")
    assert w[32:36] == struct.pack(">I", 0x80000000 | n)
    assert w[36:36 + n] == data
    assert w[36 + n:] == bytes(28 - n)


@pytest.mark.parametrize("n,ds", [(12, 2), (13, 3)])
def test_send_inline_wqe_bytes(n, ds):
    data = PAYLOAD[:n]
    w = W.inline_wqe(W.OP_SEND_IMM, 5, 0x100, data, fm_ce_se=0, imm=0xCAFEF00D)
    assert w[0:16] == bytes([0, 0, 5, 0x0B, 0, 1, 0, ds, 0, 0, 0, 0, 0xCA, 0xFE, 0xF0, 0x0D])
    assert w[16:20] == struct.pack(">I", 0x80000000 | n)
    assert w[20:20 + n] == data
    assert w[20 + n:] == bytes(44 - n)


def test_mirror_refuses_empty_and_oversized_payloads():
    for data in (b"", bytes(29)):
        with pytest.raises(ValueError):
            W.inline_wqe(W.OP_RDMA_WRITE, 0, 1, data)


CASES = [(op, n) for op in (W.OP_RDMA_WRITE, W.OP_RDMA_WRITE_IMM, W.OP_SEND, W.OP_SEND_IMM) for n in (1, 7, 12, 13, 27, 28)]


def _native_build(lib, op, idx, qpn, ra, rk, data, fl, imm):
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_inline_wqe(buf, op, idx, qpn, ra, rk, (C.c_uint8 * len(data))(*data), len(data), fl, imm)
    return bytes(buf)


def test_native_encoder_matches_python_mirror():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    for k, (op, n) in enumerate(CASES):
        data = PAYLOAD[k % 3:k % 3 + n] if n < 28 else PAYLOAD
        ra, rk = (2 ** 64 - 1 - k, 0xFFFFFFFF - k) if op in (W.OP_RDMA_WRITE, W.OP_RDMA_WRITE_IMM) else (0, 0)
        fl = [0, W.CTRL_CQ_UPDATE, W.CTRL_CQ_UPDATE | W.CTRL_FENCE][k % 3]
        assert _native_build(lib, op, 0xFFFF - k, 0xFFFFFF - k, ra, rk, data, fl, 0x01020304 + k) == \
            W.inline_wqe(op, 0xFFFF - k, 0xFFFFFF - k, data, ra, rk, fl, 0x01020304 + k)


@pytest.mark.parametrize("op,n", CASES)
def test_decode_round_trip(op, n):
    from rocnrdma_b200 import _native as N
    lib = N.load()
    data = PAYLOAD[28 - n:]
    rdma = op in (W.OP_RDMA_WRITE, W.OP_RDMA_WRITE_IMM)
    ra, rk = (0x1122334455667788, 0x0A0B0C0D) if rdma else (0, 0)
    w = W.inline_wqe(op, 77, 0x4242, data, ra, rk, W.CTRL_CQ_UPDATE, 9)
    v = W.decode_wqe(w)
    assert v.inline_data == data and v.nbytes == n
    assert (v.opcode, v.wqe_idx, v.qpn, v.raddr, v.rkey, v.laddr, v.lkey) == (op, 77, 0x4242, ra, rk, 0, 0)
    out = (C.c_uint64 * 15)()
    assert lib.rn_wire_decode_wqe_inline((C.c_uint8 * 64)(*w), out) == 1
    off = 36 if rdma else 20
    assert list(out) == [op, 77, 0x4242, v.ds, W.CTRL_CQ_UPDATE, 9, ra, rk, 0, 0, n, 0, 0, 1, off]
    assert w[off:off + n] == data
    # the 13-field hook is unchanged and still reads the WQE
    out13 = (C.c_uint64 * 13)()
    assert lib.rn_wire_decode_wqe((C.c_uint8 * 64)(*w), out13) == 1 and list(out13) == list(out)[:13]


def test_gather_wqes_decode_as_not_inline():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    out = (C.c_uint64 * 15)()
    for w in (W.rdma_wqe(W.OP_RDMA_WRITE, 1, 2, 0x1000, 3, 0x2000, 4, 64), W.send_wqe(W.OP_SEND, 1, 2, 0x1000, 3, 12),
              W.rdma_wqe(W.OP_RDMA_READ, 1, 2, 0x1000, 3, 0x2000, 4, 8), W.atomic_wqe(W.OP_ATOMIC_FA, 1, 2, 8, 3, 16, 4, 1)):
        assert lib.rn_wire_decode_wqe_inline((C.c_uint8 * 64)(*w), out) == 1
        assert list(out)[13:] == [0, 0]
        assert W.decode_wqe(w).inline_data is None


def _with_count(w, off, word):
    b = bytearray(w)
    b[off:off + 4] = struct.pack(">I", word)
    return bytes(b)


def _with_ds(w, ds):
    b = bytearray(w)
    b[7] = ds
    return bytes(b)


def _bad_wqes():
    wr = W.inline_wqe(W.OP_RDMA_WRITE, 3, 5, b"12345678", 0x1000, 7)
    sd = W.inline_wqe(W.OP_SEND, 3, 5, b"12345678")
    return {
        "write_n0": _with_count(wr, 32, 0x80000000),
        "write_n29": _with_ds(_with_count(wr, 32, 0x80000000 | 29), 4),
        "write_ds4_for_8_bytes": _with_ds(wr, 4),
        "write_ds3_for_13_bytes": _with_ds(W.inline_wqe(W.OP_RDMA_WRITE_IMM, 3, 5, bytes(13), 0x1000, 7), 3),
        "send_n0": _with_count(sd, 16, 0x80000000),
        "send_ds3_for_8_bytes": _with_ds(sd, 3),
        "read_inline": _with_count(W.rdma_wqe(W.OP_RDMA_READ, 3, 5, 0x1000, 1, 0x2000, 7, 8), 32, 0x80000000 | 8),
        "fetch_add_inline": _with_count(W.atomic_wqe(W.OP_ATOMIC_FA, 3, 5, 8, 1, 16, 7, 1), 48, 0x80000000 | 8),
    }


@pytest.mark.parametrize("case", list(_bad_wqes()))
def test_native_decoder_rejects_malformed_inline(case):
    from rocnrdma_b200 import _native as N
    lib = N.load()
    w = _bad_wqes()[case]
    assert lib.rn_wire_decode_wqe_inline((C.c_uint8 * 64)(*w), (C.c_uint64 * 15)()) == 0
    assert lib.rn_wire_decode_wqe((C.c_uint8 * 64)(*w), (C.c_uint64 * 13)()) == 0
    if case != "fetch_add_inline":         # the mirror checks inline segments of the opcodes that may carry one
        with pytest.raises(ValueError):
            W.decode_wqe(w)
