"""Pure-Python mirror of ``csrc/wire/mlx5_wire.h`` (mlx5 WQE / CQE wire format).

Used by the tier-0 unit tests (no GPU, no NIC: SURVEY.md section 4.3) to check the native
encoders byte for byte, and by tools that want to pretty-print a queue dump.
All multi-byte fields are big-endian on the wire.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import Optional

WQEBB = 64
CQE_SIZE = 64
MAX_INLINE = 28            # largest inline payload: ctrl + raddr + a 4-byte inline header + 28 bytes fill one WQEBB
INLINE_SEG = 0x80000000    # byte_count flag of an inline data segment
MAX_BYTE_COUNT = 0x7FFFFFFF  # largest byte count a gather data segment carries
MAX_MSG = 1 << 30          # longest message, inclusive; a longer WRITE / READ / SEND completes with LOCAL_LENGTH_ERR
MAX_SGE = 2                # scatter-gather entries per WRITE / READ / SEND: ctrl + raddr + two data segments fill one WQEBB

OP_NOP = 0x00
OP_SEND_INVAL = 0x01
OP_RDMA_WRITE = 0x08
OP_RDMA_WRITE_IMM = 0x09
OP_SEND = 0x0A
OP_SEND_IMM = 0x0B
OP_RDMA_READ = 0x10
OP_ATOMIC_CS = 0x11
OP_ATOMIC_FA = 0x12

CTRL_SOLICITED = 0x02
CTRL_CQ_UPDATE = 0x08
CTRL_FENCE = 0x80

CQE_REQ = 0x0
CQE_RESP_WR_IMM = 0x1
CQE_RESP_SEND = 0x2
CQE_RESP_SEND_IMM = 0x3
CQE_RESP_SEND_INV = 0x4
CQE_REQ_ERR = 0xD
CQE_RESP_ERR = 0xE
CQE_INVALID = 0xF

SYNDROMES = {
    0x00: "OK", 0x01: "LOCAL_LENGTH_ERR", 0x02: "LOCAL_QP_OP_ERR", 0x04: "LOCAL_PROT_ERR",
    0x05: "WR_FLUSH_ERR", 0x06: "MW_BIND_ERR", 0x10: "BAD_RESP_ERR", 0x11: "LOCAL_ACCESS_ERR",
    0x12: "REMOTE_INVAL_REQ_ERR", 0x13: "REMOTE_ACCESS_ERR", 0x14: "REMOTE_OP_ERR",
    0x15: "TRANSPORT_RETRY_EXC_ERR", 0x16: "RNR_RETRY_EXC_ERR", 0x22: "REMOTE_ABORTED_ERR",
}
SYN = {v: k for k, v in SYNDROMES.items()}

ACC_LOCAL_WRITE, ACC_REMOTE_WRITE, ACC_REMOTE_READ, ACC_REMOTE_ATOMIC = 1, 2, 4, 8
ACC_ALL = 15

MEM_DEVICE, MEM_HOST_PINNED, MEM_PEER = 0, 1, 2

QPS_RESET, QPS_INIT, QPS_RTR, QPS_RTS, QPS_SQD, QPS_SQE, QPS_ERR = range(7)
QP_STATE_NAMES = ["RESET", "INIT", "RTR", "RTS", "SQD", "SQE", "ERR"]


def ctrl_seg(opcode: int, wqe_idx: int, qpn: int, ds: int, fm_ce_se: int = 0, imm: int = 0, opmod: int = 0) -> bytes:
    w0 = ((opmod & 0xFF) << 24) | ((wqe_idx & 0xFFFF) << 8) | (opcode & 0xFF)
    w1 = ((qpn & 0xFFFFFF) << 8) | (ds & 0x3F)
    return struct.pack(">IIBBBBI", w0, w1, 0, 0, 0, fm_ce_se & 0xFF, imm & 0xFFFFFFFF)


def raddr_seg(raddr: int, rkey: int) -> bytes:
    return struct.pack(">QII", raddr, rkey, 0)


def data_seg(addr: int, lkey: int, nbytes: int) -> bytes:
    """A gather data segment.  A byte count past ``MAX_BYTE_COUNT`` saturates (it then fails as over-long, rather than
    reaching the HCA as a shorter valid message)."""
    return struct.pack(">IIQ", min(nbytes, MAX_BYTE_COUNT), lkey, addr)


def rdma_wqe(opcode, wqe_idx, qpn, laddr, lkey, raddr, rkey, nbytes, fm_ce_se=CTRL_CQ_UPDATE, imm=0) -> bytes:
    """One WQEBB: ctrl + raddr + data, zero padded to 64 bytes (ds = 3)."""
    b = ctrl_seg(opcode, wqe_idx, qpn, 3, fm_ce_se, imm) + raddr_seg(raddr, rkey) + data_seg(laddr, lkey, nbytes)
    return b + bytes(WQEBB - len(b))


def send_wqe(opcode, wqe_idx, qpn, laddr, lkey, nbytes, fm_ce_se=CTRL_CQ_UPDATE, imm=0) -> bytes:
    b = ctrl_seg(opcode, wqe_idx, qpn, 2, fm_ce_se, imm) + data_seg(laddr, lkey, nbytes)
    return b + bytes(WQEBB - len(b))


def _nonempty(sges):
    return [tuple(e) for e in sges if e[2]]


def rdma_sg_wqe(opcode, wqe_idx, qpn, sges, raddr, rkey, fm_ce_se=CTRL_CQ_UPDATE, imm=0) -> bytes:
    """Gather WRITE / WRITE_IMM or scatter READ of up to ``MAX_SGE`` ``(addr, lkey, nbytes)`` entries; the message is
    their concatenation in list order.  Zero-length entries are dropped; two remaining: ctrl + raddr + two data segments
    (ds = 4).  At most one: exactly :func:`rdma_wqe` of it (of entry 0 with 0 bytes when none remains)."""
    e = _nonempty(sges)
    if len(e) < 2:
        a, k, n = e[0] if e else (sges[0][0], sges[0][1], 0)
        return rdma_wqe(opcode, wqe_idx, qpn, a, k, raddr, rkey, n, fm_ce_se, imm)
    return (ctrl_seg(opcode, wqe_idx, qpn, 4, fm_ce_se, imm) + raddr_seg(raddr, rkey)
            + data_seg(e[0][0], e[0][1], e[0][2]) + data_seg(e[1][0], e[1][1], e[1][2]))


def send_sg_wqe(opcode, wqe_idx, qpn, sges, fm_ce_se=CTRL_CQ_UPDATE, imm=0) -> bytes:
    """Gather SEND / SEND_IMM: ctrl + two data segments (ds = 3); at most one non-empty entry: :func:`send_wqe` of it."""
    e = _nonempty(sges)
    if len(e) < 2:
        a, k, n = e[0] if e else (sges[0][0], sges[0][1], 0)
        return send_wqe(opcode, wqe_idx, qpn, a, k, n, fm_ce_se, imm)
    b = ctrl_seg(opcode, wqe_idx, qpn, 3, fm_ce_se, imm) + data_seg(e[0][0], e[0][1], e[0][2]) + data_seg(e[1][0], e[1][1], e[1][2])
    return b + bytes(WQEBB - len(b))


def atomic_seg(swap_add: int, compare: int = 0) -> bytes:
    """The 16-byte atomic segment: big-endian ``swap_add`` (FA: the addend; CS: the swap value), then ``compare``."""
    return struct.pack(">QQ", swap_add & 0xFFFFFFFFFFFFFFFF, compare & 0xFFFFFFFFFFFFFFFF)


def atomic_wqe(opcode, wqe_idx, qpn, laddr, lkey, raddr, rkey, swap_add, compare=0, fm_ce_se=CTRL_CQ_UPDATE,
               nbytes=8) -> bytes:
    """One WQEBB: ctrl + raddr + atomic + data (ds = 4).  FA: ``swap_add`` is the addend and compare is written as 0;
    CS: ``swap_add`` is the swap value.  The data segment names the local 8 bytes that receive the original value."""
    cmp = compare if opcode == OP_ATOMIC_CS else 0
    return (ctrl_seg(opcode, wqe_idx, qpn, 4, fm_ce_se) + raddr_seg(raddr, rkey) + atomic_seg(swap_add, cmp)
            + data_seg(laddr, lkey, nbytes))


def inline_seg(data: bytes) -> bytes:
    """The inline data segment: be32 ``len(data) | INLINE_SEG``, then the payload, zero padded to a 16-byte boundary."""
    b = struct.pack(">I", len(data) | INLINE_SEG) + bytes(data)
    return b + bytes(-len(b) % 16)


def inline_wqe(opcode, wqe_idx, qpn, data: bytes, raddr=0, rkey=0, fm_ce_se=CTRL_CQ_UPDATE, imm=0) -> bytes:
    """One WQEBB carrying ``data`` (1..MAX_INLINE bytes) in the WQE itself.  RDMA_WRITE / WRITE_IMM: ctrl + raddr + inline
    segment (ds 3 up to 12 bytes, else 4); SEND / SEND_IMM: ctrl + inline segment (ds 2 up to 12 bytes, else 3)."""
    if not 1 <= len(data) <= MAX_INLINE:
        raise ValueError(f"inline payload of {len(data)} bytes (1..{MAX_INLINE})")
    seg = inline_seg(data)
    if opcode in (OP_SEND, OP_SEND_IMM):
        b = ctrl_seg(opcode, wqe_idx, qpn, 1 + len(seg) // 16, fm_ce_se, imm) + seg
    else:
        b = ctrl_seg(opcode, wqe_idx, qpn, 2 + len(seg) // 16, fm_ce_se, imm) + raddr_seg(raddr, rkey) + seg
    return b + bytes(WQEBB - len(b))


def _inline_payload(b: bytes, off: int, ds: int, head_segs: int) -> bytes:
    n = struct.unpack_from(">I", b, off - 4)[0] & ~INLINE_SEG
    if not 1 <= n <= MAX_INLINE or ds != head_segs + (4 + n + 15) // 16:
        raise ValueError(f"malformed inline WQE: {n} bytes with ds = {ds}")
    return bytes(b[off:off + n])


@dataclass
class WqeView:
    opcode: int
    opmod: int
    wqe_idx: int
    qpn: int
    ds: int
    fm_ce_se: int
    imm: int
    raddr: int = 0
    rkey: int = 0
    laddr: int = 0
    lkey: int = 0
    nbytes: int = 0
    swap_add: int = 0
    compare: int = 0
    inline_data: Optional[bytes] = None    # the payload of an inline WQE (laddr / lkey are then 0)
    sges: Optional[list] = None            # WRITE / READ / SEND: the (addr, lkey, nbytes) entries; nbytes above is their total


def _second_seg(b: bytes, off: int, v: WqeView):
    n, lkey, addr = struct.unpack_from(">IIQ", b, off)
    if n & INLINE_SEG:
        raise ValueError("the second data segment of a scatter-gather list cannot be inline")
    v.sges.append((addr, lkey, n))
    v.nbytes += n


def decode_wqe(b: bytes) -> WqeView:
    """Decode one WQEBB.  An inline WQE (INLINE_SEG set on a WRITE, WRITE_IMM, SEND or SEND_IMM) fills ``inline_data``;
    one whose length or ds is out of range raises ``ValueError``, as does the flag on a READ.  A WRITE, READ or SEND fills
    ``sges``: two entries for RDMA ds = 4 or SEND ds = 3, whose second segment must not carry the inline flag."""
    assert len(b) >= WQEBB
    w0, w1, _sig, _r0, _r1, fm, imm = struct.unpack_from(">IIBBBBI", b, 0)
    v = WqeView(opcode=w0 & 0xFF, opmod=w0 >> 24, wqe_idx=(w0 >> 8) & 0xFFFF, qpn=w1 >> 8, ds=w1 & 0x3F,
                fm_ce_se=fm, imm=imm)
    if v.opcode in (OP_RDMA_WRITE, OP_RDMA_WRITE_IMM, OP_RDMA_READ) and struct.unpack_from(">I", b, 32)[0] & INLINE_SEG:
        if v.opcode == OP_RDMA_READ:
            raise ValueError("a READ cannot carry inline data")
        v.raddr, v.rkey, _ = struct.unpack_from(">QII", b, 16)
        v.inline_data = _inline_payload(b, 36, v.ds, 2)
        v.nbytes = len(v.inline_data)
    elif v.opcode in (OP_SEND, OP_SEND_IMM) and struct.unpack_from(">I", b, 16)[0] & INLINE_SEG:
        v.inline_data = _inline_payload(b, 20, v.ds, 1)
        v.nbytes = len(v.inline_data)
    elif v.opcode in (OP_RDMA_WRITE, OP_RDMA_WRITE_IMM, OP_RDMA_READ):
        v.raddr, v.rkey, _ = struct.unpack_from(">QII", b, 16)
        n, v.lkey, v.laddr = struct.unpack_from(">IIQ", b, 32)
        v.nbytes = n & 0x7FFFFFFF
        v.sges = [(v.laddr, v.lkey, v.nbytes)]
        if v.ds == 4:
            _second_seg(b, 48, v)
    elif v.opcode in (OP_ATOMIC_CS, OP_ATOMIC_FA):
        v.raddr, v.rkey, _ = struct.unpack_from(">QII", b, 16)
        v.swap_add, v.compare = struct.unpack_from(">QQ", b, 32)
        n, v.lkey, v.laddr = struct.unpack_from(">IIQ", b, 48)
        v.nbytes = n & 0x7FFFFFFF
    elif v.opcode in (OP_SEND, OP_SEND_IMM):
        n, v.lkey, v.laddr = struct.unpack_from(">IIQ", b, 16)
        v.nbytes = n & 0x7FFFFFFF
        v.sges = [(v.laddr, v.lkey, v.nbytes)]
        if v.ds == 3:
            _second_seg(b, 32, v)
    return v


@dataclass
class CqeView:
    opcode: int
    owner: int
    wqe_counter: int
    qpn: int
    wqe_opcode: int
    byte_cnt: int
    imm: int
    syndrome: int
    vendor_synd: int

    @property
    def is_error(self) -> bool:
        return self.opcode in (CQE_REQ_ERR, CQE_RESP_ERR)


def cqe(opcode, owner, wqe_counter, qpn, wqe_opcode=0, byte_cnt=0, imm=0, syndrome=0, timestamp=0) -> bytes:
    b = bytearray(CQE_SIZE)
    err = opcode in (CQE_REQ_ERR, CQE_RESP_ERR)
    if not err:
        struct.pack_into(">I", b, 36, imm)
        struct.pack_into(">I", b, 44, byte_cnt)
        struct.pack_into(">II", b, 48, (timestamp >> 32) & 0xFFFFFFFF, timestamp & 0xFFFFFFFF)
    else:
        b[54] = 0
        b[55] = syndrome
    struct.pack_into(">I", b, 56, ((wqe_opcode & 0xFF) << 24) | (qpn & 0xFFFFFF))
    struct.pack_into(">H", b, 60, wqe_counter & 0xFFFF)
    b[63] = ((opcode & 0xF) << 4) | (owner & 1)
    return bytes(b)


def decode_cqe(b: bytes) -> CqeView:
    assert len(b) >= CQE_SIZE
    op_own = b[63]
    opcode = op_own >> 4
    sq, = struct.unpack_from(">I", b, 56)
    wc, = struct.unpack_from(">H", b, 60)
    err = opcode in (CQE_REQ_ERR, CQE_RESP_ERR)
    return CqeView(opcode=opcode, owner=op_own & 1, wqe_counter=wc, qpn=sq & 0xFFFFFF, wqe_opcode=sq >> 24,
                   byte_cnt=0 if err else struct.unpack_from(">I", b, 44)[0],
                   imm=0 if err else struct.unpack_from(">I", b, 36)[0],
                   syndrome=b[55] if err else 0, vendor_synd=b[54] if err else 0)


def cqe_valid(op_own: int, ci: int, log_n: int) -> bool:
    return (op_own >> 4) != CQE_INVALID and (op_own & 1) == ((ci >> log_n) & 1)


def doorbell_value(wqe_idx: int, qpn: int) -> int:
    """The 8 bytes stored to the doorbell register, as the little-endian u64 the GPU writes."""
    lo = struct.unpack("<I", struct.pack(">I", ((wqe_idx & 0xFFFF) << 8) | OP_NOP))[0]
    hi = struct.unpack("<I", struct.pack(">I", (qpn & 0xFFFFFF) << 8))[0]
    return lo | (hi << 32)


def expand16(counter16: int, near: int) -> int:
    """Expand a 16-bit wire counter to the 64-bit index closest above ``near``."""
    return near + ((counter16 - near) & 0xFFFF)
