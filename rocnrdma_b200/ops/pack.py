"""K3 / K5 wrappers: bf16 -> fp8 block-scaled pack fused with GPU-initiated RDMA write,
the receive-side unpack, and the bit-exact PyTorch reference of both."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from .. import _native as N
from .rdma import WAIT_STATUS, _stream_ptr, _device_words, work_stream

TILE_ELEMS = 8192
BLOCK = 32


def record_bytes(chunk_elems: int) -> int:
    b = chunk_elems + chunk_elems // BLOCK
    return (b + 63) // 64 * 64


def staging_bytes(n_elems: int, chunk_elems: int) -> int:
    return (n_elems // chunk_elems) * record_bytes(chunk_elems)


@dataclass
class PackResult:
    status: str
    t_start_ns: int
    t_end_ns: int
    wqes: int
    t_first_post_ns: int
    t_pack_end_ns: int
    n_elems: int
    wire_bytes: int

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    @property
    def device_ns(self) -> int:
        return self.t_end_ns - self.t_start_ns

    @property
    def payload_gbps(self) -> float:
        """fp8 record bytes delivered per second (what crosses the wire)."""
        return self.wire_bytes / max(self.device_ns, 1)

    @property
    def source_gbps(self) -> float:
        """bf16 source bytes consumed per second."""
        return 2 * self.n_elems / max(self.device_ns, 1)


def _parse(view, n_elems, wire) -> PackResult:
    w = (C.c_int64 * 8).from_buffer(view)
    return PackResult(WAIT_STATUS.get(w[0], str(w[0])), w[1], w[2], w[3], w[4], w[5], n_elems, wire)


def pack_fp8_write(ctx, src: torch.Tensor, staging_mr, qp=None, dst_mr=None, chunk_elems: int = 1 << 20,
                   with_imm: bool = False, signal_every: int = 1, grid: int = 0, timeout_ms: int = 2000,
                   stream=None, sync: bool = True, scratch_slot: int = 0, post_only: bool = False, direct: bool = False):
    """Pack ``src`` (bf16) into fp8 chunk records in ``staging_mr`` and, if ``qp`` is given,
    RDMA-write every record to the same offset of ``dst_mr`` from inside the kernel.
    ``direct``: ``staging_mr`` is the *peer's* buffer registered with this context (NVLink-mapped, ``ctx.reg_mr(tensor_on_the_peer)``):
    the kernel's own stores deliver the records and each one is announced by a zero-length RDMA_WRITE_IMM (needs ``with_imm``)."""
    if direct and not (with_imm and qp is not None and dst_mr is not None):
        raise ValueError("direct mode announces records with RDMA_WRITE_IMM: pass qp, dst_mr and with_imm=True")
    assert src.dtype == torch.bfloat16 and src.is_contiguous()
    n = src.numel()
    if n % TILE_ELEMS or chunk_elems % TILE_ELEMS or n % chunk_elems:
        raise ValueError(f"n_elems and chunk_elems must be multiples of {TILE_ELEMS}, n_elems of chunk_elems")
    wire = staging_bytes(n, chunk_elems)
    if staging_mr.length < wire or (dst_mr is not None and dst_mr.length < wire):
        raise ValueError("staging / destination region too small for the records")
    lib = N.load()
    ws = work_stream(ctx, stream)
    n_chunks = n // chunk_elems
    counters = ctx.dev_scratch((n_chunks + 1) * 4 + 64, offset=scratch_slot * (256 << 10))
    out_addr, out_view = ctx.scratch(64, offset=4096 + scratch_slot * 64)
    rc = lib.rn_k_pack_fp8_write(_stream_ptr(ws), grid, src.data_ptr(), staging_mr.addr, n, chunk_elems,
                                 qp.dev_ptr if qp is not None else 0, staging_mr.addr, staging_mr.lkey,
                                 dst_mr.addr if dst_mr is not None else 0, dst_mr.rkey if dst_mr is not None else 0,
                                 int(with_imm) | (2 if post_only else 0) | (4 if direct else 0), signal_every, counters, out_addr, timeout_ms)
    if rc:
        raise N.NativeError(f"pack_fp8_write launch failed ({rc})")
    if not sync:
        return out_view, ws
    ws.synchronize()
    if qp is None:
        return None
    return _parse(out_view, n, wire)


def unpack_fp8(ctx, staging: torch.Tensor, dst: torch.Tensor, chunk_elems: int = 1 << 20, qp=None, grid: int = 0,
               timeout_ms: int = 2000, stream=None, sync: bool = True, scratch_slot: int = 1, ready=None):
    """fp8 chunk records -> bf16.  With ``qp`` the kernel waits for each record's receive
    CQE (RDMA_WRITE_IMM, immediate = chunk id) before touching it.  With ``ready`` (int64 CUDA tensor, one arrival word
    per record, as :func:`~rocnrdma_b200.ops.read_records` and ``recv_consume`` set them) every worker waits for the word of
    the record it is about to read; a word still 0 after ``timeout_ms`` ends the kernel with ``TIMEOUT``.  ``qp`` and
    ``ready`` exclude each other.  ``records_seen``: records announced on the CQ, or, with ``ready``, the words that are
    nonzero when the kernel ends (after a ``TIMEOUT`` that can include records it never waited for or unpacked)."""
    assert dst.dtype == torch.bfloat16 and dst.is_contiguous()
    if (staging.data_ptr() | dst.data_ptr()) & 31:
        raise ValueError("unpack_fp8: records and output must be 32-byte aligned (256-bit loads / stores)")
    n = dst.numel()
    n_chunks = n // chunk_elems
    if qp is not None and ready is not None:
        raise ValueError("unpack_fp8 waits on a receive CQ (qp) or on arrival words (ready), not both")
    ready_addr = 0 if ready is None else _device_words(ready, torch.int64, n_chunks, ctx.device, "ready")
    lib = N.load()
    ws = work_stream(ctx, stream)
    arrived = ctx.dev_scratch((n_chunks + 3) * 4, offset=scratch_slot * (256 << 10))
    out_addr, out_view = ctx.scratch(64, offset=4096 + scratch_slot * 64)
    rc = lib.rn_k_unpack_fp8(_stream_ptr(ws), grid, staging.data_ptr(), dst.data_ptr(), n, chunk_elems,
                             qp.dev_ptr if qp is not None else 0, arrived, out_addr, timeout_ms, ready_addr)
    if rc:
        raise N.NativeError(f"unpack_fp8 launch failed ({rc})")
    if not sync:
        return out_view, ws
    ws.synchronize()
    w = (C.c_int64 * 8).from_buffer(out_view)
    return parse_unpack(out_view)


def parse_unpack(view) -> dict:
    w = (C.c_int64 * 8).from_buffer(view)
    return dict(status=WAIT_STATUS.get(w[0], str(w[0])), device_ns=w[2] - w[1], records_seen=w[3])


# ------------------------------------------------------------------ bit-exact references
# Non-finite rule (the kernels' behaviour, which these references reproduce bit for bit):
#   * the block amax ignores NaN (the kernels reduce with fmaxf), so a NaN stays in its own element and its
#     finite neighbours quantise as if it were absent;
#   * a block holding +-Inf gets exponent 127 (scale byte 254) and multiplier 2^-127 == 0.0, so the Inf becomes
#     NaN and every finite neighbour becomes +-0;
#   * decoding, scale byte 0x00 is 2^-127 (the OCP MX value, an fp32 denormal) and 0xFF is 2^128 == Inf.
def _scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """e = smallest integer with amax / 2^e <= 448, computed on the fp32 bit pattern exactly
    as the kernel does (no log2 rounding)."""
    v = (amax.float() * (1.0 / 448.0)).contiguous()
    bits = v.view(torch.int32)
    e = ((bits >> 23) & 0xFF) - 127 + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    return e.clamp(-127, 127)


def _pow2(e: torch.Tensor) -> torch.Tensor:
    """2^e for e in [-127, 128] from the biased exponent alone: 2^-127 comes out as 0.0, which is what the
    quantiser multiplies by (the kernels' ``inv``).  Decoders use ``ue8m0`` instead."""
    return ((e + 127).to(torch.int32) << 23).view(torch.float32)


def ue8m0(scale_bytes: torch.Tensor) -> torch.Tensor:
    """The fp32 value of UE8M0 scale bytes: 2^(byte - 127), with byte 0x00 = 2^-127 (fp32 0x00400000), 0xFF = Inf."""
    b = scale_bytes.to(torch.int32)
    return torch.where(b == 0, torch.full_like(b, 0x00400000), b << 23).view(torch.float32)


def quantize_blocks(x: torch.Tensor):
    """Block-scaled e4m3 quantisation of fp32 ``x[..., 32]`` (one block per row of the last dim), the rule every
    producer kernel applies: returns (e4m3 bytes shaped like ``x``, UE8M0 scale bytes ``x.shape[:-1]``)."""
    a = x.abs()
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)       # fmaxf drops NaN; +Inf stays
    e = _scale_exponent(a.amax(dim=-1))
    q = (x * _pow2(-e)[..., None]).to(torch.float8_e4m3fn).view(torch.uint8)
    return q, (e + 127).to(torch.uint8)


def ref_pack_fp8(src: torch.Tensor, chunk_elems: int) -> torch.Tensor:
    """Reference chunk records (uint8) for a bf16 tensor; runs on CPU or GPU."""
    q, sc = quantize_blocks(src.float().reshape(-1, BLOCK))
    n = src.numel()
    n_chunks = n // chunk_elems
    rec = record_bytes(chunk_elems)
    out = torch.zeros(n_chunks, rec, dtype=torch.uint8, device=src.device)
    out[:, :chunk_elems] = q.reshape(n_chunks, chunk_elems)
    out[:, chunk_elems:chunk_elems + chunk_elems // BLOCK] = sc.reshape(n_chunks, -1)
    return out.reshape(-1)


def ref_unpack_fp8(records: torch.Tensor, n_elems: int, chunk_elems: int) -> torch.Tensor:
    n_chunks = n_elems // chunk_elems
    rec = record_bytes(chunk_elems)
    r = records.reshape(n_chunks, rec)
    q = r[:, :chunk_elems].contiguous().view(torch.float8_e4m3fn).float().reshape(-1, BLOCK)
    s = ue8m0(r[:, chunk_elems:chunk_elems + chunk_elems // BLOCK].reshape(-1))
    return (q * s[:, None]).to(torch.bfloat16).reshape(-1)
