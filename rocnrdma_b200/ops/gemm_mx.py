"""K7 wrapper: block-scaled fp8 GEMM (e4m3 ``wgmma`` per 32-deep MX block, scales applied in registers) whose operands are the records
the send side produces -- so a receiver multiplies straight out of its receive buffer."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from .. import _native as N
from .pack import BLOCK, _pow2, _scale_exponent, record_bytes
from .rdma import WAIT_STATUS, _stream_ptr, work_stream

PANEL_ROWS = 128


@dataclass
class MxOperand:
    """An fp8 operand [rows, K] with UE8M0 block scales [rows, K/32], possibly living inside records."""
    q_ptr: int
    s_ptr: int
    rows: int
    K: int
    rows_per_rec: int = 0        # 0: one plain matrix
    rec_stride: int = 0
    keepalive: object = None

    @staticmethod
    def from_tensors(q: torch.Tensor, s: torch.Tensor) -> "MxOperand":
        assert q.dtype == torch.uint8 and s.dtype == torch.uint8 and q.is_contiguous() and s.is_contiguous()
        rows, K = q.shape
        assert tuple(s.shape) == (rows, K // BLOCK)
        return MxOperand(q.data_ptr(), s.data_ptr(), rows, K, keepalive=(q, s))

    @staticmethod
    def from_panel_records(rec: torch.Tensor, rows: int, K: int) -> "MxOperand":
        """The output of ``ops.gemm_send(..., out_fp8=True)`` (or its copy on the receiving side): one record per 128-row
        panel, ``[128 x K fp8][128 x K/32 scales]``.  ``rows`` need not be a multiple of 128: the last record is whole (the
        epilogue quantises zeros for the rows past the end) and the GEMM only uses its first ``rows % 128`` rows."""
        assert rec.dtype == torch.uint8
        stride = PANEL_ROWS * K + PANEL_ROWS * (K // BLOCK)
        assert rec.numel() >= -(-rows // PANEL_ROWS) * stride
        return MxOperand(rec.data_ptr(), rec.data_ptr() + PANEL_ROWS * K, rows, K, PANEL_ROWS, stride, keepalive=rec)

    @staticmethod
    def from_chunk_records(rec: torch.Tensor, rows: int, K: int, chunk_elems: int) -> "MxOperand":
        """The output of ``ops.pack_fp8_write`` for a row-major [rows, K] bf16 matrix packed with ``chunk_elems`` a
        multiple of 128 rows: ``[chunk fp8][chunk/32 scales][pad]`` per record."""
        assert rec.dtype == torch.uint8 and chunk_elems % (PANEL_ROWS * K) == 0 and (rows * K) % chunk_elems == 0
        return MxOperand(rec.data_ptr(), rec.data_ptr() + chunk_elems, rows, K, chunk_elems // K, record_bytes(chunk_elems), keepalive=rec)


@dataclass
class MxResult:
    status: str
    device_ns: int
    M: int
    N: int
    K: int
    variant: int = 0                       # 1 = single-CTA kernel, 2 = CTA-pair kernel

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    @property
    def tflops(self) -> float:
        return 2.0 * self.M * self.N * self.K / max(self.device_ns, 1) / 1e3


def gemm_mxfp8(ctx, a: MxOperand, b: MxOperand, c: torch.Tensor, grid: int = 0, stream=None, sync: bool = True, scratch_slot: int = 3,
               cta_group: int = 0, a_ready=None, timeout_ms: int = 2000):
    """``c[M,N] (bf16) = dequant(a)[M,K] @ dequant(b)[N,K].T`` with the block scales applied by the tensor core.
    Any M and N; K a multiple of 32 (one MX block) and of 16 bytes.
    ``cta_group``: 2 = CTA-pair kernel (256 x 128 per 2-CTA cluster, B multicast: half the B traffic per FLOP), 1 = single-CTA kernel
    (128 x 128), 0 = pair for M > 128.  ``RN_MX_CTA_GROUP`` overrides (A/B switch).
    ``a_ready``: receive-side fusion.  An int64 tensor with one word per 128-row panel of ``a`` (``a`` living in panel or chunk
    records of a registered receive buffer); the kernel starts a tile only once the word of the panel it reads is nonzero --
    ``ops.recv_consume(..., stamps=a_ready)`` sets it when the panel's receive completion arrives -- so the product overlaps
    the transfer panel by panel.  Launch with a ``grid`` that leaves SMs for whatever produces the panels (a persistent
    kernel spinning on all SMs would starve it)."""
    import os
    if os.environ.get("RN_MX_CTA_GROUP"):
        cta_group = int(os.environ["RN_MX_CTA_GROUP"])
    M, Nn, K = a.rows, b.rows, a.K
    assert b.K == K and c.dtype == torch.bfloat16 and tuple(c.shape) == (M, Nn) and c.is_contiguous()
    if a_ready is not None:
        assert a_ready.dtype == torch.int64 and a_ready.numel() >= -(-M // PANEL_ROWS) and a_ready.is_cuda
    lib = N.load()
    ws = work_stream(ctx, stream)
    out_addr, out_view = ctx.scratch(64, offset=4096 + scratch_slot * 64)
    done = ctx.dev_scratch(64, offset=scratch_slot * (256 << 10))          # zeroed device counter, cleaned by the kernel
    rc = lib.rn_k_gemm_mxfp8(_stream_ptr(ws), grid, a.q_ptr, a.s_ptr, a.rows_per_rec, a.rec_stride, b.q_ptr, b.s_ptr, b.rows_per_rec,
                             b.rec_stride, c.data_ptr(), M, Nn, K, out_addr, cta_group, done,
                             a_ready.data_ptr() if a_ready is not None else 0, timeout_ms)
    if rc:
        raise N.NativeError(f"gemm_mxfp8 launch failed ({rc})")
    if not sync:
        return out_view, ws
    ws.synchronize()
    w = (C.c_int64 * 8).from_buffer(out_view)
    r = MxResult(WAIT_STATUS.get(w[0], str(w[0])), w[2] - w[1], M, Nn, K, variant=int(w[6]))
    return r


# ------------------------------------------------------------------ PyTorch references
def quantize_mx(x: torch.Tensor):
    """bf16 / fp32 [rows, K] -> (e4m3 bytes [rows, K], UE8M0 scale bytes [rows, K/32]); same rule as the pack kernel."""
    rows, K = x.shape
    xb = x.float().reshape(rows, K // BLOCK, BLOCK)
    e = _scale_exponent(xb.abs().amax(dim=2))
    q = (xb * _pow2(-e)[..., None]).to(torch.float8_e4m3fn).view(torch.uint8).reshape(rows, K)
    return q.contiguous(), (e + 127).to(torch.uint8).contiguous()


def dequantize_mx(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    rows, K = q.shape
    v = q.view(torch.float8_e4m3fn).float().reshape(rows, K // BLOCK, BLOCK)
    return (v * _pow2(s.to(torch.int32) - 127)[..., None]).reshape(rows, K)
