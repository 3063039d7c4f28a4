"""K7 wrapper: block-scaled fp8 GEMM (e4m3 ``wgmma`` per 32-deep MX block, scales applied in registers) whose operands are the records
the send side produces -- so a receiver multiplies straight out of its receive buffer."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import _native as N
from . import launch as L
from .pack import BLOCK, quantize_blocks, record_bytes, ue8m0
from .rdma import _stream_ptr, work_stream

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


def gemm_mxfp8(ctx, a: MxOperand, b: MxOperand, c: torch.Tensor, grid: int = 0, stream=None, sync: bool = True, scratch_slot: int = L.SLOT["gemm_mxfp8"],
               cta_group: int = 0, a_ready=None, timeout_ms: int = 2000, a_order=None, result_off=None):
    """``c[M,N] (bf16) = dequant(a)[M,K] @ dequant(b)[N,K].T`` with the block scales applied by the tensor core.
    Any M and N; K a multiple of 32 (one MX block) and of 16 bytes.
    ``cta_group``: 2 = CTA-pair kernel (256 x 128 per 2-CTA cluster, B multicast: half the B traffic per FLOP), 1 = single-CTA kernel
    (128 x 128), 0 = pair for M > 128.  ``RN_MX_CTA_GROUP`` overrides (A/B switch).
    ``a_ready``: receive-side fusion.  An int64 CUDA tensor with one word per record of ``a``, nonzero once that record has
    landed (``a`` living in panel or chunk records of a registered receive buffer; a plain ``a`` is one record).  The
    kernel starts a tile only once the word of the record it reads is nonzero, so the product overlaps the transfer record
    by record.  ``ops.recv_consume(..., stamps=a_ready)`` produces exactly these words when every record arrives by
    RDMA_WRITE_IMM with its index as the immediate: the chunk id for K3 records, the panel id for K4 records.  Launch with
    a ``grid`` that leaves SMs for whatever produces the records (a persistent kernel spinning on all SMs would starve it).
    ``a_order``: an int32 CUDA tensor with one entry per record of ``a``, a permutation of the record ids.  The
    single-CTA kernel then walks its tiles record by record in that order (each record's 128-row blocks in row order,
    every column block of a row block before the next), so that with ``a_ready`` it starts on the records that land
    first.  C does not depend on the order.  It needs ``a`` in whole records of whole 128-row blocks (M a multiple of
    ``rows_per_rec``, ``rows_per_rec`` a multiple of 128) and refuses ``cta_group=2``; with 0 it runs the single-CTA
    kernel.  An entry outside the record ids leaves that record's rows of C unwritten.
    ``result_off``: where in the mapped scratch the kernel writes its result words (default: the record of
    ``scratch_slot``)."""
    import os
    if os.environ.get("RN_MX_CTA_GROUP"):
        cta_group = int(os.environ["RN_MX_CTA_GROUP"])
    M, Nn, K = a.rows, b.rows, a.K
    assert b.K == K and c.dtype == torch.bfloat16 and tuple(c.shape) == (M, Nn) and c.is_contiguous()
    ready_addr = 0 if a_ready is None else L.tensor_ptr(a_ready, torch.int64, ctx.device,
                                                        "a_ready (one word per record of a)", -(-M // (a.rows_per_rec or M)))
    if a_order is not None:
        rpr = a.rows_per_rec or M
        if cta_group == 2:
            raise ValueError("a_order walks the single-CTA kernel: cta_group=2 (the CTA-pair kernel) has no ordered walk")
        if rpr % PANEL_ROWS or M % rpr:
            raise ValueError(f"a_order needs a in whole records of whole 128-row blocks: M={M}, rows_per_rec={rpr}")
        order_addr = L.tensor_ptr(a_order, torch.int32, ctx.device, "a_order (one id per record of a)", M // rpr, exact=True)
    lib = N.load()
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    done = L.counters(ctx, 1, scratch_slot)          # zeroed device counter, cleaned by the kernel
    args = (_stream_ptr(ws), grid, a.q_ptr, a.s_ptr, a.rows_per_rec, a.rec_stride, b.q_ptr, b.s_ptr, b.rows_per_rec,
            b.rec_stride, c.data_ptr(), M, Nn, K, out_addr, cta_group, done, ready_addr, timeout_ms)
    rc = lib.rn_k_gemm_mxfp8(*args) if a_order is None else lib.rn_k_gemm_mxfp8_ordered(*args, order_addr)
    return L.finish(rc, "gemm_mxfp8", out_view, ws, sync, _parse, M, Nn, K)


def _parse(view, M, Nn, K) -> MxResult:
    return L.decode_as(MxResult, view, (None, None, None, "variant"), M=M, N=Nn, K=K)


# ------------------------------------------------------------------ PyTorch references
def quantize_mx(x: torch.Tensor):
    """bf16 / fp32 [rows, K] -> (e4m3 bytes [rows, K], UE8M0 scale bytes [rows, K/32]); same rule as the pack kernel."""
    rows, K = x.shape
    q, s = quantize_blocks(x.float().reshape(rows, K // BLOCK, BLOCK))
    return q.reshape(rows, K).contiguous(), s.contiguous()


def dequantize_mx(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    rows, K = q.shape
    v = q.view(torch.float8_e4m3fn).float().reshape(rows, K // BLOCK, BLOCK)
    return (v * ue8m0(s)[..., None]).reshape(rows, K)


def _add_rn32(acc: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """fp32 ``acc`` + fp64 ``x`` rounded once to fp32 (what ``fmaf`` does with an exact product).  The fp64 sum is made
    round-to-odd first (two-sum error, then a step to the odd neighbour when it is inexact), which the final round to
    nearest-even fp32 cannot round a second time: 53 bits is more than 24 + 2."""
    a = acc.double()
    s = a + x
    bb = s - a
    err = (a - (s - bb)) + (x - bb)
    even = (s.view(torch.int64) & 1) == 0
    fix = torch.isfinite(s) & (err != 0) & even
    s = torch.where(fix, torch.nextafter(s, torch.where(err > 0, torch.inf, -torch.inf).to(s)), s)
    return s.float()


def ref_gemm_mxfp8(a_q: torch.Tensor, a_s: torch.Tensor, b_q: torch.Tensor, b_s: torch.Tensor) -> torch.Tensor:
    """Bit-exact reference of ``gemm_mxfp8``'s arithmetic over every pair of scale bytes: bf16 ``C[M, N]`` from e4m3
    bytes ``a_q [M, K]`` / ``b_q [N, K]`` and UE8M0 scale bytes ``a_s [M, K/32]`` / ``b_s [N, K/32]``, computed in fp64 on
    the operands' device, with each MX block added into an fp32 accumulator in k order with one rounding.

    For every output:

    * the MX blocks are taken in k order, into an fp32 accumulator that starts at +0;
    * a block's partial ``p`` is the exact sum of its 32 e4m3 products (fp64 holds it exactly: products span
      2^-18 .. 2^17.6; a NaN code makes it NaN; it is -0 only when every product is -0);
    * its contribution is ``x = p * 2^(ea + eb)`` with ``ea``, ``eb`` the row's and column's scale bytes minus 127 (byte 0 is
      2^-127, as in every decoder).  A byte 0xFF in either operand makes ``x = p * Inf``: +-Inf, or NaN where p = 0;
    * ``acc = fl32(acc + x)``: one rounding of the exact sum per block, over the whole range of ``ea + eb`` (-254 .. 254);
    * the output is ``acc`` rounded to nearest-even bf16.

    The kernel follows this rule only where the tensor core forms ``p`` exactly.  Its internal accumulator width is not
    measured (at least 11 bits, DESIGN.md), so a bit-for-bit comparison needs data whose block partials fit in 11
    significant bits; elsewhere compare against a bound."""
    M, K = a_q.shape
    Nn = b_q.shape[0]
    kb = K // BLOCK
    assert b_q.shape[1] == K and tuple(a_s.shape) == (M, kb) and tuple(b_s.shape) == (Nn, kb)
    A = a_q.view(torch.float8_e4m3fn).double().reshape(M, kb, BLOCK)
    B = b_q.view(torch.float8_e4m3fn).double().reshape(Nn, kb, BLOCK)
    ea, eb = a_s.to(torch.int32) - 127, b_s.to(torch.int32) - 127
    a_inf, b_inf = a_s == 255, b_s == 255
    # sign bits and nonzero indicators of the codes (a NaN code counts as nonzero: its partial is NaN anyway)
    na, nb = ((a_q & 0x80) != 0).double().reshape(M, kb, BLOCK), ((b_q & 0x80) != 0).double().reshape(Nn, kb, BLOCK)
    za, zb = ((a_q & 0x7F) != 0).double().reshape(M, kb, BLOCK), ((b_q & 0x7F) != 0).double().reshape(Nn, kb, BLOCK)
    acc = torch.zeros(M, Nn, dtype=torch.float32, device=a_q.device)
    for k in range(kb):
        p = A[:, k] @ B[:, k].T
        # IEEE sign of an exact zero sum: -0 only when all 32 products are -0 (zero, with signs that differ)
        opposite = na[:, k] @ (1 - nb[:, k]).T + (1 - na[:, k]) @ nb[:, k].T
        nonzero = za[:, k] @ zb[:, k].T
        neg_zero = (opposite == BLOCK) & (nonzero == 0)
        p = torch.where(p == 0, torch.where(neg_zero, -0.0, 0.0).to(p), p)
        x = p * torch.exp2((ea[:, k, None] + eb[None, :, k]).double())
        x = torch.where(a_inf[:, k, None] | b_inf[None, :, k], p * torch.inf, x)
        acc = _add_rn32(acc, x)
    return acc.to(torch.bfloat16)
