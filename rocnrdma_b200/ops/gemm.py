"""K4 wrapper: Hopper wgmma/TMA bf16 GEMM whose epilogue RDMA-writes finished 128-row panels."""
from __future__ import annotations

import os

from dataclasses import dataclass

import torch

from .. import _native as N
from . import launch as L
from .rdma import _stream_ptr, work_stream

BM, BN, BK = 128, 256, 64


@dataclass
class GemmResult:
    status: str
    t_start_ns: int
    t_end_ns: int
    panels_posted: int
    t_first_post_ns: int
    t_compute_end_ns: int
    M: int
    N: int
    K: int
    variant: int = 0          # kernel that ran: 1 = single CTA, 2 = CTA pair, 3 = CTA pair with the stream-K tail
    stream_k: bool = False    # the last, partial wave of tiles was split along K

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    @property
    def device_ns(self) -> int:
        return self.t_end_ns - self.t_start_ns

    @property
    def tflops(self) -> float:
        return 2.0 * self.M * self.N * self.K / max(self.device_ns, 1) / 1e3

    @property
    def wire_gbps(self) -> float:
        return 2.0 * self.M * self.N / max(self.device_ns, 1)   # bf16 panels (fp8 records carry 33/64 of this)


def panel_record_bytes(N: int) -> int:
    """Bytes of one fp8 panel record: 128 x N e4m3 values followed by 128 x N/32 UE8M0 scales."""
    return BM * N + BM * (N // 32)


def ref_fp8_panels(c_fp32: torch.Tensor) -> torch.Tensor:
    """PyTorch reference of the fp8 epilogue: quantise an fp32 [M, N] result into panel records."""
    from .pack import quantize_blocks
    M0, Nn = c_fp32.shape
    M = -(-M0 // BM) * BM                    # records are whole panels: rows past M quantise zeros
    x = torch.zeros(M, Nn, dtype=torch.float32, device=c_fp32.device)
    x[:M0] = c_fp32.float()
    q, sc = quantize_blocks(x.reshape(M, Nn // 32, 32))
    q = q.reshape(M, Nn)
    out = torch.empty(M // BM, panel_record_bytes(Nn), dtype=torch.uint8, device=c_fp32.device)
    out[:, :BM * Nn] = q.reshape(M // BM, BM * Nn)
    out[:, BM * Nn:] = sc.reshape(M // BM, BM * (Nn // 32))
    return out.reshape(-1)


def dequant_fp8_panels(rec: torch.Tensor, M: int, Nn: int) -> torch.Tensor:
    from .pack import ue8m0
    P = -(-M // BM)
    r = rec[:P * panel_record_bytes(Nn)].reshape(P, panel_record_bytes(Nn))
    q = r[:, :BM * Nn].contiguous().view(torch.float8_e4m3fn).float().reshape(P * BM, Nn // 32, 32)
    s = ue8m0(r[:, BM * Nn:].reshape(P * BM, Nn // 32))
    return (q * s[..., None]).reshape(P * BM, Nn)[:M]


def gemm_send(ctx, a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, c_mr=None, qp=None, dst_mr=None,
              signal_every: int = 1, with_imm: bool = False, out_fp8: bool = False, cta_group: int = 0, group_m: int = 0, direct: bool = False, plain_stores: bool = False, grid: int = 0, timeout_ms: int = 2000, stream=None, sync: bool = True, post_only: bool = False, stream_k: bool = False,
              scratch_slot: int = L.SLOT["gemm_send"]):
    """``c[M,N] = a[M,K] @ b[N,K].T`` (bf16 in/out, fp32 accumulate: wgmma on the H100 tensor cores).

    With ``qp``/``c_mr``/``dst_mr`` every finished 128-row panel of ``c`` is RDMA-written to the same
    offset of ``dst_mr`` from inside the kernel; the call returns when the last panel has landed.
    Shapes: any M; N % 8 == 0 and K % 8 == 0 (16-byte rows for TMA), N % 32 == 0 for fp8 output.  Tiles that hang over an
    edge are zero-filled on load and clipped on store by TMA; the last panel sent may be short.  ``direct`` and
    ``plain_stores`` keep the tile-multiple restriction (M % 128, N % 256, K % 64).
    ``direct``: ``c`` is itself the peer's registered buffer (a tensor on the other GPU): the epilogue stores
    rows over NVLink and each panel is announced by a zero-length RDMA_WRITE_IMM (needs ``qp``, ``c_mr`` = the
    peer region as seen locally, ``dst_mr``).
    ``plain_stores``: bf16 epilogue with per-thread row stores instead of staged TMA tensor stores (A/B switch).
    ``group_m``: M blocks that advance together across N (L2 reuse of B; 0 = 8 for compute only, 4 when sending).
    ``cta_group``: 2 = CTA-pair kernel (a 2-CTA cluster per 256x256 tile, B multicast to both CTAs), 1 = single-CTA
    128x256 kernel, 3 = the pair kernel with the stream-K tail available, 0 (default) = the pair kernel when M % 256 == 0,
    else the single-CTA kernel.
    ``stream_k`` (cta_group 3 only): split the tiles of the last, partial wave along K over all CTA pairs and fold the
    fp32 partials back in the owner's epilogue.  Off by default; its speed on H100 has not been measured.
    """
    for t in (a, b):
        assert t.dtype == torch.bfloat16 and t.is_contiguous()
    M, K = a.shape
    Nn, K2 = b.shape
    assert K == K2 and c.is_contiguous()
    if out_fp8:
        # c is a uint8 buffer of ceil(M/128) panel records (block-scaled e4m3 + UE8M0 scales)
        assert c.dtype == torch.uint8 and c.numel() >= -(-M // BM) * panel_record_bytes(Nn)
    else:
        assert c.dtype == torch.bfloat16 and tuple(c.shape) == (M, Nn)
    if Nn % 8 or K % 8 or (out_fp8 and Nn % 32):
        raise ValueError(f"shape ({M},{Nn},{K}): N and K must be multiples of 8 (16-byte rows), N of 32 for fp8 output")
    if (direct or plain_stores) and (M % BM or Nn % BN or K % BK):
        raise ValueError(f"direct / plain_stores need multiples of the ({BM},{BN},{BK}) tile, got ({M},{Nn},{K})")
    if qp is not None and (c_mr is None or dst_mr is None):
        raise ValueError("sending needs c_mr (registration of c) and dst_mr")
    if cta_group == 0:
        cta_group = 2 if M % (2 * BM) == 0 else 1
    if os.environ.get("RN_GEMM_CTA_GROUP"):            # A/B switch for benchmarks
        cta_group = int(os.environ["RN_GEMM_CTA_GROUP"])
    if group_m == 0:
        # tile rasterisation: M blocks (pairs for cta_group 2) that advance together across N; more = better
        # L2 reuse of B, fewer = panels complete (and are sent) more evenly
        group_m = 8 if qp is None else 4
    lib = N.load()
    ws = work_stream(ctx, stream)
    m_blks = -(-M // BM)
    counters = L.counters(ctx, m_blks + 1, scratch_slot)
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot))
    rc = lib.rn_k_gemm_send(_stream_ptr(ws), grid, a.data_ptr(), b.data_ptr(), c.data_ptr(), M, Nn, K,
                            qp.dev_ptr if qp is not None else 0, c_mr.addr if c_mr is not None else 0,
                            c_mr.lkey if c_mr is not None else 0, dst_mr.addr if dst_mr is not None else 0,
                            dst_mr.rkey if dst_mr is not None else 0, signal_every, int(with_imm) | (2 if post_only else 0), int(out_fp8), cta_group, group_m, int(direct) | (2 if plain_stores else 0) | (4 if os.environ.get("RN_GEMM_DENSE_PROBE") else 0) | (8 if (not stream_k or os.environ.get("RN_GEMM_NO_STREAMK")) else 0), counters, out_addr, timeout_ms)
    return L.finish(rc, "gemm_send", out_view, ws, sync, parse, M, Nn, K)


def parse(view, M, Nn, K) -> GemmResult:
    r = L.decode_as(GemmResult, view, ("panels_posted", "t_first_post_ns", "t_compute_end_ns", "variant", "stream_k"),
                    M=M, N=Nn, K=K)
    r.stream_k = bool(r.stream_k)
    return r
