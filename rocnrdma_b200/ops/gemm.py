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


# ------------------------------------------------------------------ K4 with a landed addend
RS_WORDS = ("records_posted", "t_first_post_ns", "t_compute_end_ns", "records_added")


@dataclass
class ReduceSendResult:
    status: str
    t_start_ns: int
    t_end_ns: int
    records_posted: int
    t_first_post_ns: int
    t_compute_end_ns: int
    records_added: int

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    @property
    def device_ns(self) -> int:
        return self.t_end_ns - self.t_start_ns


def parse_reduce_send(view) -> ReduceSendResult:
    """Decode the record :func:`gemm_reduce_send` leaves in the mapped scratch (for ``sync=False`` callers)."""
    return L.decode_as(ReduceSendResult, view, RS_WORDS)


def _host_ids(t, what: str, n: int, device: int, host) -> list:
    L.tensor_ptr(t, torch.int32, device, what, n, exact=True, align=4)
    return [int(v) for v in (t.tolist() if host is None else host)]


def gemm_reduce_send(ctx, a: torch.Tensor, b: torch.Tensor, *, walk, add_ids, send_ids, qp, staging_mr=None, dst_mr=None,
                     landing=None, ready=None, out=None, ids_host=None, with_imm: bool = True, signal_every: int = 1,
                     post_only: bool = False, cta_group: int = 1, group_m: int = 0, direct: bool = False,
                     plain_stores: bool = False, stream_k: bool = False, grid: int = 0, timeout_ms: int = 2000, stream=None,
                     sync: bool = True, scratch_slot: int = L.SLOT["gemm_send"], result_off=None):
    """K4 with a landed addend: one hop of a reduce-scatter of ``a @ b.T``, in one launch.

    ``a`` [M, K] and ``b`` [Nb, K] are contiguous bf16, M a multiple of 128, Nb of 32, K of 8.  The P = M / 128 m-blocks
    of ``a`` are computed in the order ``walk`` gives (int32 [P], a permutation of 0..P-1); the tile raster runs over
    walk positions, ``group_m`` of them advancing together across Nb.  Walk position p's 128 x Nb panel, accumulated in
    fp32, then:

    * adds landed record ``add_ids[p]`` of ``landing`` (uint8 CUDA tensor of fp8 panel records, ``panel_record_bytes(Nb)``
      apart) once its arrival word ``ready[add_ids[p]]`` (int64) is set, or nothing for -1.  The gate runs after the
      tile's MMAs, so the tile computes while its record is on the wire.  Each element is ``acc + code * 2^(byte - 127)``,
      one fp32 multiply and one fp32 add, the bits of :func:`~rocnrdma_b200.ops.reduce_fp8` with an fp32 ``local``;
    * becomes staging record ``send_ids[p]``: quantised by the fp8 epilogue's rule into ``staging_mr`` at ``id * rec`` and
      posted by the CTA that finishes it, as one RDMA WRITE (WRITE_IMM with immediate ``id`` when ``with_imm``) to the same
      offset of ``dst_mr``; or, for -1, the j-th such position stores bf16 rows ``[128 j, 128 j + 128)`` of ``out``
      (contiguous bf16 [128 * #(-1), Nb]), rounded to nearest even.

    The last CTA posts a flush and waits for it unless ``post_only``.  A word still 0 after ``timeout_ms`` raises a
    grid-wide flag that ends every other wait too, so a failed launch ends ``TIMEOUT`` within about one timeout; a panel
    that is not finished is never posted, and fewer posted records than ``send_ids`` holds is ``TIMEOUT``.

    ``walk``, ``add_ids`` and ``send_ids`` are int32 tensors on the context's device.  They are checked on the host from
    ``ids_host`` (three lists) when given, else by reading them back (which waits for the stream that wrote them).
    Refused: ids out of range, a walk entry that repeats, a send id used twice, ``cta_group`` other than 1, ``direct``,
    ``plain_stores`` and ``stream_k``.  With ``ids_host`` the kernel still reads the tensors, and nothing compares the
    two: lists that differ from the tensors leave the tensors' ids unchecked (out-of-range TMA coordinates and record
    offsets).  Pass ``ids_host`` only with the values the tensors hold, as ``RingReduceScatterFp8`` does with the ids it
    built them from.  Returns a :class:`ReduceSendResult`, or ``(view, stream)``
    with ``sync=False`` (decode with :func:`parse_reduce_send`)."""
    dev = ctx.device
    if cta_group != 1:
        raise ValueError(f"cta_group={cta_group}: the walk runs on the single-CTA tile (cta_group=1)")
    if direct or plain_stores or stream_k:
        raise ValueError("gemm_reduce_send has no direct, plain_stores or stream_k variant")
    for t, what in ((a, "a"), (b, "b")):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.bfloat16 or t.dim() != 2 or not t.is_contiguous():
            raise ValueError(f"{what} must be a contiguous 2-D bf16 tensor")
        L.tensor_ptr(t, torch.bfloat16, dev, what, t.numel(), align=16)
    M, K = a.shape
    Nn, K2 = b.shape
    if K != K2:
        raise ValueError(f"a has K={K}, b has K={K2}")
    if M <= 0 or M % BM or Nn <= 0 or Nn % 32 or K <= 0 or K % 8:
        raise ValueError(f"shape ({M},{Nn},{K}): M must be a multiple of {BM}, Nb of 32 and K of 8")
    if qp is None:
        raise ValueError("gemm_reduce_send posts its records and flushes: pass qp")
    P, rec = M // BM, panel_record_bytes(Nn)
    hw, ha, hs = ids_host if ids_host is not None else (None, None, None)
    walk_l = _host_ids(walk, "walk", P, dev, hw)
    add_l = _host_ids(add_ids, "add_ids", P, dev, ha)
    send_l = _host_ids(send_ids, "send_ids", P, dev, hs)
    if sorted(walk_l) != list(range(P)):
        raise ValueError(f"walk must hold every m-block 0..{P - 1} once")
    n_land = 0
    if landing is not None:
        if not isinstance(landing, torch.Tensor) or landing.dtype != torch.uint8:
            raise ValueError("landing must be a uint8 tensor of fp8 panel records")
        L.tensor_ptr(landing, torch.uint8, dev, "landing", landing.numel(), align=16)
        n_land = landing.numel() // rec
    if any(i < -1 or i >= n_land for i in add_l):
        raise ValueError(f"add_ids must lie in [-1, {n_land}): landing holds {n_land} records of {rec} bytes")
    if n_land and any(i >= 0 for i in add_l):
        if ready is None:
            raise ValueError("an addend needs its arrival words: pass ready")
        L.tensor_ptr(ready, torch.int64, dev, "ready", n_land, align=8)
    sends = [i for i in send_l if i >= 0]
    n_staging = 0 if staging_mr is None else staging_mr.length // rec
    if any(i < -1 for i in send_l) or any(i >= n_staging for i in sends):
        raise ValueError(f"send_ids must lie in [-1, {n_staging}): staging_mr holds {n_staging} records of {rec} bytes")
    if len(set(sends)) != len(sends):
        raise ValueError("a send id may be used once")
    if sends and (dst_mr is None or dst_mr.length < (max(sends) + 1) * rec):
        raise ValueError("dst_mr must hold every posted record at its id's offset")
    if sends and staging_mr.addr % 16:
        raise ValueError("staging_mr must be 16-byte aligned")
    out_rows = BM * (P - len(sends))
    if out_rows:
        if out is None or out.dtype != torch.bfloat16 or tuple(out.shape) != (out_rows, Nn) or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous bf16 [{out_rows}, {Nn}] tensor: one 128-row block per send id -1")
        L.tensor_ptr(out, torch.bfloat16, dev, "out", out.numel(), align=16)
        lo, hi = out.data_ptr(), out.data_ptr() + out.numel() * 2
        for t in (a, landing):
            if t is not None and lo < t.data_ptr() + t.numel() * t.element_size() and t.data_ptr() < hi:
                raise ValueError("out must not overlap a or landing")
    if group_m == 0:
        group_m = next(g for g in (4, 2, 1) if P % g == 0)
    lib = N.load()
    ws = work_stream(ctx, stream)
    counters = L.counters(ctx, P + 3, scratch_slot)      # per m-block ; CTAs done ; abort flag ; records added
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    rc = lib.rn_k_gemm_reduce_send(
        _stream_ptr(ws), grid, a.data_ptr(), b.data_ptr(), M, Nn, K, walk.data_ptr(), add_ids.data_ptr(),
        send_ids.data_ptr(), len(sends), staging_mr.addr if staging_mr is not None else 0, n_staging,
        landing.data_ptr() if landing is not None else 0, n_land, ready.data_ptr() if ready is not None else 0,
        out.data_ptr() if out_rows else 0, out_rows, qp.dev_ptr, staging_mr.addr if staging_mr is not None else 0,
        staging_mr.lkey if staging_mr is not None else 0, dst_mr.addr if dst_mr is not None else 0,
        dst_mr.rkey if dst_mr is not None else 0, signal_every, int(with_imm) | (2 if post_only else 0), cta_group, group_m,
        counters, out_addr, timeout_ms)
    return L.finish(rc, "gemm_reduce_send", out_view, ws, sync, parse_reduce_send)
