"""K3 / K5 wrappers: bf16 -> fp8 block-scaled pack fused with GPU-initiated RDMA write,
the receive-side unpack, the reduction of several sources' records, and the bit-exact PyTorch references of all three."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import torch

from .. import _native as N
from . import launch as L
from .launch import SLOT
from .rdma import _stream_ptr, work_stream

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


PACK_WORDS = ("wqes", "t_first_post_ns", "t_pack_end_ns")
UNPACK_WORDS = ("records_seen", "records_forwarded", "t_first_post_ns")
REDUCE_WORDS = ("records_reduced", "records_posted", "t_first_post_ns", "t_reduce_end_ns")


def _parse(view, n_elems, wire) -> PackResult:
    return L.decode_as(PackResult, view, PACK_WORDS, n_elems=n_elems, wire_bytes=wire)


def pack_fp8_write(ctx, src: torch.Tensor, staging_mr, qp=None, dst_mr=None, chunk_elems: int = 1 << 20,
                   with_imm: bool = False, signal_every: int = 1, grid: int = 0, timeout_ms: int = 2000,
                   stream=None, sync: bool = True, scratch_slot: int = SLOT["pack"], post_only: bool = False, direct: bool = False,
                   result_off=None, residual=None, staging_off: int = 0):
    """Pack ``src`` (bf16) into fp8 chunk records in ``staging_mr`` and, if ``qp`` is given,
    RDMA-write every record to the same offset of ``dst_mr`` from inside the kernel.
    ``staging_off``: the records start that many bytes into ``staging_mr`` (a multiple of 64), and land at the same
    offset of ``dst_mr``.
    ``result_off``: where in the mapped scratch the kernel writes its result words (default: the record of
    ``scratch_slot``, see :func:`~rocnrdma_b200.ops.launch.result_offset`).
    ``direct``: ``staging_mr`` is the *peer's* buffer registered with this context (NVLink-mapped, ``ctx.reg_mr(tensor_on_the_peer)``):
    the kernel's own stores deliver the records and each one is announced by a zero-length RDMA_WRITE_IMM (needs ``with_imm``).
    ``residual``: error feedback, an fp32 CUDA tensor of ``src.numel()`` values (contiguous, 32-byte aligned) read and
    written in place: the kernel quantises ``v = src + residual`` and leaves there what the records lost, ``v - decode``
    (0 where either is not finite).  The add saturates: where finite operands overflow fp32, ``v`` is +-FLT_MAX, so
    finite inputs always give finite records and residuals.  :func:`ref_pack_fp8` reproduces both bit for bit."""
    if direct and not (with_imm and qp is not None and dst_mr is not None):
        raise ValueError("direct mode announces records with RDMA_WRITE_IMM: pass qp, dst_mr and with_imm=True")
    assert src.dtype == torch.bfloat16 and src.is_contiguous()
    n = src.numel()
    if n % TILE_ELEMS or chunk_elems % TILE_ELEMS or n % chunk_elems:
        raise ValueError(f"n_elems and chunk_elems must be multiples of {TILE_ELEMS}, n_elems of chunk_elems")
    wire = staging_bytes(n, chunk_elems)
    staging_off = int(staging_off)
    if staging_off < 0 or staging_off % 64:
        raise ValueError(f"staging_off={staging_off}: a non-negative multiple of 64")
    if staging_mr.length < staging_off + wire or (dst_mr is not None and dst_mr.length < staging_off + wire):
        raise ValueError("staging / destination region too small for the records")
    res_addr = 0 if residual is None else L.tensor_ptr(residual, torch.float32, ctx.device, "residual", n, exact=True, align=32)
    lib = N.load()
    ws = work_stream(ctx, stream)
    # [n_chunks] groups packed per record ; CTAs done
    counters = L.counters(ctx, n // chunk_elems + 1, scratch_slot)
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    rc = lib.rn_k_pack_fp8_write(_stream_ptr(ws), grid, src.data_ptr(), staging_mr.addr + staging_off, n, chunk_elems,
                                 qp.dev_ptr if qp is not None else 0, staging_mr.addr + staging_off, staging_mr.lkey,
                                 dst_mr.addr + staging_off if dst_mr is not None else 0, dst_mr.rkey if dst_mr is not None else 0,
                                 int(with_imm) | (2 if post_only else 0) | (4 if direct else 0), signal_every, counters, out_addr, timeout_ms,
                                 res_addr)
    return L.finish(rc, "pack_fp8_write", out_view, ws, sync, None if qp is None else _parse, n, wire)


def unpack_fp8(ctx, staging: torch.Tensor, dst: torch.Tensor, chunk_elems: int = 1 << 20, qp=None, grid: int = 0,
               timeout_ms: int = 2000, stream=None, sync: bool = True, scratch_slot: int = SLOT["unpack"], ready=None, *,
               fwd_qp=None, fwd_src_mr=None, fwd_dst_mr=None, fwd_dst_off: int = 0, with_imm: bool = False,
               imm_base: int = 0, signal_every: int = 1, post_only: bool = False, result_off=None):
    """fp8 chunk records -> bf16.  With ``qp`` the kernel waits for each record's receive
    CQE (RDMA_WRITE_IMM, immediate = chunk id) before touching it.  With ``ready`` (int64 CUDA tensor, one arrival word
    per record, as :func:`~rocnrdma_b200.ops.read_records` and ``recv_consume`` set them) every worker waits for the word of
    the record it is about to read; a word still 0 after ``timeout_ms`` ends the kernel with ``TIMEOUT``.  ``qp`` and
    ``ready`` exclude each other.  ``records_seen``: records announced on the CQ, or, with ``ready``, the words that are
    nonzero when the kernel ends (after a ``TIMEOUT`` that can include records it never waited for or unpacked).

    Forwarding (``fwd_qp``, with ``fwd_src_mr`` -- the registered region that holds ``staging`` -- and ``fwd_dst_mr``):
    each record is also posted unchanged, straight from where it landed, as one RDMA WRITE (WRITE_IMM with immediate
    ``imm_base + r`` when ``with_imm``) from ``staging`` to ``fwd_dst_mr`` at ``fwd_dst_off + r * record_bytes``.  The
    first CTA that sees record r's word (or, without ``ready``, the first that reads it) posts it, before unpacking it,
    so each record is posted exactly once and a record whose word never comes is never posted.  The last CTA posts a
    flush and waits for it unless ``post_only``; the status is ``TIMEOUT`` when fewer records were posted than exist.
    Forwarding works with ``ready`` or with no wait at all, never with ``qp``.  ``records_forwarded`` and
    ``t_first_post_ns`` are then set in the result."""
    assert dst.dtype == torch.bfloat16 and dst.is_contiguous()
    if (staging.data_ptr() | dst.data_ptr()) & 31:
        raise ValueError("unpack_fp8: records and output must be 32-byte aligned (256-bit loads / stores)")
    n = dst.numel()
    n_chunks = n // chunk_elems
    if qp is not None and ready is not None:
        raise ValueError("unpack_fp8 waits on a receive CQ (qp) or on arrival words (ready), not both")
    fwd = (fwd_qp, fwd_src_mr, fwd_dst_mr)
    if any(f is not None for f in fwd) and any(f is None for f in fwd):
        raise ValueError("forwarding needs fwd_qp, fwd_src_mr and fwd_dst_mr together")
    if fwd_qp is not None:
        if qp is not None:
            raise ValueError("unpack_fp8 forwards with ready= or with no wait, not with the CQ poller (qp)")
        if n <= 0 or chunk_elems <= 0 or n % TILE_ELEMS or chunk_elems % TILE_ELEMS or n % chunk_elems:
            raise ValueError(f"n_elems and chunk_elems must be multiples of {TILE_ELEMS}, n_elems of chunk_elems")
        wire = staging_bytes(n, chunk_elems)
        src_off = staging.data_ptr() - fwd_src_mr.addr
        if src_off < 0 or src_off + wire > fwd_src_mr.length:
            raise ValueError(f"the {n_chunks} records in staging do not lie inside fwd_src_mr")
        if fwd_dst_off < 0 or fwd_dst_off + wire > fwd_dst_mr.length:
            raise ValueError(f"{n_chunks} records of {record_bytes(chunk_elems)} bytes at fwd_dst_off={fwd_dst_off} do not "
                             f"fit fwd_dst_mr ({fwd_dst_mr.length} bytes)")
        if not 0 <= imm_base or imm_base + n_chunks > 1 << 32:
            raise ValueError(f"imm_base={imm_base}: the immediates imm_base + r of {n_chunks} records must fit 32 bits")
    ready_addr = 0 if ready is None else L.tensor_ptr(ready, torch.int64, ctx.device, "ready", n_chunks)
    lib = N.load()
    ws = work_stream(ctx, stream)
    # [n_chunks] flags (claims when forwarding) ; CTAs done ; records seen ; abort flag
    arrived = L.counters(ctx, n_chunks + 3, scratch_slot)
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    rc = lib.rn_k_unpack_fp8(_stream_ptr(ws), grid, staging.data_ptr(), dst.data_ptr(), n, chunk_elems,
                             qp.dev_ptr if qp is not None else 0, arrived, out_addr, timeout_ms, ready_addr,
                             fwd_qp.dev_ptr if fwd_qp is not None else 0,
                             fwd_src_mr.addr + src_off if fwd_qp is not None else 0,
                             fwd_src_mr.lkey if fwd_qp is not None else 0,
                             fwd_dst_mr.addr + fwd_dst_off if fwd_qp is not None else 0,
                             fwd_dst_mr.rkey if fwd_qp is not None else 0, int(with_imm) | (2 if post_only else 0),
                             imm_base, signal_every)
    return L.finish(rc, "unpack_fp8", out_view, ws, sync, parse_unpack)


def parse_unpack(view) -> dict:
    """Decode the record :func:`unpack_fp8` leaves in the mapped scratch (for ``sync=False`` callers)."""
    return L.decode(view, UNPACK_WORDS)


# ------------------------------------------------------------------ relay
RELAY_WORDS = ("records_posted", "t_first_post_ns")


def relay_records(qp, src_mr, dst_mr, rec_bytes: int, ids, *, ready=None, with_imm: bool = True, signal_every: int = 1,
                  post_only: bool = False, timeout_ms: int = 2000, stream=None, sync: bool = True,
                  scratch_slot: int = SLOT["unpack"], result_off=None):
    """Pass records on unchanged, in a given order, each as soon as it has landed: one thread on the GPU that does the
    forwarding unpack's per-record step without the unpack.

    ``src_mr`` and ``dst_mr`` hold records of ``rec_bytes`` back to back; record r goes from ``src_mr.addr + r *
    rec_bytes`` to ``dst_mr.addr + r * rec_bytes``.  ``ids`` (int32 CUDA tensor) lists the record ids in posting order.
    For each id r the kernel waits for ``ready[r]`` (int64 CUDA tensor, one arrival word per record of ``src_mr``, as
    ``recv_consume`` sets them; None: the records are in place), then posts one RDMA WRITE, or WRITE_IMM with immediate
    r when ``with_imm``.  Then it posts one flush and waits for it, unless ``post_only``.  A word still 0 after
    ``timeout_ms`` ends the kernel ``TIMEOUT``: that record and every later one are never posted.  An id outside the
    records ends it with status ``-22`` the same way.  Nothing else may post to ``qp`` while the relay runs.

    Its counters are the last 32 bytes of ``scratch_slot``, so it can run beside a launch that keeps its counters at the
    start of the same slot (the unpack's, the GEMM's).  Returns a dict with ``records_posted`` and ``t_first_post_ns``,
    or ``(result view, stream)`` with ``sync=False`` (decode with :func:`parse_relay`)."""
    rec_bytes = int(rec_bytes)
    if rec_bytes <= 0 or rec_bytes % 64 or rec_bytes >= 1 << 32:
        raise ValueError(f"rec_bytes={rec_bytes}: a positive multiple of 64 below 2**32")
    n_rec = min(src_mr.length, dst_mr.length) // rec_bytes
    if n_rec == 0:
        raise ValueError(f"src_mr ({src_mr.length} bytes) and dst_mr ({dst_mr.length} bytes) must hold a record of {rec_bytes}")
    if not isinstance(ids, torch.Tensor) or ids.dim() != 1 or ids.numel() == 0:
        raise ValueError("ids must be a non-empty 1-D int32 tensor of record ids")
    ctx = qp.ctx
    ids_addr = L.tensor_ptr(ids, torch.int32, ctx.device, "ids", 1)
    if ids.numel() >= 1 << 32:
        raise ValueError(f"{ids.numel()} ids: at most 2**32 - 1")
    ready_addr = 0 if ready is None else L.tensor_ptr(ready, torch.int64, ctx.device, "ready", n_rec)
    lib = N.load()
    ws = work_stream(ctx, stream)
    nb = L.counter_bytes(1)                 # abort flag ; post_record's three words
    L.counters(ctx, 1, scratch_slot)        # checks the slot
    counters = ctx.dev_scratch(nb, offset=(scratch_slot + 1) * L.SLOT_BYTES - nb)
    out_addr, out_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    rc = lib.rn_k_relay_records(_stream_ptr(ws), qp.dev_ptr, ids_addr, ids.numel(), min(n_rec, (1 << 32) - 1), ready_addr,
                                src_mr.addr, src_mr.lkey, dst_mr.addr, dst_mr.rkey, rec_bytes,
                                int(with_imm) | (2 if post_only else 0), signal_every, counters, out_addr, timeout_ms)
    return L.finish(rc, "relay_records", out_view, ws, sync, parse_relay)


def parse_relay(view) -> dict:
    """Decode the record :func:`relay_records` leaves in the mapped scratch (for ``sync=False`` callers)."""
    return L.decode(view, RELAY_WORDS)


# ------------------------------------------------------------------ scatter
MAX_SCATTER = 8                 # ranks of one pack_fp8_scatter launch (pack_fp8.cu kMaxScatter)
SCATTER_WORDS = PACK_WORDS


def pack_fp8_scatter(ctx, x: torch.Tensor, rank: int, world: int, staging_mr, own: torch.Tensor, own_words: torch.Tensor,
                     qps, dst_mrs, chunk_elems: int = 1 << 20, *, with_imm: bool = True, signal_every: int = 1,
                     post_only: bool = False, residual=None, grid: int = 0, timeout_ms: int = 2000, stream=None,
                     sync: bool = True, scratch_slot: int = SLOT["pack"], result_off=None):
    """K3 of an all-to-all: pack ``world`` shards of ``x`` (bf16, shard d = ``x[d * n:(d + 1) * n]``, R = n /
    ``chunk_elems`` records each) in one launch and post shard d to rank d as its records complete.

    Shards are packed in phase order: phase j is shard ``(rank + j) % world``, phase 0 the own shard.  Record r of shard
    d != ``rank`` is packed into ``staging_mr`` at record ``d * R + r`` and posted on ``qps[d]`` to ``dst_mrs[d]`` at
    record ``rank * R + r`` -- slot ``rank`` of rank d's landing region -- as an RDMA WRITE_IMM with immediate ``rank * R
    + r`` (WRITE without ``with_imm``).  The own shard's R records are written into ``own`` (uint8, R records: this rank's
    landing slot) and nothing is posted for them; the CTA that completes record r stamps ``own_words[r]`` (int64, R words)
    with a release store, as the receive consumer stamps landed records, so a reader gated on those words starts on
    them while the pack still runs.  ``qps[rank]`` and ``dst_mrs[rank]`` are ignored (None is fine).

    The last CTA posts one flush on every destination's queue pair and waits for them unless ``post_only``; the status is
    ``TIMEOUT`` when fewer than R records went to some destination.  There is no error feedback: an all-to-all quantises
    every value once, so ``residual`` is refused.  The counters sit at the top of ``scratch_slot`` (as the relay's), so the
    pack runs beside a launch that keeps its counters at the start of the same slot.  Two result records at
    ``result_off`` (default: the first two ring records of ``scratch_slot``): the first is K3's (``wqes`` = records
    posted in all), word d of the second the records posted to rank d.  Returns ``(PackResult, counts)`` or, with
    ``sync=False``, ``(view, stream)`` (decode with :func:`parse_scatter`)."""
    if residual is not None:
        raise ValueError("pack_fp8_scatter has no error feedback: an all-to-all quantises every value once, so there is "
                         "no error to carry into a later call")
    rank, world, chunk_elems = int(rank), int(world), int(chunk_elems)
    if not 2 <= world <= MAX_SCATTER or not 0 <= rank < world:
        raise ValueError(f"rank={rank}, world={world}: 2..{MAX_SCATTER} ranks")
    dev = ctx.device
    L.tensor_ptr(x, torch.bfloat16, dev, "x", 1, align=32)
    total = x.numel()
    n = total // world
    if total % world or n % TILE_ELEMS or chunk_elems <= 0 or chunk_elems % TILE_ELEMS or n % chunk_elems:
        raise ValueError(f"x holds {total} elements: {world} shards of a multiple of chunk_elems={chunk_elems}, itself a "
                         f"multiple of {TILE_ELEMS}")
    R, rec = n // chunk_elems, record_bytes(chunk_elems)
    L.tensor_ptr(own, torch.uint8, dev, "own", R * rec, exact=True, align=32)
    L.tensor_ptr(own_words, torch.int64, dev, "own_words", R, exact=True)
    if staging_mr.length < world * R * rec:
        raise ValueError(f"staging_mr holds {staging_mr.length} bytes; {world} shards of {R} records need {world * R * rec}")
    if staging_mr.addr & 31:
        raise ValueError("staging_mr must be 32-byte aligned")
    if len(qps) != world or len(dst_mrs) != world:
        raise ValueError(f"qps and dst_mrs: one entry per rank ({world})")
    peers = [d for d in range(world) if d != rank]
    if any(qps[d] is None or dst_mrs[d] is None for d in peers):
        raise ValueError("every other rank needs a queue pair and a landing region")
    if any(dst_mrs[d].length < (rank + 1) * R * rec for d in peers):
        raise ValueError(f"a destination's landing region cannot hold slot {rank} ({R} records of {rec} bytes)")
    U64, U32 = C.c_uint64 * world, C.c_uint32 * world
    qp_arr = U64(*[0 if d == rank else qps[d].dev_ptr for d in range(world)])
    va_arr = U64(*[0 if d == rank else dst_mrs[d].addr for d in range(world)])
    rk_arr = U32(*[0 if d == rank else dst_mrs[d].rkey for d in range(world)])
    lib = N.load()
    ws = work_stream(ctx, stream)
    # [world R] groups packed per record ; CTAs done ; then post_record's three words per destination
    nb = L.counter_bytes(world * R + 1) + 24 * (world - 1)
    L.counters(ctx, 1, scratch_slot)        # checks the slot
    if nb > L.SLOT_BYTES:
        raise ValueError(f"{world} shards of {R} records need {nb} bytes of counters; a scratch slot holds {L.SLOT_BYTES}")
    counters = ctx.dev_scratch(nb, offset=(scratch_slot + 1) * L.SLOT_BYTES - nb)
    off = L.ring_result_offset(scratch_slot, 0) if result_off is None else L.scratch_offset(result_off, 2)
    out_addr, out_view = L.result(ctx, off, 2)
    rc = lib.rn_k_pack_fp8_scatter(_stream_ptr(ws), grid, x.data_ptr(), staging_mr.addr, n, chunk_elems, rank, world,
                                   qp_arr, va_arr, rk_arr, staging_mr.addr, staging_mr.lkey, own.data_ptr(),
                                   own_words.data_ptr(), int(with_imm) | (2 if post_only else 0), signal_every, counters,
                                   out_addr, timeout_ms)
    return L.finish(rc, "pack_fp8_scatter", out_view, ws, sync, parse_scatter, total, world * R * rec - R * rec)


def parse_scatter(view, n_elems: int = 0, wire: int = 0):
    """Decode the two records :func:`pack_fp8_scatter` leaves: ``(PackResult, counts)``, ``counts[d]`` the records posted
    to rank d (0 for the own rank)."""
    counts = list((C.c_int64 * 8).from_buffer(view, L.RECORD_BYTES))
    return _parse(view, n_elems, wire), counts

# Non-finite rule (the kernels' behaviour, which these references reproduce bit for bit):
#   * the block amax ignores NaN (the kernels reduce with fmaxf), so a NaN stays in its own element and its
#     finite neighbours quantise as if it were absent;
#   * a block holding +-Inf gets exponent 127 (scale byte 254) and multiplier 2^-127 == 0.0, so the Inf becomes
#     NaN and every finite neighbour becomes +-0;
#   * decoding, scale byte 0x00 is 2^-127 (the OCP MX value, an fp32 denormal) and 0xFF is 2^128 == Inf.
#   * at e = 120, the one exponent whose codes 248 and 256 would decode past fp32 max (to 2^128 = Inf), a scaled value
#     above 240 in magnitude saturates to +-240, so every finite input decodes finite (NaN is kept).
#   * error feedback (``residual=``) adds with _ef_add: finite operands whose fp32 sum overflows give +-FLT_MAX, not
#     +-Inf, so that what the e = 120 saturation leaves in a residual (up to FLT_MAX - 240 * 2^120) cannot overflow the
#     next add; NaN and Inf operands propagate.  Without a residual an overflowing sum is Inf.
def _scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """e = smallest integer with amax / 2^e <= 448, clamped to [-127, 127], computed on the fp32 bit pattern of
    amax * (1/448) exactly as the kernels do (no log2 rounding): a value at or below 2^-127 (fp32 0x00400000) gives
    -127, any other exponent(v) + (mantissa(v) != 0)."""
    v = (amax.float() * (1.0 / 448.0)).contiguous()
    bits = v.view(torch.int32)
    e = ((bits >> 23) & 0xFF) - 127 + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    return torch.where(bits <= 0x00400000, torch.full_like(e, -127), e.clamp(max=127))


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
    y = x * _pow2(-e)[..., None]
    lim = torch.where(e == 120, 240.0, 448.0)[..., None]
    y = torch.where(y.abs() > lim, torch.copysign(lim, y), y)     # NaN compares false and stays
    q = y.to(torch.float8_e4m3fn).view(torch.uint8)
    return q, (e + 127).to(torch.uint8)


def _quantized_records(x: torch.Tensor, chunk_elems: int) -> torch.Tensor:
    """Chunk records (uint8) of the fp32 values ``x``, quantised by :func:`quantize_blocks`."""
    q, sc = quantize_blocks(x.reshape(-1, BLOCK))
    n_chunks = x.numel() // chunk_elems
    rec = record_bytes(chunk_elems)
    out = torch.zeros(n_chunks, rec, dtype=torch.uint8, device=x.device)
    out[:, :chunk_elems] = q.reshape(n_chunks, chunk_elems)
    out[:, chunk_elems:chunk_elems + chunk_elems // BLOCK] = sc.reshape(n_chunks, -1)
    return out.reshape(-1)


FLT_MAX = torch.finfo(torch.float32).max


def _ef_add(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Error feedback's fp32 add (``ef_add`` in pack_fp8.cu): ``a + b`` rounded to nearest, except that finite operands
    whose sum overflows give +-FLT_MAX with the sign of the sum.  A NaN or Inf operand propagates as in ``a + b``."""
    s = a + b
    sat = torch.isinf(s) & torch.isfinite(a) & torch.isfinite(b)
    return torch.where(sat, torch.copysign(torch.full_like(s, FLT_MAX), s), s)


def _ef_residual(v: torch.Tensor, records: torch.Tensor, chunk_elems: int) -> torch.Tensor:
    """The residual error feedback keeps: ``v - d`` with ``d`` the decode of ``v``'s records, and 0 wherever that is
    not finite (``v`` or ``d`` is not).  For finite ``v`` and ``d`` the difference is exact in fp32, so ``d + r == v``."""
    d = _decode_records(records, 1, v.numel(), chunk_elems)[0]
    r = v.reshape(-1) - d
    return torch.where(torch.isfinite(r), r, torch.zeros_like(r))


def ref_pack_fp8(src: torch.Tensor, chunk_elems: int, residual=None):
    """Reference chunk records (uint8) for a bf16 tensor; runs on CPU or GPU.  With ``residual`` (fp32, ``src.numel()``)
    it quantises ``src + residual`` (one saturating fp32 add, :func:`_ef_add`) and returns ``(records, new residual)``,
    as :func:`pack_fp8_write` does with ``residual=``."""
    if residual is None:
        return _quantized_records(src.float(), chunk_elems)
    v = _ef_add(src.reshape(-1).float(), residual.reshape(-1).float().to(src.device))
    recs = _quantized_records(v, chunk_elems)
    return recs, _ef_residual(v, recs, chunk_elems)


def ref_unpack_fp8(records: torch.Tensor, n_elems: int, chunk_elems: int) -> torch.Tensor:
    return _decode_records(records, 1, n_elems, chunk_elems)[0].to(torch.bfloat16)


def _decode_records(records: torch.Tensor, n_src: int, n_elems: int, chunk_elems: int) -> torch.Tensor:
    """fp32 values [n_src, n_elems] of source-major records: q * 2^(byte - 127), exact (or +-Inf where it overflows)."""
    n_chunks = n_elems // chunk_elems
    rec = record_bytes(chunk_elems)
    r = records.reshape(-1)[:n_src * n_chunks * rec].reshape(n_src * n_chunks, rec)
    q = r[:, :chunk_elems].contiguous().view(torch.float8_e4m3fn).float().reshape(-1, BLOCK)
    s = ue8m0(r[:, chunk_elems:chunk_elems + chunk_elems // BLOCK].reshape(-1))
    return (q * s[:, None]).reshape(n_src, n_elems)


def ref_reduce_fp8(records: torch.Tensor, n_src: int, n_elems: int, chunk_elems: int, local=None, residual=None):
    """Reference of :func:`reduce_fp8`; runs on CPU or GPU.  Returns (bf16 sum, K3 records of the sum), and with
    ``residual`` (fp32, ``n_elems``) ``(bf16, records, new residual)``: the residual is added to the sum last, one fp32
    add, and the bf16 output and the records both hold that value.  With a residual every add saturates
    (:func:`_ef_add`): finite operands whose sum overflows give +-FLT_MAX, so finite records and a finite addend give
    finite records and residuals.

    The sum starts from ``local`` (bf16, exact in fp32) when given, else from source 0, and adds the other sources in
    source order, one fp32 add each: only the adds round.  The records quantise that fp32 sum with the rule of every
    producer (:func:`quantize_blocks`), so a block whose finite sum overflows to +-Inf gets scale byte 254, NaN where the
    Inf is and +-0 beside it."""
    d = _decode_records(records, n_src, n_elems, chunk_elems)
    if local is not None:
        acc, first = local.reshape(-1).float().to(d.device), 0
    else:
        acc, first = d[0], 1
    add = torch.add if residual is None else _ef_add
    for s in range(first, n_src):
        acc = add(acc, d[s])
    if residual is None:
        return acc.to(torch.bfloat16), _quantized_records(acc, chunk_elems)
    acc = _ef_add(acc, residual.reshape(-1).float().to(acc.device))
    recs = _quantized_records(acc, chunk_elems)
    return acc.to(torch.bfloat16), recs, _ef_residual(acc, recs, chunk_elems)


def ref_allreduce_fp8(xs, chunk_elems: int, residuals=None):
    """Reference of the fp8 ring all-reduce (:class:`~rocnrdma_b200.parallel.ring_fp8.RingAllreduceFp8`), bit for bit;
    runs on CPU or GPU.  ``xs``: the N ranks' bf16 tensors of n elements each.  Returns the bf16 result every rank holds.

    ``residuals``: the N ranks' fp32 error-feedback residuals of n elements each (``error_feedback=True``); then returns
    ``(out, new residuals)``.  Rank q quantises every shard once -- shard q in its pack, shard (q-1-k) mod N in reduce hop
    k -- and shard s of its residual is the error it made there: the pack and each hop quantise ``value + residual`` and
    keep what the records lost (:func:`ref_pack_fp8`, :func:`ref_reduce_fp8`).  Every add of those steps saturates at
    +-FLT_MAX, so finite inputs give a finite output and finite residuals on every run.

    Shard s (elements ``[s * n / N, (s + 1) * n / N)``) starts as ``ref_pack_fp8(xs[s])`` on rank s and is reduced with
    ``xs[s + 1], ..., xs[s - 1]`` (indices mod N) in ring order, one :func:`ref_reduce_fp8` hop each (the addend first,
    then the decoded records, one fp32 add, then re-quantised); the final records are unpacked.  The order is fixed, so
    the result is deterministic, but it depends on which rank holds which tensor."""
    N = len(xs)
    n = xs[0].numel()
    m = n // N
    out = torch.empty(n, dtype=torch.bfloat16, device=xs[0].device)
    ef = residuals is not None
    if ef:
        new = [r.reshape(-1).float().clone() for r in residuals]
    for s in range(N):
        part = slice(s * m, (s + 1) * m)
        if ef:
            recs, new[s][part] = ref_pack_fp8(xs[s].reshape(-1)[part], chunk_elems, residual=residuals[s].reshape(-1)[part])
        else:
            recs = ref_pack_fp8(xs[s].reshape(-1)[part], chunk_elems)
        for h in range(1, N):
            q = (s + h) % N
            if ef:
                _, recs, new[q][part] = ref_reduce_fp8(recs, 1, m, chunk_elems, local=xs[q].reshape(-1)[part],
                                                       residual=residuals[q].reshape(-1)[part])
            else:
                _, recs = ref_reduce_fp8(recs, 1, m, chunk_elems, local=xs[q].reshape(-1)[part])
        out[part] = ref_unpack_fp8(recs, m, chunk_elems).to(out.device)
    return (out, new) if ef else out


def ref_allgather_fp8(shards, chunk_elems: int):
    """Reference of the fp8 ring all-gather (:class:`~rocnrdma_b200.parallel.allgather_fp8.RingAllgatherFp8`), bit for
    bit; runs on CPU or GPU.  ``shards``: the N ranks' bf16 tensors of the same number of elements, a multiple of
    ``chunk_elems``.  Returns ``(bf16 gathered, gathered records)``: shard s's K3 records (:func:`ref_pack_fp8`) at record
    ``s * R``, and their dequantisation (:func:`ref_unpack_fp8`) at element ``s * n``.  Every rank holds both."""
    recs = torch.cat([ref_pack_fp8(x.reshape(-1), chunk_elems) for x in shards])
    n = sum(x.numel() for x in shards)
    return ref_unpack_fp8(recs, n, chunk_elems), recs


def ref_alltoall_fp8(xs, chunk_elems: int):
    """Reference of the fp8 all-to-all (:class:`~rocnrdma_b200.parallel.alltoall_fp8.AllToAllFp8`), bit for bit; runs on
    CPU or GPU.  ``xs``: the N ranks' bf16 tensors of N equal shards each, shard d going to rank d.  Returns ``(outs,
    records)``, one entry per rank q: ``records[q]`` is what lands on rank q, slot s holding :func:`ref_pack_fp8` of rank
    s's shard q, and ``outs[q]`` its dequantisation (:func:`ref_unpack_fp8`), shard s at element ``s * n``, as
    ``torch.distributed.all_to_all_single`` lays it out with equal splits."""
    N = len(xs)
    m = xs[0].numel() // N
    records = [torch.cat([ref_pack_fp8(xs[s].reshape(-1)[q * m:(q + 1) * m], chunk_elems) for s in range(N)])
               for q in range(N)]
    return [ref_unpack_fp8(r, N * m, chunk_elems) for r in records], records


# ------------------------------------------------------------------ reduce
MAX_SOURCES = 8


@dataclass
class ReduceResult:
    status: str
    t_start_ns: int
    t_end_ns: int
    records_reduced: int
    records_posted: int
    t_first_post_ns: int
    t_reduce_end_ns: int
    hbm_bytes: int = 0            # bytes the kernel reads and writes in HBM (sources, addend, outputs); 0 from parse_reduce

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    @property
    def device_ns(self) -> int:
        return self.t_end_ns - self.t_start_ns

    @property
    def hbm_gbps(self) -> float:
        """HBM bytes moved (read + written) per second of device time."""
        return self.hbm_bytes / max(self.device_ns, 1)


def parse_reduce(view, hbm_bytes: int = 0) -> ReduceResult:
    """Decode the record :func:`reduce_fp8` leaves in its scratch slot (for ``sync=False`` callers)."""
    return L.decode_as(ReduceResult, view, REDUCE_WORDS, hbm_bytes=hbm_bytes)


def reduce_fp8(ctx, records: torch.Tensor, n_src: int, n_elems: int, chunk_elems: int = 1 << 20, *, local=None, out=None,
               out_mr=None, qp=None, dst_mr=None, dst_off: int = 0, with_imm: bool = False, signal_every: int = 1,
               post_only: bool = False, ready=None, grid: int = 0, timeout_ms: int = 2000, stream=None, sync: bool = True,
               scratch_slot: int = SLOT["reduce"], imm_base: int = 0, result_off=None, residual=None):
    """Sum ``n_src`` sources of K3 chunk records, plus an optional bf16 addend, as the records land, and re-pack and forward
    the sum: one hop of a reduce-scatter ring in one kernel.

    ``records`` holds the sources back to back: record r of source s at ``(s * n_rec + r) * record_bytes(chunk_elems)``
    (``n_rec = n_elems // chunk_elems``).  Every decoded element is q * 2^(byte - 127) in fp32; the sum starts from
    ``local`` (bf16, ``n_elems``) or from source 0 and adds the other sources in source order, one fp32 add each
    (:func:`ref_reduce_fp8` reproduces it bit for bit).  Outputs, at least one: ``out`` (bf16, ``n_elems``, round to
    nearest even) and ``out_mr`` (a registered region that receives the K3 records of the fp32 sum).

    With ``qp`` and ``dst_mr`` each record of ``out_mr`` is one RDMA WRITE (WRITE_IMM with immediate = record id when
    ``with_imm``) to ``dst_mr`` at ``dst_off + r * record_bytes``, posted by the CTA that completes the record; the last
    CTA posts a flush and waits for it unless ``post_only``, as :func:`pack_fp8_write` does.  With ``ready`` (int64 CUDA
    tensor of ``n_src * n_rec`` arrival words, source s in ``ready[s * n_rec:(s + 1) * n_rec]``, as ``recv_consume`` and
    :func:`~rocnrdma_b200.ops.read_records` set them) every step waits for the words of all sources of the records it
    reads; a word still 0 after ``timeout_ms`` ends the kernel with ``TIMEOUT``, and a record not reduced is never posted.
    Two reductions that run at once need different ``scratch_slot`` values (0..7; the defaults are ``ops.launch.SLOT``).
    ``imm_base`` offsets the immediates (``imm_base + r``), so that the records of several hops that reach one QP stamp
    different arrival words; ``result_off`` is :func:`~rocnrdma_b200.ops.launch.result_offset`'s.

    ``residual``: error feedback, an fp32 CUDA tensor of ``n_elems`` (contiguous, 32-byte aligned) read and written in
    place.  It is added to the sum last, one fp32 add; ``out`` and the records hold that value, and the residual then
    holds what the records lost (0 where the value or its decode is not finite), as :func:`ref_reduce_fp8` computes it.
    With a residual every add (the addend's, each source's and the residual's) saturates: finite operands whose sum
    overflows give +-FLT_MAX, so finite inputs give finite records and residuals.  ``out`` is still that value rounded
    to bf16, which is +-Inf above bf16's largest value.
    It needs ``out_mr``, and P = 1, or P = 2 with ``local`` (the variants a ring hop uses).

    Returns a :class:`ReduceResult`, or ``(result view, stream)`` with ``sync=False`` (decode with :func:`parse_reduce`)."""
    n_src, n_elems, chunk_elems = int(n_src), int(n_elems), int(chunk_elems)
    if not 1 <= n_src <= MAX_SOURCES:
        raise ValueError(f"n_src={n_src}: 1..{MAX_SOURCES} sources")
    if n_elems <= 0 or chunk_elems <= 0 or n_elems % TILE_ELEMS or chunk_elems % TILE_ELEMS or n_elems % chunk_elems:
        raise ValueError(f"n_elems and chunk_elems must be multiples of {TILE_ELEMS}, n_elems of chunk_elems")
    dev = ctx.device
    n_rec = n_elems // chunk_elems
    wire = staging_bytes(n_elems, chunk_elems)
    if not isinstance(records, torch.Tensor) or not records.is_cuda or records.device.index != dev or not records.is_contiguous():
        raise ValueError(f"records must be a contiguous tensor on cuda:{dev}")
    if records.numel() * records.element_size() < n_src * wire:
        raise ValueError(f"records hold {records.numel() * records.element_size()} bytes; {n_src} sources of {n_rec} "
                         f"records need {n_src * wire}")
    if records.data_ptr() & 31:
        raise ValueError("records must be 32-byte aligned (256-bit loads)")
    local_addr = 0 if local is None else L.tensor_ptr(local, torch.bfloat16, dev, "local", n_elems, exact=True, align=32)
    out_addr = 0 if out is None else L.tensor_ptr(out, torch.bfloat16, dev, "out", n_elems, exact=True, align=32)
    if out is None and out_mr is None:
        raise ValueError("reduce_fp8 needs an output: out (bf16) and / or out_mr (records)")
    if out_mr is not None:
        if out_mr.length < wire:
            raise ValueError(f"out_mr holds {out_mr.length} bytes; the records of the sum need {wire}")
        if out_mr.addr & 31:
            raise ValueError("out_mr must be 32-byte aligned")
    if qp is not None and (out_mr is None or dst_mr is None):
        raise ValueError("posting (qp) needs out_mr and dst_mr")
    if dst_mr is not None and qp is None:
        raise ValueError("dst_mr without qp: nothing would post to it")
    if dst_mr is not None and (dst_off < 0 or dst_off + wire > dst_mr.length):
        raise ValueError(f"{n_rec} records of {record_bytes(chunk_elems)} bytes at dst_off={dst_off} do not fit dst_mr "
                         f"({dst_mr.length} bytes)")
    if not 0 <= imm_base or imm_base + n_rec > 1 << 32:
        raise ValueError(f"imm_base={imm_base}: the immediates imm_base + r of {n_rec} records must fit 32 bits")
    res_ptr = 0
    if residual is not None:
        if out_mr is None:
            raise ValueError("residual= needs out_mr: the residual is what the records of the sum lose")
        if n_src > (2 if local is not None else 1):
            raise ValueError(f"residual= with n_src={n_src}: error feedback runs with P = 1, or P = 2 with local")
        res_ptr = L.tensor_ptr(residual, torch.float32, dev, "residual", n_elems, exact=True, align=32)
    ready_addr = 0 if ready is None else L.tensor_ptr(ready, torch.int64, dev, "ready", n_src * n_rec)
    # [n_rec] tiles done per record ; CTAs done ; abort flag ; records reduced
    counters = L.counters(ctx, n_rec + 3, scratch_slot)
    lib = N.load()
    ws = work_stream(ctx, stream)
    res_addr, res_view = L.result(ctx, L.result_offset(scratch_slot, result_off))
    hbm = n_src * wire + (2 * n_elems if local is not None else 0) + (2 * n_elems if out is not None else 0) + \
        (wire if out_mr is not None else 0) + (8 * n_elems if residual is not None else 0)
    rc = lib.rn_k_reduce_fp8(_stream_ptr(ws), grid, records.data_ptr(), n_src, local_addr, out_addr,
                             out_mr.addr if out_mr is not None else 0, n_elems, chunk_elems, ready_addr,
                             qp.dev_ptr if qp is not None else 0, out_mr.addr if out_mr is not None else 0,
                             out_mr.lkey if out_mr is not None else 0, dst_mr.addr + dst_off if dst_mr is not None else 0,
                             dst_mr.rkey if dst_mr is not None else 0, int(with_imm) | (2 if post_only else 0), signal_every,
                             counters, res_addr, timeout_ms, imm_base, res_ptr)
    return L.finish(rc, "reduce_fp8", res_view, ws, sync, parse_reduce, hbm)


def ref_reduce_scatter_fp8(xs, chunk_elems: int):
    """Reference of the fp8 ring reduce-scatter (:class:`~rocnrdma_b200.parallel.reduce_scatter_fp8.RingReduceScatterFp8`),
    bit for bit; runs on CPU or GPU.  ``xs``: the N ranks' tensors of n elements each, bf16 (``run``) or fp32 partials
    (``run_gemm``, whose records are one 128-row panel each: ``chunk_elems = 128 * Nb``).  Returns the list of the N
    ranks' bf16 shards, rank s's being the reduction of elements ``[s * n / N, (s + 1) * n / N)``.

    Shard s starts as :func:`ref_pack_fp8` of rank s+1's part and is reduced with the parts of ranks s+2, ..., s (indices
    mod N), in that order, one :func:`ref_reduce_fp8` hop each (the addend first, then the decoded records, one fp32 add).
    The last hop's bf16 sum is the output: unlike the all-reduce, nothing is quantised after it."""
    N = len(xs)
    m = xs[0].numel() // N
    out = []
    for s in range(N):
        part = slice(s * m, (s + 1) * m)
        recs = ref_pack_fp8(xs[(s + 1) % N].reshape(-1)[part], chunk_elems)
        for h in range(2, N + 1):
            y, recs = ref_reduce_fp8(recs, 1, m, chunk_elems, local=xs[(s + h) % N].reshape(-1)[part])
        out.append(y)
    return out
