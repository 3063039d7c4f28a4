"""What every ops launch shares: where its result record and counters live, how the record is read back, and the end
of the launch.

Every kernel writes a 64-byte result record, 8 int64 words, into the context's 256 KiB mapped scratch: word 0 is the
status (:data:`WAIT_STATUS`), words 1 and 2 the %globaltimer at its start and end, words 3-7 its own.  Kernels that
count keep their counters in the 2 MiB device scratch, eight 256 KiB slots (``scratch_slot``): two launches that may
run at the same time need different slots.  :data:`MAPPED` and :data:`SLOT` give every default place; a caller that
runs two launches of one kind at once passes another ``scratch_off`` / ``result_off`` / ``scratch_slot``."""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import NamedTuple

import torch

from .. import _native as N

WAIT_STATUS = {0: "OK", -1: "TIMEOUT", -2: "CQE_ERROR", -3: "QP_ERROR"}

RECORD_BYTES = 64
MAPPED_BYTES = 256 << 10        # the mapped scratch (hca_host.cu)
SLOT_BYTES = 256 << 10          # one launch's share of the device scratch
N_SLOTS = 8                     # the device scratch is 2 MiB
MAX_QPS = 64                    # queue pairs of one multi-QP launch (rdma_ops.cu kMaxStreamQps)
RING_SLOT_BYTES = 4096          # the ring's result records of one device-scratch slot


class Region(NamedTuple):
    offset: int
    nbytes: int                 # at its largest: 64 per QP at MAX_QPS for the multi-QP launches


# Mapped scratch: the default result records of every launch.  The multi-QP ones take one record per QP.
MAPPED = {
    "rdma_stream": Region(0, RECORD_BYTES * MAX_QPS),
    "slot_results": Region(4096, RECORD_BYTES * N_SLOTS),       # K3, K5, the reduce and the GEMMs: one per scratch_slot
    "recv_consume": Region(8192, RECORD_BYTES),
    "shared_post_stress": Region(12288, RECORD_BYTES),
    "atomic_stream": Region(16384, RECORD_BYTES * MAX_QPS),
    "put_signal": Region(20480, RECORD_BYTES),
    "signal_wait": Region(20544, RECORD_BYTES),
    "put_inline": Region(24576, RECORD_BYTES * MAX_QPS),
    "cq_watch": Region(30720, RECORD_BYTES),
    "write_read": Region(32768, RECORD_BYTES),
    "gather_stream": Region(36864, RECORD_BYTES * MAX_QPS),
    "read_records": Region(40960, RECORD_BYTES),
    "ring_results": Region(128 << 10, RING_SLOT_BYTES * N_SLOTS),  # parallel.ring_fp8: RING_SLOT_BYTES per scratch_slot
}

# Device scratch: the default slot of every launch that keeps counters.
SLOT = {"pack": 0, "unpack": 1, "gemm_send": 2, "gemm_mxfp8": 3, "reduce": 4}
# shared_post_stress's one counter lies inside slot 3, gemm_mxfp8's: the two never run at the same time.
SHARED_POST_STRESS_COUNTER = Region(900 << 10, RECORD_BYTES)


def scratch_offset(offset, n: int = 1) -> int:
    """``offset`` of ``n`` result records in the mapped scratch: a non-negative multiple of 64 that leaves room for them."""
    offset = int(offset)
    if offset < 0 or offset % RECORD_BYTES or offset + n * RECORD_BYTES > MAPPED_BYTES:
        raise ValueError(f"scratch offset {offset}: a non-negative multiple of {RECORD_BYTES} with {n} records of room in "
                         f"the {MAPPED_BYTES}-byte mapped scratch")
    return offset


def result_offset(scratch_slot: int, result_off=None) -> int:
    """Offset in the mapped scratch of a launch's 64-byte result record: ``result_off``, else ``4096 + scratch_slot * 64``.
    The host zeroes the record when it enqueues the launch, not when the launch runs, so launches queued on one stream
    before the first of them has run need one record each."""
    if result_off is None:
        return MAPPED["slot_results"].offset + scratch_slot * RECORD_BYTES
    return scratch_offset(result_off)


def ring_result_offset(scratch_slot: int, i: int) -> int:
    """Offset of the ring's result record ``i`` (< ``RING_SLOT_BYTES // 64``) for the plan in ``scratch_slot``."""
    return MAPPED["ring_results"].offset + scratch_slot * RING_SLOT_BYTES + RECORD_BYTES * i


def result(ctx, offset, n: int = 1):
    """(address, view) of ``n`` result records at ``offset`` in ``ctx``'s mapped scratch (see :func:`scratch_offset`)."""
    return ctx.scratch(n * RECORD_BYTES, offset=scratch_offset(offset, n))


def counter_bytes(n_words: int) -> int:
    """Device scratch a launch with ``n_words`` 32-bit counters takes: the counters, rounded up to 8 bytes, then the
    three 64-bit words the kernels post records through."""
    return (int(n_words) * 4 + 7) // 8 * 8 + 24


def counters(ctx, n_words: int, scratch_slot: int) -> int:
    """Address of a launch's zeroed counters in device-scratch slot ``scratch_slot``."""
    nb = counter_bytes(n_words)
    if nb > SLOT_BYTES:
        raise ValueError(f"{n_words} counters need {nb} bytes; a scratch slot holds {SLOT_BYTES}")
    if not 0 <= scratch_slot < ctx.dev_scratch_bytes // SLOT_BYTES:
        raise ValueError(f"scratch_slot={scratch_slot}: the device scratch has {ctx.dev_scratch_bytes // SLOT_BYTES} slots")
    return ctx.dev_scratch(nb, offset=scratch_slot * SLOT_BYTES)


# ---------------------------------------------------------------- result records
def decode(view, fields=(), i: int = 0) -> dict:
    """Result record ``i`` of ``view``: the header every kernel writes -- ``status``, ``t_start_ns``, ``t_end_ns`` and
    ``device_ns`` -- and words 3, 4, ... named by ``fields`` (``None`` skips a word)."""
    w = (C.c_int64 * 8).from_buffer(view, i * RECORD_BYTES)
    d = dict(status=WAIT_STATUS.get(w[0], str(w[0])), t_start_ns=w[1], t_end_ns=w[2], device_ns=w[2] - w[1])
    d.update((f, w[3 + k]) for k, f in enumerate(fields) if f is not None)
    return d


def decode_as(cls, view, fields, **extra):
    """A ``cls`` dataclass of :func:`decode`'s words (each header word only where ``cls`` has that field) and ``extra``."""
    names = {f.name for f in dataclasses.fields(cls)}
    return cls(**{k: v for k, v in decode(view, fields).items() if k in names}, **extra)


# ---------------------------------------------------------------- the launch
def finish(rc: int, name: str, view, ws, sync: bool, parse, *args):
    """The end of every launch: raise if it failed; else ``(view, ws)`` without ``sync``, or wait and return
    ``parse(view, *args)`` (None when ``parse`` is None)."""
    if rc:
        raise N.NativeError(f"{name} launch failed ({rc})")
    if not sync:
        return view, ws
    ws.synchronize()
    return None if parse is None else parse(view, *args)


def qp_array(qps):
    """``qps`` (one queue pair or a list of them) as a list, and the ``c_uint64`` array of their device pointers."""
    if not isinstance(qps, (list, tuple)):
        qps = [qps]
    return qps, (C.c_uint64 * len(qps))(*[q.dev_ptr for q in qps])


def tensor_ptr(t, dtype, device: int, what: str, n: int, exact: bool = False, align: int = 1) -> int:
    """Address of ``t``: a contiguous ``dtype`` tensor on cuda:``device``, ``align``-byte aligned, of ``n`` elements (at
    least ``n`` unless ``exact``); ``ValueError`` naming ``what`` otherwise.  The values are never read on the host (that
    would synchronise)."""
    if not isinstance(t, torch.Tensor) or t.dtype != dtype:
        raise ValueError(f"{what} must be a {str(dtype).removeprefix('torch.')} tensor, not "
                         f"{getattr(t, 'dtype', type(t).__name__)}")
    if not t.is_cuda or t.device.index != device:
        raise ValueError(f"{what} must be on cuda:{device}, not {t.device}")
    if not t.is_contiguous() or t.data_ptr() % align:
        raise ValueError(f"{what} must be contiguous" + (f" and {align}-byte aligned (256-bit loads / stores)" if align > 1 else ""))
    if t.numel() < n or (exact and t.numel() != n):
        raise ValueError(f"{what} holds {t.numel()} elements; {'' if exact else 'at least '}{n} are needed")
    return t.data_ptr()
