"""K1 / K2 / K6 wrappers: GPU-initiated RDMA streams and verification helpers."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List

import torch

from .. import _native as N
from . import launch as L
from .launch import MAPPED, WAIT_STATUS  # noqa: F401  (WAIT_STATUS: ops.rdma.WAIT_STATUS is public)


def _stream_ptr(stream=None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def work_stream(ctx, stream=None):
    """Stream for engine-facing kernels: never the legacy default stream (see Context.stream)."""
    # native launchers use the calling thread's current device: make it this context's (creating a
    # second Context, or torch work on another GPU, may have changed it)
    N.load().rn_set_device(ctx.device)
    if getattr(ctx, "auto_sweep", True):
        ctx.sweep_revoked()               # driver-originated revocation check before a kernel may post (one driver query per MR)
    if stream is not None and int(stream.cuda_stream) != 0:
        return stream
    cur = torch.cuda.current_stream(ctx.device)
    if int(cur.cuda_stream) != 0:
        return cur
    ws = ctx.stream
    # The caller's tensors were produced on the legacy default stream (torch.zeros / randn / copies): order the work stream
    # after it, or the kernel races with their initialisation (compute-sanitizer's slower kernels made exactly that visible:
    # a zero-fill landing after the GEMM had written C).  Not while an engine is resident: anything recorded on the legacy
    # stream then queues behind the persistent kernel (DESIGN.md 3.2) and the poster it gates would never start --
    # allocate and initialise before engine_start(), as the residency rules say.
    if not ctx.engine_running:
        ws.wait_stream(cur)
    return ws


@dataclass
class StreamResult:
    status: List[str]
    t_start_ns: List[int]
    t_end_ns: List[int]
    done: List[int]
    bytes_per_msg: int

    @property
    def ok(self) -> bool:
        return all(s == "OK" for s in self.status)

    @property
    def device_ns(self) -> int:
        """Device-timed span: first QP start to last QP end (%globaltimer)."""
        return max(self.t_end_ns) - min(self.t_start_ns)

    @property
    def gbps(self) -> float:
        return sum(self.done) * self.bytes_per_msg / max(self.device_ns, 1)

    @property
    def us_per_msg(self) -> float:
        return self.device_ns / 1e3 / max(max(self.done), 1)


def rdma_stream(qps, opcode: int, src_mr, dst_mr, nbytes: int, iters: int = 1, window: int = 0,
                signal_every: int = 1, burst: int = 1, stride: int = 0, slot_stride: int = 0, nslots: int = 1,
                timeout_ms: int = 2000, stream=None, sync: bool = True, out=None, post_only: bool = False,
                fence_every: int = 0):
    """Launch the device poster: one CTA per QP posts ``iters`` work requests of
    ``nbytes`` (window-limited), polls its CQ on the device and returns device times.
    ``burst`` work requests share one slot reservation and one doorbell (perftest ``--post_list``),
    ``signal_every`` is the CQ moderation (``--cq-mod``); both are clamped so the window can always drain.
    ``fence_every=k`` sets the fence flag (``IBV_SEND_FENCE``) on every k-th work request of each QP (the k-th, 2k-th,
    ...): it moves no byte before every earlier work request of its QP has finished.  0 fences nothing.

    For RDMA_READ ``src_mr`` is the local destination and ``dst_mr`` the remote source,
    mirroring the laddr/raddr roles in the WQE.  ``post_only`` skips the final completion wait (``iters`` must fit
    the window): the work is reaped later -- by ``Context.engine_run_oneshot`` under a profiler, or by the caller.
    A work request longer than ``Context.max_msg_bytes`` completes with ``LOCAL_LENGTH_ERR`` (status ``CQE_ERROR``);
    ``nbytes`` outside ``[0, 2**32)`` raises ``ValueError``.
    """
    nbytes = N.byte_count(nbytes)
    lib = N.load()
    qps, qp_arr = L.qp_array(qps)
    ctx = qps[0].ctx
    ws = work_stream(ctx, stream)
    nq = len(qps)
    out_addr, out_view = L.result(ctx, MAPPED["rdma_stream"].offset, nq) if out is None else out
    rc = lib.rn_k_rdma_stream(_stream_ptr(ws), qp_arr, nq, opcode | (0x80000000 if post_only else 0), src_mr.addr, src_mr.lkey,
                              dst_mr.addr if dst_mr is not None else 0, dst_mr.rkey if dst_mr is not None else 0,
                              stride, nbytes, iters, window, signal_every, burst, slot_stride, nslots, timeout_ms, out_addr,
                              fence_every)
    return L.finish(rc, "rdma_stream", out_view, ws, sync, parse_stream_out, nq, nbytes)


def parse_stream_out(out, nqp: int, nbytes: int) -> StreamResult:
    o = [L.decode(out, ("done",), i) for i in range(nqp)]
    return StreamResult(status=[r["status"] for r in o], t_start_ns=[r["t_start_ns"] for r in o],
                        t_end_ns=[r["t_end_ns"] for r in o], done=[r["done"] for r in o], bytes_per_msg=nbytes)


WRITE_READ_MODES = {"fenced": 0, "wait": 1, "one_call": 2}


def write_read(qp, src_mr, dst_mr, back_mr, nbytes: int, iters: int = 1, mode: str = "fenced", timeout_ms: int = 2000,
               stream=None, scratch_off: int = MAPPED["write_read"].offset) -> dict:
    """A WRITE followed by a READ of the same bytes, posted from one GPU thread ``iters`` times: ``nbytes`` from
    ``src_mr`` to ``dst_mr``, then back from ``dst_mr`` into ``back_mr`` (all at offset 0), waiting for the READ's
    completion each time.  ``mode`` says how the READ is kept behind the WRITE: ``"fenced"`` posts both under one doorbell
    with the READ fenced; ``"wait"`` waits for the WRITE's completion before posting the READ (the only way without the
    fence); ``"one_call"`` posts them with ``dev::rdma_write`` and ``dev::rdma_read(..., fence=true)``.  Returns
    ``dict(status, done, device_ns, mean_ns, min_ns)`` (per pair: post to the READ's completion).  ``nbytes`` as in
    :func:`rdma_stream`."""
    nbytes = N.byte_count(nbytes)
    ctx = qp.ctx
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    rc = N.load().rn_k_write_read(_stream_ptr(ws), qp.dev_ptr, src_mr.addr, src_mr.lkey, dst_mr.addr, dst_mr.rkey, back_mr.addr,
                                  back_mr.lkey, nbytes, iters, WRITE_READ_MODES[mode], timeout_ms, out_addr)
    return L.finish(rc, "write_read", out_view, ws, True, _parse_write_read)


def _parse_write_read(view) -> dict:
    d = L.decode(view, ("done", "sum_ns", "min_ns"))
    return dict(status=d["status"], done=d["done"], device_ns=d["device_ns"], mean_ns=d["sum_ns"] / max(d["done"], 1),
                min_ns=d["min_ns"] if d["done"] else 0)


def fill_random(t: torch.Tensor, seed: int = 1, stream=None):
    N.load().rn_k_fill_random(_stream_ptr(stream), t.data_ptr(), t.numel() * t.element_size(), seed)
    return t


def fill_bf16(t: torch.Tensor, seed: int = 1, scale: float = 1.0, stream=None):
    assert t.dtype == torch.bfloat16
    N.load().rn_k_fill_bf16(_stream_ptr(stream), t.data_ptr(), t.numel(), seed, scale)
    return t


def checksum(t: torch.Tensor, stream=None) -> int:
    out = torch.zeros(1, dtype=torch.int64, device=t.device)
    N.load().rn_k_checksum(_stream_ptr(stream), t.data_ptr(), t.numel() * t.element_size(), out.data_ptr())
    return int(out.item()) & 0xFFFFFFFFFFFFFFFF


def compare(a: torch.Tensor, b: torch.Tensor, nbytes=None, stream=None) -> int:
    """Number of mismatching 16-byte words (aligned) or bytes (unaligned)."""
    n = a.numel() * a.element_size() if nbytes is None else nbytes
    out = torch.zeros(1, dtype=torch.int64, device=a.device)
    N.load().rn_k_compare(_stream_ptr(stream), a.data_ptr(), b.data_ptr(), n, out.data_ptr())
    return int(out.item())


def l2_flush(scratch: torch.Tensor, value: int = 0, stream=None):
    N.load().rn_k_l2_flush(_stream_ptr(stream), scratch.data_ptr(), scratch.numel() * scratch.element_size(), value)


def recv_consume(qp, n: int, max_imm: int = 0, stamps=None, timeout_ms: int = 2000, stream=None, sync: bool = True,
                 scratch_off: int = MAPPED["recv_consume"].offset, prepost_mr=None, prepost_bytes: int = 0):
    """Receive-side consumer kernel on ``qp``'s GPU: waits for ``n`` arrivals (SEND / RDMA_WRITE_IMM) on the
    receive CQ and, if ``stamps`` (int64 tensor on that GPU) is given, stamps %globaltimer per immediate."""
    ctx = qp.ctx
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    # prepost_mr: the kernel posts its own n receive WQEs from the device before polling (buffer i at offset i * prepost_bytes)
    rc = N.load().rn_k_recv_consume(_stream_ptr(ws), qp.dev_ptr, n, max_imm, stamps.data_ptr() if stamps is not None else 0,
                                    out_addr, timeout_ms, prepost_mr.addr if prepost_mr is not None else 0,
                                    prepost_mr.lkey if prepost_mr is not None else 0,
                                    prepost_bytes if prepost_mr is not None else 0xFFFFFFFF)
    return L.finish(rc, "recv_consume", out_view, ws, sync, parse_recv)


RECV_WORDS = ("seen", "bytes")
MAX_RECV_QPS = 7                # queue pairs of one recv_consume_qps launch (rdma_ops.cu kMaxRecvQps)


def parse_recv(view) -> dict:
    return L.decode(view, RECV_WORDS)


def recv_consume_qps(qps, n: int, prepost, prepost_mr, max_imm: int = 0, stamps=None, timeout_ms: int = 2000,
                     stream=None, sync: bool = True, scratch_off: int = MAPPED["recv_consume"].offset):
    """:func:`recv_consume` over several receive queue pairs that share one receive CQ (a mesh's receiver: one QP per
    source).  The kernel first posts ``prepost[i]`` zero-length receive WQEs on ``qps[i]`` (``prepost_mr`` gives their
    address and lkey; RDMA_WRITE_IMM ignores the buffer), then takes ``n`` completions from the shared CQ, whichever QP
    they belong to, and with ``stamps`` stamps %globaltimer into word ``imm`` of each one whose immediate is below
    ``max_imm``.  1..7 queue pairs.  Returns ``dict(status, seen, bytes, ...)``, or ``(view, stream)`` with
    ``sync=False`` (decode with :func:`parse_recv`)."""
    qps, qp_arr = L.qp_array(qps)
    if not 1 <= len(qps) <= MAX_RECV_QPS:
        raise ValueError(f"{len(qps)} queue pairs: recv_consume_qps takes 1..{MAX_RECV_QPS}")
    if any(q.rcq is not qps[0].rcq for q in qps):
        raise ValueError("recv_consume_qps: the queue pairs must share one receive CQ")
    prepost = [int(k) for k in prepost]
    if len(prepost) != len(qps) or any(k < 0 or k > q.rq_depth for k, q in zip(prepost, qps)):
        raise ValueError("prepost: one count per queue pair, each between 0 and its receive queue's depth")
    ctx = qps[0].ctx
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    rc = N.load().rn_k_recv_consume_qps(_stream_ptr(ws), qp_arr, (C.c_uint32 * len(qps))(*prepost), len(qps), n, max_imm,
                                        stamps.data_ptr() if stamps is not None else 0, out_addr, timeout_ms,
                                        prepost_mr.addr, prepost_mr.lkey)
    return L.finish(rc, "recv_consume_qps", out_view, ws, sync, parse_recv)


def shared_post_stress(qp, src_mr, dst_mr, ctas: int = 64, per_cta: int = 64, timeout_ms: int = 3000, stream=None):
    """``ctas`` CTAs hammer one QP with ``per_cta`` 64-byte writes each through the shared submit."""
    ctx = qp.ctx
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, MAPPED["shared_post_stress"].offset)
    counter = ctx.dev_scratch(L.SHARED_POST_STRESS_COUNTER.nbytes, offset=L.SHARED_POST_STRESS_COUNTER.offset)
    rc = N.load().rn_k_shared_post_stress(_stream_ptr(ws), qp.dev_ptr, ctas, src_mr.addr, src_mr.lkey, dst_mr.addr, dst_mr.rkey,
                                          per_cta, counter, out_addr, timeout_ms)
    return L.finish(rc, "shared_post_stress", out_view, ws, True, L.decode, ("posted",))


# ---------------------------------------------------------------- remote atomics and put-with-signal
_OP_CS, _OP_FA = 0x11, 0x12


def atomic_stream(qps, op: str, target_mr, fetch_mr, iters: int, add: int = 1, compare: int = 0, swap: int = 0,
                  chain: bool = False, target_stride: int = 0, window: int = 0, burst: int = 1, signal_every: int = 1,
                  timeout_ms: int = 2000, stream=None, sync: bool = True, scratch_off: int = MAPPED["atomic_stream"].offset):
    """Device-posted 8-byte remote atomics: one warp per QP posts ``iters`` FETCH_AND_ADD (``op="fa"``: ``add``) or
    COMPARE_AND_SWAP (``op="cs"``: ``compare`` / ``swap``) work requests with the same windowed, bursted poster as
    :func:`rdma_stream`.  QP ``c`` targets the u64 at ``target_mr.addr + c * target_stride`` (``target_stride=0``: every
    QP on one word); its op ``i`` writes the original value to ``fetch_mr.addr + (c * iters + i) * 8``, so ``fetch_mr``
    needs ``len(qps) * iters * 8`` bytes.  ``chain=True`` (CS only) posts CS(compare=i, swap=i+1): on a word that
    starts at 0 every one of them succeeds exactly when the QP executes its atomics in order.  Returns a
    :class:`StreamResult` (``us_per_msg`` = device time per atomic of one QP)."""
    if op not in ("fa", "cs"):
        raise ValueError("op must be 'fa' or 'cs'")
    lib = N.load()
    qps, qp_arr = L.qp_array(qps)
    ctx = qps[0].ctx
    nq = len(qps)
    if fetch_mr.length < nq * iters * 8:
        raise ValueError(f"fetch_mr holds {fetch_mr.length} bytes; {nq} QPs x {iters} atomics need {nq * iters * 8}")
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off, nq)
    m = 0xFFFFFFFFFFFFFFFF
    rc = lib.rn_k_atomic_stream(_stream_ptr(ws), qp_arr, nq, _OP_FA if op == "fa" else _OP_CS, int(chain), target_mr.addr,
                                target_mr.rkey, target_stride, fetch_mr.addr, fetch_mr.lkey, add & m, compare & m, swap & m,
                                iters, window, signal_every, burst, timeout_ms, out_addr)
    return L.finish(rc, "atomic_stream", out_view, ws, sync, parse_stream_out, nq, 8)


def _fetch_sink(ctx):
    """An 8-byte-per-slot local buffer for fetched values nobody reads (registered once per context)."""
    if getattr(ctx, "_atomic_sink", None) is None:
        t = torch.zeros(4096, dtype=torch.uint8, device=f"cuda:{ctx.device}")
        ctx._atomic_sink = ctx.reg_mr(t)
    return ctx._atomic_sink


def put_signal(qp, src_mr, dst_mr, nbytes: int, sig_mr, sig_off: int = 0, fetch_mr=None, add: int = 1, iters: int = 1,
               window: int = 0, slot_stride: int = 0, nslots: int = 1, timeout_ms: int = 2000, stream=None,
               sync: bool = True, scratch_off: int = MAPPED["put_signal"].offset):
    """Device-posted put-with-signal: message ``i`` is an RDMA WRITE of ``nbytes`` from ``src_mr`` to ``dst_mr`` (slot
    ``i % nslots`` at ``slot_stride``) followed by a FETCH_AND_ADD of ``add`` on the remote u64 at
    ``sig_mr.addr + sig_off``, both published with one doorbell.  The atomic executes only after the WRITE has landed,
    so a receiver that sees the signal reach ``k`` (:func:`signal_wait`) may read messages ``0..k-1``.  The fetched
    values go to ``fetch_mr`` (message ``i`` at ``(i % (fetch_mr.length // 8)) * 8``); by default to a small buffer the
    context registers the first time it is needed -- pass ``fetch_mr`` when the engine is already running, since a
    first allocation then waits for it.  ``window`` bounds the messages in flight (0: the send queue does).  Returns a
    :class:`StreamResult` (``us_per_msg`` = device time per message).  ``nbytes`` as in :func:`rdma_stream`."""
    nbytes = N.byte_count(nbytes)
    lib = N.load()
    ctx = qp.ctx
    if fetch_mr is None:
        fetch_mr = _fetch_sink(ctx)
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    rc = lib.rn_k_put_signal(_stream_ptr(ws), qp.dev_ptr, src_mr.addr, src_mr.lkey, dst_mr.addr, dst_mr.rkey, nbytes,
                             slot_stride, nslots, sig_mr.addr + sig_off, sig_mr.rkey, fetch_mr.addr, fetch_mr.lkey,
                             max(fetch_mr.length // 8, 1), add & 0xFFFFFFFFFFFFFFFF, iters, window, timeout_ms, out_addr)
    return L.finish(rc, "put_signal", out_view, ws, sync, parse_stream_out, 1, nbytes)


def put_inline(qps, values, dst_mr, nbytes: int, iters: int = 1, window: int = 0, burst: int = 1, signal_every: int = 1,
               slot_stride=None, nslots: int = 1, sig_mr=None, sig_off: int = 0, fetch_mr=None, add: int = 1,
               timeout_ms: int = 2000, stream=None, sync: bool = True, scratch_off: int = MAPPED["put_inline"].offset):
    """Device-posted inline puts (DOCA ``p`` / ``p_signal``, ``nvshmem_p``): one warp per QP posts ``iters`` RDMA WRITEs
    whose ``nbytes`` (1..28) travel inside the WQE, with the windowed, bursted poster of :func:`rdma_stream`.  Message
    ``i`` of QP ``c`` (``m = c * iters + i``) reads its bytes into registers from row ``m % rows`` of ``values`` -- a CUDA
    tensor on the QP's GPU that is never registered (a 2-D tensor: one row per message value; 1-D: rows of ``nbytes``)
    -- and writes them to ``dst_mr`` slot ``m % nslots`` at ``slot_stride`` (default ``nbytes``).
    With ``sig_mr`` each message is the inline WRITE plus a FETCH_AND_ADD of ``add`` on the u64 at
    ``sig_mr.addr + sig_off + c * 8``, built by two lanes and published with one doorbell; the atomic executes after the
    WRITE has landed, so a receiver may use :func:`signal_wait` unchanged.  Fetched values go to ``fetch_mr`` (default: the
    context's sink, see :func:`put_signal`).  ``window`` and ``burst`` count messages.  Returns a :class:`StreamResult`."""
    lib = N.load()
    qps, qp_arr = L.qp_array(qps)
    if not 1 <= nbytes <= 28:
        raise ValueError(f"inline puts carry 1..28 bytes, not {nbytes}")
    if not values.is_cuda or not values.is_contiguous():
        raise ValueError("values must be a contiguous CUDA tensor")
    row_bytes = values.stride(0) * values.element_size() if values.dim() == 2 else nbytes
    total = values.numel() * values.element_size()
    if row_bytes < nbytes or total < nbytes:
        raise ValueError(f"values rows hold {row_bytes} bytes; each message needs {nbytes}")
    rows = (total - nbytes) // row_bytes + 1
    ctx = qps[0].ctx
    nq = len(qps)
    if slot_stride is None:
        slot_stride = nbytes
    if sig_mr is not None and fetch_mr is None:
        fetch_mr = _fetch_sink(ctx)
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off, nq)
    sig = (sig_mr.addr + sig_off) if sig_mr is not None else 0
    rc = lib.rn_k_put_inline(_stream_ptr(ws), qp_arr, nq, values.data_ptr(), row_bytes, rows, dst_mr.addr, dst_mr.rkey, nbytes,
                             slot_stride, nslots, sig, sig_mr.rkey if sig_mr is not None else 0,
                             fetch_mr.addr if fetch_mr is not None else 0, fetch_mr.lkey if fetch_mr is not None else 0,
                             max(fetch_mr.length // 8, 1) if fetch_mr is not None else 1, add & 0xFFFFFFFFFFFFFFFF, iters, window,
                             signal_every, burst, timeout_ms, out_addr)
    return L.finish(rc, "put_inline", out_view, ws, sync, parse_stream_out, nq, nbytes)


GATHER_VIA = {"poster": 0, "one_call": 1}
_OP_WRITE, _OP_SEND, _OP_READ = 0x08, 0x0A, 0x10


def gather_stream(qps, opcode: int, mr0, mr1, remote_mr, nbytes: int, split: int, iters: int = 1, window: int = 0,
                  signal_every: int = 1, burst: int = 1, stride: int = 0, slot_stride: int = 0, nslots: int = 1,
                  via: str = "poster", timeout_ms: int = 2000, stream=None, sync: bool = True,
                  scratch_off: int = MAPPED["gather_stream"].offset) -> StreamResult:
    """Device-posted two-entry work requests: one warp per QP posts ``iters`` messages of ``nbytes``, each one work
    request whose scatter-gather list is cut at ``split`` bytes.  Message ``i`` of QP ``c`` uses slot offset
    ``o = c * stride + (i % nslots) * slot_stride``: entry 0 is ``split`` bytes at ``mr0.addr + o``, entry 1 the other
    ``nbytes - split`` at ``mr1.addr + o`` (the same slot of a second MR), and the remote side is ``nbytes`` at
    ``remote_mr.addr + o``.  ``OP_RDMA_WRITE`` gathers the entries there, ``OP_SEND`` into the responder's next receive
    (``remote_mr`` unused), ``OP_RDMA_READ`` scatters the remote bytes into the entries.  A zero-length entry is dropped,
    so ``split`` 0 or ``nbytes`` posts one-entry work requests.
    ``via="poster"`` uses the windowed, bursted exclusive poster of :func:`rdma_stream` (``window``, ``burst`` and
    ``signal_every`` as there); ``via="one_call"`` posts every message with ``dev::rdma_write_sg`` / ``rdma_read_sg`` /
    ``rdma_send_sg`` through the shared submit and keeps at most ``window`` in flight.  Returns a :class:`StreamResult`."""
    nbytes, split = N.byte_count(nbytes), N.byte_count(split, "split")
    if split > nbytes:
        raise ValueError(f"split={split} exceeds nbytes={nbytes}")
    if opcode not in (_OP_WRITE, _OP_READ, _OP_SEND):
        raise ValueError(f"opcode 0x{opcode:x}: gather_stream posts RDMA_WRITE, RDMA_READ or SEND")
    if via not in GATHER_VIA:
        raise ValueError(f"via must be one of {sorted(GATHER_VIA)}")
    lib = N.load()
    qps, qp_arr = L.qp_array(qps)
    ctx = qps[0].ctx
    nq = len(qps)
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off, nq)
    rc = lib.rn_k_gather_stream(_stream_ptr(ws), qp_arr, nq, opcode, mr0.addr, mr0.lkey, mr1.addr, mr1.lkey,
                                remote_mr.addr if remote_mr is not None else 0, remote_mr.rkey if remote_mr is not None else 0,
                                stride, nbytes, split, slot_stride, nslots, iters, window, signal_every, burst, GATHER_VIA[via],
                                timeout_ms, out_addr)
    return L.finish(rc, "gather_stream", out_view, ws, sync, parse_stream_out, nq, nbytes)


def signal_wait(ctx, signal, until: int, stamps=None, timeout_ms: int = 2000, stream=None, sync: bool = True,
                check=None, scratch_off: int = MAPPED["signal_wait"].offset):
    """Receiver side of :func:`put_signal`, on the GPU that holds the signal: waits until the u64 at ``signal`` (a
    tensor, a ``MemoryRegion`` or an ``(address, nbytes)`` pair; the word at its start) reaches each value ``1..until``
    in turn, with system-scope acquire loads and at most ``timeout_ms`` per arrival.  ``stamps`` (int64 tensor of at
    least ``until`` entries on that GPU) receives the %globaltimer at which value ``k + 1`` was first seen.
    ``check=(dst, src, slot_bytes, slot_stride)`` compares slot ``k`` of ``dst`` with ``src`` (``slot_bytes`` a multiple
    of 16) as soon as the signal covers message ``k``.  Returns ``dict(status, seen, mismatches, device_ns, ...)``."""
    from ..api import _ptr_len
    lib = N.load()
    addr = signal.addr if hasattr(signal, "rkey") else _ptr_len(signal, 8)[0]
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    cd = cs = cb = cst = 0
    if check is not None:
        d, s, cb, cst = check
        cd, cs = _ptr_len(d, 1)[0], _ptr_len(s, 1)[0]
        if cb % 16:
            raise ValueError("check slot_bytes must be a multiple of 16")
    rc = lib.rn_k_signal_wait(_stream_ptr(ws), addr, until, stamps.data_ptr() if stamps is not None else 0, out_addr,
                              timeout_ms, cd, cs, cb, cst)
    return L.finish(rc, "signal_wait", out_view, ws, sync, parse_signal_wait)


def cq_watch(cq, n: int, dst, src, slot_stride: int, nslots: int, msg_bytes: int, piece: int, tail: int = 16384,
             timeout_ms: int = 2000, stream=None, sync: bool = True, scratch_off: int = MAPPED["cq_watch"].offset):
    """Receiver-side check of a device send CQ that another kernel (the poster) consumes: waits for each of its first
    ``n`` CQEs in turn without consuming them (the CQ must hold ``n``), and the moment CQE ``k`` is visible compares the
    message it names -- slot ``wqe_counter % nslots`` of ``dst`` and ``src`` (tensors or ``(address, nbytes)`` pairs) at
    ``slot_stride`` -- with every ``piece`` bytes checked on their last ``tail`` bytes.  Returns
    ``dict(status, seen, mismatches, error_cqes, device_ns)``."""
    from ..api import _ptr_len
    ctx = cq.ctx
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    rc = N.load().rn_k_cq_watch(_stream_ptr(ws), cq.dev_ptr, n, _ptr_len(dst, 1)[0], _ptr_len(src, 1)[0], slot_stride, nslots,
                                msg_bytes, piece, tail, timeout_ms, out_addr)
    return L.finish(rc, "cq_watch", out_view, ws, sync, parse_cq_watch)


def parse_cq_watch(view) -> dict:
    """Decode the record :func:`cq_watch` leaves in its scratch slot (for ``sync=False`` callers)."""
    return L.decode(view, ("seen", "mismatches", "error_cqes"))


def parse_signal_wait(view) -> dict:
    """Decode the record :func:`signal_wait` leaves in its scratch slot (for ``sync=False`` callers)."""
    return L.decode(view, ("seen", "mismatches"))


def read_records(qp, src_mr, dst_mr, rec_bytes: int, n: int, *, indices=None, src_off: int = 0, src_stride=None,
                 dst_off: int = 0, ready=None, window: int = 16, burst: int = 1, signal_every: int = 1, timeout_ms: int = 2000,
                 stream=None, sync: bool = True, scratch_off: int = MAPPED["read_records"].offset):
    """Pull ``n`` fixed-size records with device-posted RDMA READs and stamp an arrival word as each one lands.

    Record ``r`` is one READ of ``rec_bytes`` from ``src_mr.addr + src_off + j * src_stride`` (the remote side) into
    ``dst_mr.addr + dst_off + r * rec_bytes``, where ``j = indices[r]`` (an int32 CUDA tensor of ``n`` entries, read on
    the device only: a permutation, a subset or repeats) or ``j = r``.  ``src_stride`` defaults to ``rec_bytes``, so K3
    chunk records and K4 panel records can be pulled whole or gathered.  An index whose record does not fit the remote
    region fails on the wire like any out-of-range READ (``REMOTE_ACCESS_ERR``, the QP goes to ERR).

    ``ready`` (int64 CUDA tensor of at least ``n`` words, zeroed by the caller) gets word ``r`` set to a nonzero
    %globaltimer value, with release semantics, once record ``r`` has landed: the arrival word that
    ``unpack_fp8(ready=)`` and ``gemm_mxfp8(a_ready=)`` wait for.  One warp owns the QP and its send CQ; ``window``,
    ``burst`` and ``signal_every`` are :func:`rdma_stream`'s knobs (one CQE stamps up to ``signal_every`` records with
    one value).  ``window`` is at most the send queue's and the send CQ's depth.  When a READ fails the status is
    ``CQE_ERROR``: every earlier record has landed and is stamped, the failing one and every later one are not.

    Returns ``dict(status, done, device_ns, t_start_ns, t_end_ns, first_idx, last_idx, cons)`` (``done``: records landed),
    or ``(result view, stream)`` with ``sync=False`` (decode with :func:`parse_read_records`)."""
    ctx = qp.ctx
    rec_bytes, n = N.byte_count(rec_bytes, "rec_bytes"), int(n)
    if rec_bytes == 0 or rec_bytes > ctx.max_msg_bytes:
        raise ValueError(f"rec_bytes={rec_bytes}: a record is one READ of 1..{ctx.max_msg_bytes} bytes")
    if not 0 <= n < 1 << 32:
        raise ValueError(f"n={n}: outside [0, 2**32)")
    src_stride = rec_bytes if src_stride is None else int(src_stride)
    if src_off < 0 or src_stride < 0 or dst_off < 0:
        raise ValueError("src_off, src_stride and dst_off must be non-negative")
    if dst_off + n * rec_bytes > dst_mr.length:
        raise ValueError(f"{n} records of {rec_bytes} bytes at dst_off={dst_off} do not fit dst_mr ({dst_mr.length} bytes)")
    idx_addr = 0 if indices is None else L.tensor_ptr(indices, torch.int32, ctx.device, "indices", n)
    ready_addr = 0 if ready is None else L.tensor_ptr(ready, torch.int64, ctx.device, "ready", n)
    depth = min(qp.sq_depth, qp.scq.depth)
    window = depth if window <= 0 else min(int(window), depth)
    ws = work_stream(ctx, stream)
    out_addr, out_view = L.result(ctx, scratch_off)
    rc = N.load().rn_k_read_records(_stream_ptr(ws), qp.dev_ptr, dst_mr.addr + dst_off, dst_mr.lkey, src_mr.addr + src_off,
                                    src_mr.rkey, src_stride, rec_bytes, n, idx_addr, ready_addr, window, burst, signal_every,
                                    timeout_ms, out_addr)
    return L.finish(rc, "read_records", out_view, ws, sync, parse_read_records)


def parse_read_records(view) -> dict:
    """Decode the record :func:`read_records` leaves in its scratch slot (for ``sync=False`` callers)."""
    return L.decode(view, ("done", "first_idx", "last_idx", "cons"))
