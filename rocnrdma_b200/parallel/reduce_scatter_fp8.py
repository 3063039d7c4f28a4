"""fp8 ring reduce-scatter, and the GEMM-reduce-scatter of a row-parallel layer that reduces each panel as it finishes.

N ranks each hold a tensor of N shards of ``shard_elems`` elements (shard s is ``[s * shard, (s + 1) * shard)``), moved
as R = shard_elems / chunk K3 chunk records.  Rank q ends with the sum over ranks of shard q, as
``torch.distributed.reduce_scatter_tensor`` lays it out.  Step k of rank q handles shard (q-1-k) mod N, so its last step,
N-1, is its own shard q.  The landing region has N-1 slots of R records; record r of slot m has the id m * R + r, its
immediate and the index of its arrival word, as in ring_fp8.  Rank q:

* consumer stream: clears the words and runs one ``recv_consume`` for the (N-1)R records it receives (as ring_fp8);
* main stream, :meth:`RingReduceScatterFp8.run`, with no host step in between:
  1. ``pack_fp8_write`` packs ``x[shard q-1]`` into the send staging and posts it to the next rank's slot 0;
  2. reduce hop k = 0..N-2 (``reduce_fp8``) waits on slot k's words and adds ``x[shard (q-2-k) mod N]``; hops k <= N-3
     re-pack the sum into the send staging (reused from hop to hop: every posting launch waits for its flush) and post
     it to the next rank's slot k+1, hop N-2 writes the bf16 sum into ``out``;
* main stream, :meth:`RingReduceScatterFp8.run_gemm`: one ``gemm_reduce_send`` (K4 with a landed addend) walks the
  m-blocks of shard q-1, q-2, ..., q.  Step 0's panels are posted as records of the product to the next rank's slot 0;
  step k's (1..N-2) add landed record (k-1)R + r and are posted as id kR + r; step N-1's add record (N-2)R + r and are
  stored as bf16 rows of ``out``.  A panel waits for its record after its MMAs, so it computes while the record is on
  the wire.

Every rank applies the same hops in the same order, so the result is ``ops.ref_reduce_scatter_fp8`` bit for bit.
DESIGN.md 3.4 has the deadlock argument, the limits and the measurements.
"""
from __future__ import annotations

from typing import List, NamedTuple, Tuple

import torch

from .. import ops
from ..ops import launch as L
from ..ops.gemm import BM
from .ring_fp8 import GUARD, MAX_QUEUE_DEPTH, _pow2, _RingPlan, _run_ranks, link_in_process  # noqa: F401


class Step(NamedTuple):
    """Step k of a rank: the shard it handles, the landing slot whose records it adds (None: none) and the next rank's
    slot it posts to (None: it writes ``out`` instead)."""
    shard: int
    read_slot: object
    send_slot: object


def schedule(rank: int, world: int) -> List[Step]:
    """Rank ``rank``'s N steps, in order: step k handles shard (q-1-k) mod N, adds slot k-1 and posts to slot k."""
    N, q = world, rank
    return [Step((q - 1 - k) % N, k - 1 if k else None, k if k < N - 1 else None) for k in range(N)]


def max_records(world: int) -> int:
    """The most records per shard a plan of ``world`` ranks can have: its receive queue and CQ hold
    ``_pow2(2 (N-1) R)`` entries, at most ``MAX_QUEUE_DEPTH``."""
    return MAX_QUEUE_DEPTH // (2 * (int(world) - 1))


def gemm_ids(rank: int, world: int, R: int) -> Tuple[List[int], List[int], List[int]]:
    """``gemm_reduce_send``'s walk, add_ids and send_ids of rank ``rank`` for R 128-row blocks per shard: walk position
    k * R + r is m-block ``shard(k) * R + r``, adds landed record (k-1)R + r from step 1 on, and becomes record kR + r up
    to step N-2 (-1 at step N-1: bf16 rows r of ``out``)."""
    walk, add, send = [], [], []
    for k, st in enumerate(schedule(rank, world)):
        for r in range(R):
            walk.append(st.shard * R + r)
            add.append(-1 if st.read_slot is None else st.read_slot * R + r)
            send.append(-1 if st.send_slot is None else st.send_slot * R + r)
    return walk, add, send


class RingReduceScatterFp8(_RingPlan):
    """One rank's plan of the fp8 ring reduce-scatter of ``world`` shards of ``shard_elems`` elements, as a collective
    (:meth:`run`) or fused with the GEMM of a row-parallel layer (:meth:`run_gemm`).

    Everything is allocated and registered here, before any engine runs (DESIGN.md 3.2): the landing region (N-1 slots
    of R records), the arrival words with guard words behind them, one send staging of (N-1)R records (``run`` uses its
    first R), the GEMM's walk and ids, and the streams.  Link the plans with :func:`link_in_process` (N simulated ranks
    in one context) or :meth:`connect` (one process per GPU), start the engine, then run.

    ``grid`` is the CTAs of every launch (0: as many as the SM budget allows).  Every kernel that waits must be resident
    as a whole beside the engine and the consumers, so ``engine_ctas + ranks on the GPU * (grid + 1)`` may not exceed
    the device's SMs.  ``timeout_ms`` bounds every wait; a rank whose input never comes ends ``TIMEOUT``.  After a run
    that did not end OK the output is undefined; in one process the next run reaps what the failed one left, between
    processes connect new plans (as ring_fp8)."""

    def __init__(self, ctx, shard_elems: int, chunk_elems: int, rank: int, world: int, *, grid: int = 0,
                 timeout_ms: int = 2000, signal_every: int = 1, engine_ctas: int = 16):
        super().__init__(ctx, chunk_elems, rank, world, grid, timeout_ms, signal_every, engine_ctas)
        shard_elems, world, chunk_elems = int(shard_elems), self.world, self.chunk
        if shard_elems <= 0 or shard_elems % chunk_elems:
            raise ValueError(f"shard_elems={shard_elems} must be a multiple of chunk_elems = {chunk_elems}: "
                             "every shard is whole records")
        self.shard = shard_elems
        self.n = world * shard_elems
        self.R = shard_elems // chunk_elems
        if self.R > max_records(world):
            raise ValueError(f"R={self.R} records per shard: the receive queue would need "
                             f"{_pow2(2 * (world - 1) * self.R)} entries, above {MAX_QUEUE_DEPTH}; at world={world} R "
                             f"may be at most {max_records(world)}")
        # the reduce's counters (R records and 3 words), the GEMM's (one per m-block of the whole product and 3 words)
        if L.counter_bytes(world * self.R + 3) > L.SLOT_BYTES:
            raise ValueError(f"{self.R} records per shard need more counters than a scratch slot holds")
        # result records: 0 receive, 1.. the pack and the N-1 hops of run (run_gemm uses 1)
        n_ids = (world - 1) * self.R
        self._allocate(n_ids, n_ids, world + 1)
        dev = ctx.device
        self.staging = torch.zeros(n_ids * self.rec, dtype=torch.uint8, device=f"cuda:{dev}")
        self.staging_mr = ctx.reg_mr(self.staging)
        self.ids_host = gemm_ids(self.rank, world, self.R)
        self.walk, self.add_ids, self.send_ids = (torch.tensor(v, dtype=torch.int32, device=f"cuda:{dev}")
                                                   for v in self.ids_host)
        # rows of a step advance together in the GEMM's raster: a group never holds two steps (the deadlock argument)
        self.group_m = next(g for g in (4, 2, 1) if self.R % g == 0)
        with torch.cuda.stream(self.consumer_stream):
            self.words.zero_()              # loads the fill kernel now: a first load later would wait for the engine
        self._cleared.record(self.consumer_stream)
        torch.cuda.synchronize(dev)

    # ---------------------------------------------------------------- run
    def _check_run(self, x, out):
        L.tensor_ptr(x, torch.bfloat16, self.ctx.device, "x", self.n, exact=True, align=32)
        L.tensor_ptr(out, torch.bfloat16, self.ctx.device, "out", self.shard, exact=True, align=32)
        _no_overlap(out, x, "x")

    def _check_gemm(self, a, b, out):
        N = self.world
        for t, what in ((a, "a"), (b, "b"), (out, "out")):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.bfloat16 or t.dim() != 2 or not t.is_contiguous():
                raise ValueError(f"{what} must be a contiguous 2-D bf16 tensor")
        M, K = a.shape
        Nb, Kb = b.shape
        if K != Kb:
            raise ValueError(f"a is [M, {K}] and b is [Nb, {Kb}]: both hold the rank's K slice")
        if M % (N * BM) or Nb % 64 or K % 8:
            raise ValueError(f"shape ({M}, {Nb}, {K}): M must be a multiple of world * 128 = {N * BM}, Nb of 64, K of 8")
        if self.chunk != BM * Nb:
            raise ValueError(f"chunk_elems={self.chunk}: run_gemm needs one 128-row panel per record, 128 * Nb = {BM * Nb}")
        if self.shard != (M // N) * Nb:
            raise ValueError(f"shard_elems={self.shard}: run_gemm's shard is (M / world) * Nb = {(M // N) * Nb}")
        if tuple(out.shape) != (M // N, Nb):
            raise ValueError(f"out must be [{M // N}, {Nb}]")
        _no_overlap(out, a, "a")

    def enqueue_main(self, x: torch.Tensor, out: torch.Tensor):
        """Enqueue this rank's main stream of :meth:`run` (after :meth:`start_consumer`): K3 and the N-1 reduce hops."""
        self._check_run(x, out)
        N, q, R, rec = self.world, self.rank, self.R, self.rec
        ms = self.main_stream
        ms.wait_event(self._cleared)
        common = dict(grid=self.grid, timeout_ms=self.timeout_ms, stream=ms, sync=False, scratch_slot=self.scratch_slot)
        post = dict(qp=self.send_qp, dst_mr=self.remote_landing, with_imm=True, signal_every=self.signal_every)
        st = schedule(q, N)
        v, _ = ops.pack_fp8_write(self.ctx, self._shard(x, st[0].shard), self.staging_mr, chunk_elems=self.chunk,
                                  result_off=self._res(1), **post, **common)
        self._views.append(("pack", "pack", v))
        for k in range(1, N):
            land, words = self._slot(st[k].read_slot)
            dst = dict(out=out) if st[k].send_slot is None else dict(
                out_mr=self.staging_mr, dst_off=st[k].send_slot * R * rec, imm_base=st[k].send_slot * R, **post)
            v, _ = ops.reduce_fp8(self.ctx, land, 1, self.shard, self.chunk, local=self._shard(x, st[k].shard), ready=words,
                                  result_off=self._res(1 + k), **dst, **common)
            self._views.append((f"reduce hop {k - 1}", "reduce", v))

    def enqueue_gemm(self, a: torch.Tensor, b: torch.Tensor, out: torch.Tensor):
        """Enqueue this rank's main stream of :meth:`run_gemm` (after :meth:`start_consumer`): one ``gemm_reduce_send``."""
        self._check_gemm(a, b, out)
        ms = self.main_stream
        ms.wait_event(self._cleared)
        v, _ = ops.gemm_reduce_send(self.ctx, a, b, walk=self.walk, add_ids=self.add_ids, send_ids=self.send_ids,
                                    ids_host=self.ids_host, qp=self.send_qp, staging_mr=self.staging_mr,
                                    dst_mr=self.remote_landing, landing=self.landing, ready=self.words, out=out,
                                    signal_every=self.signal_every, group_m=self.group_m, grid=self.grid,
                                    timeout_ms=self.timeout_ms, stream=ms, sync=False, scratch_slot=self.scratch_slot,
                                    result_off=self._res(1))
        self._views.append(("gemm", "gemm_rs", v))

    def run(self, x: torch.Tensor, out: torch.Tensor, sync: bool = True):
        """Reduce-scatter: ``out`` (bf16, ``shard_elems``) = shard ``rank`` of the sum over ranks of ``x`` (bf16,
        ``world * shard_elems``), each hop's sum carried as K3 records, as ``torch.distributed.reduce_scatter_tensor``
        lays it out.  ``out`` may not overlap ``x``.  With ``sync`` waits and returns a :class:`RingResult`.  Ranks
        simulated in one process must all be enqueued before any is waited for: use :func:`run_in_process`."""
        self._check_run(x, out)
        return self._run(lambda: self.enqueue_main(x, out), sync)

    def run_gemm(self, a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, sync: bool = True):
        """The GEMM-reduce-scatter of a row-parallel layer: ``out[M / N, Nb]`` = rows ``[rank * M / N, (rank + 1) * M /
        N)`` of the sum over ranks of ``a_q @ b_q.T``, each rank holding its K slice: ``a`` bf16 ``[M, K_l]``, ``b`` bf16
        ``[Nb, K_l]``.  ``M`` a multiple of ``world * 128``, ``Nb`` of 64, ``K_l`` of 8; ``chunk_elems = 128 * Nb`` and
        ``shard_elems = (M / N) * Nb``.  Every panel's fp32 partial is reduced with the landed sum of the previous ranks
        and posted on as the GEMM finishes it; ``out`` may not overlap ``a``."""
        self._check_gemm(a, b, out)
        return self._run(lambda: self.enqueue_gemm(a, b, out), sync)


def _no_overlap(out, t, what):
    lo, hi = out.data_ptr(), out.data_ptr() + out.numel() * out.element_size()
    if lo < t.data_ptr() + t.numel() * t.element_size() and t.data_ptr() < hi:
        raise ValueError(f"out must not overlap {what}: the reduce-scatter has no in-place form")


def run_in_process(plans: List[RingReduceScatterFp8], xs, outs, sync: bool = True, skip=()):
    """Run the in-process reduce-scatter: every consumer, then every main stream.  ``skip``: ranks whose main stream is
    not enqueued (a rank that never contributes; its receives are still posted).  Returns one
    :class:`~rocnrdma_b200.parallel.ring_fp8.RingResult` per rank with ``sync``."""
    return _run_ranks(plans, [lambda p=p, x=x, o=o: p.enqueue_main(x, o) for p, x, o in zip(plans, xs, outs)], sync, skip)


def run_gemm_in_process(plans: List[RingReduceScatterFp8], as_, bs, outs, sync: bool = True, skip=()):
    """:func:`run_in_process` for :meth:`RingReduceScatterFp8.run_gemm`: rank q multiplies ``as_[q]`` by ``bs[q]``."""
    return _run_ranks(plans, [lambda p=p, a=a, b=b, o=o: p.enqueue_gemm(a, b, o) for p, a, b, o in zip(plans, as_, bs, outs)],
                      sync, skip)
