"""fp8 ring all-gather of bf16 shards, and the all-gather GEMM that multiplies each shard as it lands.

Each of N ranks holds one shard of ``shard_elems`` bf16 elements and moves it as R = shard_elems / chunk K3 chunk
records.  Every rank's landing region holds all N shards in shard order: slot s is shard s's R records, and record r of
shard s has the id s * R + r, which is its immediate and the index of its arrival word.  The landing region is therefore
the gathered tensor's records in row order, and with a [rows, K] shard it is the A operand of K7 as it stands
(``MxOperand.from_chunk_records(landing, N * rows, K, chunk)``).  Rank q:

* consumer stream: clears the words and runs one ``recv_consume`` for the (N-1)R records it receives (as ring_fp8);
* main stream, with no host step in between:
  1. ``pack_fp8_write`` packs x into its own slot q of the landing region (it posts nothing);
  2. the own slot's words are set;
  3. ``relay_records`` posts slot q, then each arriving slot q-1, q-2, ..., q-N+2 (mod N), in that order, to the same
     offsets on the next rank.  Slot q+1 is not relayed: the next rank is where it came from.  This is the one poster
     and the one flush of the send queue pair in a run;
* compute stream, behind step 2:
  * :meth:`RingAllgatherFp8.run`: ``unpack_fp8(ready=)`` of each slot in arrival order (q, q-1, ..., q+1) into ``out``;
  * :meth:`RingAllgatherFp8.run_gemm`: one ``gemm_mxfp8(a_ready=words, a_order=arrival order, cta_group=1)`` over the
    whole gathered A, so every rank multiplies the shards it holds first while the others are still on the wire.

Slots arrive in the order the previous rank relays them, which is the order this rank relays them too.  Every rank
decodes the same records, so every rank holds the same bits (``ops.ref_allgather_fp8``).  DESIGN.md 3.4 has the
details and the measurements.
"""
from __future__ import annotations

from typing import List

import torch

from .. import ops
from ..ops import launch as L
from ..ops.gemm_mx import PANEL_ROWS, MxOperand
from .ring_fp8 import GUARD, MAX_QUEUE_DEPTH, _pow2, _RingPlan, _run_ranks, link_in_process  # noqa: F401


def arrival_slots(rank: int, world: int) -> List[int]:
    """The landing slots of rank ``rank`` in the order they are complete on it: its own, then q-1, ..., q+1 (mod N)."""
    return [(rank - k) % world for k in range(world)]


def relay_slots(rank: int, world: int) -> List[int]:
    """The slots rank ``rank`` relays to the next rank, in posting order: its arrival order without the last slot,
    q+1, which came from the next rank."""
    return arrival_slots(rank, world)[:world - 1]


def max_records(world: int) -> int:
    """The most records per shard a plan of ``world`` ranks can have: its receive queue and CQ hold
    ``_pow2(2 (N-1) R)`` entries, at most ``MAX_QUEUE_DEPTH``."""
    return MAX_QUEUE_DEPTH // (2 * (int(world) - 1))


class RingAllgatherFp8(_RingPlan):
    """One rank's plan of the fp8 ring all-gather of ``world`` shards of ``shard_elems`` bf16 elements, as a collective
    (:meth:`run`) or fused with the block-scaled GEMM (:meth:`run_gemm`).

    Everything is allocated and registered here, before any engine runs (DESIGN.md 3.2): the landing region (N slots of
    R records), the arrival words with guard words behind them, the relay's and the GEMM's record orders, and the
    streams.  Link the plans with :func:`link_in_process` (N simulated ranks in one context) or :meth:`connect` (one
    process per GPU), start the engine, then run.

    ``grid`` is the CTAs of the pack and of every compute launch (0: as many as the SM budget allows).  Every kernel
    that waits must be resident as a whole beside the engine and the other waiters, so ``engine_ctas + ranks on the GPU
    * (grid + 2)`` may not exceed the device's SMs: the 2 are the consumer and the relay.  ``timeout_ms`` bounds every
    wait; a rank whose input never comes ends ``TIMEOUT``.  After a run that did not end OK the output is undefined; in
    one process the next run reaps what the failed one left, between processes connect new plans (as ring_fp8)."""

    WAITERS = 2                 # the consumer and the relay

    def __init__(self, ctx, shard_elems: int, chunk_elems: int, rank: int, world: int, *, grid: int = 0,
                 timeout_ms: int = 2000, signal_every: int = 1, engine_ctas: int = 16):
        super().__init__(ctx, chunk_elems, rank, world, grid, timeout_ms, signal_every, engine_ctas)
        shard_elems, world, chunk_elems = int(shard_elems), self.world, self.chunk
        if shard_elems <= 0 or shard_elems % chunk_elems:
            raise ValueError(f"shard_elems={shard_elems} must be a multiple of chunk_elems = {chunk_elems}: "
                             "every shard is whole records")
        self.n = self.shard = shard_elems
        self.R = shard_elems // chunk_elems
        if self.R > max_records(world):
            raise ValueError(f"R={self.R} records per shard: the receive queue would need "
                             f"{_pow2(2 * (world - 1) * self.R)} entries, above {MAX_QUEUE_DEPTH}; at world={world} R "
                             f"may be at most {max_records(world)}")
        # the unpack's counters from the bottom of the plan's scratch slot, the relay's 32 bytes at its top
        if L.counter_bytes(self.R + 3) + L.counter_bytes(1) > L.SLOT_BYTES:
            raise ValueError(f"{self.R} records per shard need more counters than a scratch slot holds")
        # landing slot s holds shard s; result records: 0 receive, 1 pack, 2 relay, 3.. compute
        self._allocate(world * self.R, (world - 1) * self.R, world + 3)
        dev = ctx.device
        order = [s * self.R + r for s in arrival_slots(self.rank, world) for r in range(self.R)]
        self.a_order = torch.tensor(order, dtype=torch.int32, device=f"cuda:{dev}")   # K7's walk: every record, as it lands
        self.relay_ids = self.a_order[:self.n_recv]                                    # the relay's: all but slot q+1
        self.compute_stream = torch.cuda.Stream(device=dev)
        self._own_set, self._done = torch.cuda.Event(), torch.cuda.Event()
        with torch.cuda.stream(self.consumer_stream):
            # load the fill kernels now (step 2 and the consumer's clear): a first load later would wait for the engine.
            # Step 2 fills one slot's words, and where they start picks torch's kernel (a slot whose words are not 16-
            # or 32-byte aligned gets a narrower one), so fill every slot as step 2 does.
            for s in range(world):
                self._slot(s)[1].fill_(1)
            self.words.zero_()
        self._cleared.record(self.consumer_stream)
        torch.cuda.synchronize(dev)

    def _streams(self):
        return (self.consumer_stream, self.main_stream, self.compute_stream)

    def records(self) -> torch.Tensor:
        """The gathered records, shard s's at record s * R: after a run that ended OK, every rank's K3 records."""
        return self.landing

    # ---------------------------------------------------------------- run
    def _enqueue_gather(self, x_flat: torch.Tensor):
        """Main stream: pack x into the own slot, set its words, relay; the compute stream then waits for the own slot."""
        q, R = self.rank, self.R
        ms, cs = self.main_stream, self.compute_stream
        ms.wait_event(self._cleared)
        ms.wait_event(self._done)           # the previous run's compute has read the landing region
        ops.pack_fp8_write(self.ctx, x_flat, self.landing_mr, chunk_elems=self.chunk, staging_off=q * R * self.rec,
                           grid=self.grid, timeout_ms=self.timeout_ms, stream=ms, sync=False, scratch_slot=self.scratch_slot,
                           result_off=self._res(1))
        with torch.cuda.stream(ms):
            self.words[q * R:(q + 1) * R].fill_(1)
        self._own_set.record(ms)
        v, _ = ops.relay_records(self.send_qp, self.landing_mr, self.remote_landing, self.rec, self.relay_ids,
                                 ready=self.words, signal_every=self.signal_every, timeout_ms=self.timeout_ms, stream=ms,
                                 sync=False, scratch_slot=self.scratch_slot, result_off=self._res(2))
        self._views.append(("relay", "relay", v))
        cs.wait_event(self._own_set)

    def _check_run(self, x, out):
        L.tensor_ptr(x, torch.bfloat16, self.ctx.device, "x", self.shard, exact=True, align=32)
        L.tensor_ptr(out, torch.bfloat16, self.ctx.device, "out", self.world * self.shard, exact=True, align=32)

    def _check_gemm(self, x, b, c):
        if x.dim() != 2:
            raise ValueError(f"x must be a [rows, K] shard, not {tuple(x.shape)}")
        rows, K = x.shape
        if rows * K != self.shard:
            raise ValueError(f"x holds {rows} x {K} elements; the plan's shard is {self.shard}")
        if self.chunk % (PANEL_ROWS * K):
            raise ValueError(f"chunk_elems={self.chunk}: the GEMM needs whole 128-row blocks per record, a multiple of "
                             f"128 * K = {PANEL_ROWS * K}")
        if b.K != K:
            raise ValueError(f"b has K={b.K}; x has K={K}")
        L.tensor_ptr(x, torch.bfloat16, self.ctx.device, "x", self.shard, exact=True, align=32)
        if c.dtype != torch.bfloat16 or tuple(c.shape) != (self.world * rows, b.rows) or not c.is_contiguous():
            raise ValueError(f"c must be a contiguous bf16 [{self.world * rows}, {b.rows}] tensor")

    def enqueue_main(self, x: torch.Tensor, out: torch.Tensor):
        """Enqueue this rank's main and compute streams of :meth:`run` (after :meth:`start_consumer`)."""
        self._check_run(x, out)
        self._enqueue_gather(x.reshape(-1))
        common = dict(grid=self.grid, timeout_ms=self.timeout_ms, stream=self.compute_stream, sync=False,
                      scratch_slot=self.scratch_slot)
        for k, s in enumerate(arrival_slots(self.rank, self.world)):
            land, words = self._slot(s)
            v, _ = ops.unpack_fp8(self.ctx, land, self._shard(out, s), self.chunk, ready=words, result_off=self._res(3 + k),
                                  **common)
            self._views.append((f"unpack slot {s}", "unpack", v))
        self._done.record(self.compute_stream)

    def enqueue_gemm(self, x: torch.Tensor, b: MxOperand, c: torch.Tensor):
        """Enqueue this rank's main and compute streams of :meth:`run_gemm` (after :meth:`start_consumer`)."""
        self._check_gemm(x, b, c)
        rows, K = x.shape
        self._enqueue_gather(x.reshape(-1))
        a = MxOperand.from_chunk_records(self.landing, self.world * rows, K, self.chunk)
        v, _ = ops.gemm_mxfp8(self.ctx, a, b, c, grid=self.grid, stream=self.compute_stream, sync=False,
                              scratch_slot=self.scratch_slot, cta_group=1, a_ready=self.words, a_order=self.a_order,
                              timeout_ms=self.timeout_ms, result_off=self._res(3))
        self._views.append(("gemm", "gemm", v))
        self._done.record(self.compute_stream)

    def run(self, x: torch.Tensor, out: torch.Tensor, sync: bool = True):
        """All-gather: ``out`` (bf16, ``world * shard_elems``) = the dequantisation of every rank's K3 records of its
        ``x`` (bf16, ``shard_elems``), in rank order, as ``torch.distributed.all_gather_into_tensor`` lays it out.  ``x``
        may be ``out``'s shard ``rank`` (in place).  With ``sync`` waits and returns a :class:`RingResult`.  Ranks
        simulated in one process must all be enqueued before any is waited for: use :func:`run_in_process`."""
        self._check_run(x, out)
        return self._run(lambda: self.enqueue_main(x, out), sync)

    def run_gemm(self, x: torch.Tensor, b: MxOperand, c: torch.Tensor, sync: bool = True):
        """The all-gather GEMM of a column-parallel layer: ``c[world * rows, Nb] = dequant(gathered A) @ dequant(b).T``,
        A being every rank's K3 records of its ``x`` (bf16 ``[rows, K]``) in rank order.  K7 starts on each record as it
        lands, the records this rank holds first.  ``chunk_elems`` must be a multiple of ``128 * K``.  The gathered
        records stay in :meth:`records`."""
        self._check_gemm(x, b, c)
        return self._run(lambda: self.enqueue_gemm(x, b, c), sync)


def run_in_process(plans: List[RingAllgatherFp8], xs, outs, sync: bool = True, skip=()):
    """Run the in-process all-gather: every consumer, then every main stream.  ``skip``: ranks whose main and compute
    streams are not enqueued (a rank that never contributes; its receives are still posted).  Returns one
    :class:`~rocnrdma_b200.parallel.ring_fp8.RingResult` per rank with ``sync``."""
    return _run_ranks(plans, [lambda p=p, x=x, o=o: p.enqueue_main(x, o) for p, x, o in zip(plans, xs, outs)], sync, skip)


def run_gemm_in_process(plans: List[RingAllgatherFp8], xs, bs, cs, sync: bool = True, skip=()):
    """:func:`run_in_process` for :meth:`RingAllgatherFp8.run_gemm`: rank q multiplies by ``bs[q]`` into ``cs[q]``."""
    return _run_ranks(plans, [lambda p=p, x=x, b=b, c=c: p.enqueue_gemm(x, b, c) for p, x, b, c in zip(plans, xs, bs, cs)],
                      sync, skip)
