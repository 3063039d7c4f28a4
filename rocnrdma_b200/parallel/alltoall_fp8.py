"""fp8 all-to-all of bf16 shards over a mesh of queue pairs, and the all-to-all GEMM that multiplies each shard as it lands.

Each of N ranks holds N shards of ``shard_elems`` bf16 elements; shard d goes to rank d, as R = shard_elems / chunk K3
chunk records.  Every rank has one send queue pair to each peer and one receive queue pair from each peer, and its
receive queue pairs share one receive CQ.  Rank q's landing region has N slots of R records: slot s is what rank s sent,
and record r of slot s has the id s * R + r, which is its immediate and the index of its arrival word.  That is the
all-gather's layout, so with ``[rows, K]`` shards the landing region is K7's A as it stands
(``MxOperand.from_chunk_records(landing, N * rows, K, chunk)``).  Rank q:

* consumer stream: clears the words and runs one ``recv_consume_qps`` that preposts R receives on each receive queue
  pair and stamps the (N-1)R records it receives;
* main stream: one ``pack_fp8_scatter`` packs every shard in phase order -- phase j is shard (q + j) mod N, phase 0 the
  own shard -- and posts record r of shard d to rank d's slot q as soon as it is complete.  The own shard's records are
  written into the own slot, and their words are stamped by the pack itself;
* compute stream, behind the clear:
  * :meth:`AllToAllFp8.run`: ``unpack_fp8(ready=)`` of each slot in arrival order (q, q-1, ..., q+1) into ``out``;
  * :meth:`AllToAllFp8.run_gemm`: one ``gemm_mxfp8(a_ready=words, a_order=arrival order, cta_group=1)``.

At phase j every rank sends to rank q+j and receives from rank q-j, so rank q's slots complete in the order q, q-1, ...,
q+1, which is ``allgather_fp8.arrival_slots``.  Every rank decodes the K3 records of their sources, so the output is
``ops.ref_alltoall_fp8`` bit for bit.  DESIGN.md 3.4 has the details and the measurements.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from .. import ops
from ..ops import launch as L
from ..ops.gemm_mx import PANEL_ROWS, MxOperand
from .allgather_fp8 import arrival_slots
from .reduce_scatter_fp8 import _no_overlap
from .ring_fp8 import (MAX_IN_PROCESS, MAX_QUEUE_DEPTH, RingResult, _check_budget, _default_grid, _pow2, _RingPlan,
                       _run_ranks)

MAX_WORLD = 8                   # one NVLink node, and the scatter pack's destinations


def phase_order(rank: int, world: int) -> List[int]:
    """The shard rank ``rank`` packs and posts at each phase: phase j is shard (and destination) (rank + j) mod N."""
    return [(rank + j) % world for j in range(world)]


def posted_ids(rank: int, world: int, R: int) -> Dict[int, List[int]]:
    """The ids rank ``rank`` posts to each peer d, in posting order: slot ``rank`` of d's landing region."""
    return {d: [rank * R + r for r in range(R)] for d in phase_order(rank, world)[1:]}


def received_ids(rank: int, world: int, R: int) -> Dict[int, List[int]]:
    """The ids rank ``rank`` receives from each peer s, on its receive queue pair from s: its own slot s."""
    return {s: [s * R + r for r in range(R)] for s in range(world) if s != rank}


def max_records(world: int) -> int:
    """The most records per shard a plan of ``world`` ranks can have: the shared receive CQ takes ``(N-1)R`` completions
    per run, with room for those a failed run leaves behind, in at most ``MAX_QUEUE_DEPTH`` entries."""
    return MAX_QUEUE_DEPTH // (2 * (int(world) - 1))


def reap(rank: int, R: int, posted_to: List[List[int]], received: int) -> Tuple[int, List[int]]:
    """What a run leaves on rank ``rank``'s receive side, in one process: ``posted_to[s][d]`` records that rank s posted
    to rank d (an empty list: rank s posted nothing), ``received`` the completions its consumer took.  Returns the stale
    completions on the shared CQ (records that landed after the consumer stopped) and, per source s, the receive WQEs
    left posted on the queue pair from s (R less what s posted)."""
    arrivals = [(p[rank] if p else 0) for p in posted_to]
    backlog = [0 if s == rank else max(0, R - a) for s, a in enumerate(arrivals)]
    stale = max(0, sum(a for s, a in enumerate(arrivals) if s != rank) - received)
    return stale, backlog


class AllToAllFp8(_RingPlan):
    """One rank's plan of the fp8 all-to-all of ``world`` shards of ``shard_elems`` bf16 elements, as a collective
    (:meth:`run`) or fused with the block-scaled GEMM (:meth:`run_gemm`).

    Everything is allocated and registered here, before any engine runs (DESIGN.md 3.2): the send staging (N shards of R
    records), the landing region (N slots of R records), the arrival words with guard words behind them, the GEMM's
    record order and the streams.  Link the plans with :func:`link_in_process` (N simulated ranks in one context) or
    :meth:`connect` (one process per GPU, through ``parallel.peer.connect_mesh``), start the engine, then run.

    ``grid`` is the CTAs of the pack and of every compute launch (0: as many as the SM budget allows).  The consumer and
    the compute grid wait for other ranks and must be resident as a whole beside the engine; the pack waits only for its
    own flushes.  So ``engine_ctas + ranks on the GPU * (grid + 1)`` may not exceed the device's SMs.  ``timeout_ms``
    bounds every wait; a rank whose input never comes ends ``TIMEOUT``.  After a run that did not end OK the output is
    undefined; in one process the next run reaps what the failed one left, between processes connect new plans."""

    def __init__(self, ctx, shard_elems: int, chunk_elems: int, rank: int, world: int, *, grid: int = 0,
                 timeout_ms: int = 2000, signal_every: int = 1, engine_ctas: int = 16):
        super().__init__(ctx, chunk_elems, rank, world, grid, timeout_ms, signal_every, engine_ctas)
        shard_elems, world, chunk_elems = int(shard_elems), self.world, self.chunk
        if world > MAX_WORLD:
            raise ValueError(f"world={world}: the all-to-all runs on 2..{MAX_WORLD} ranks")
        if shard_elems <= 0 or shard_elems % chunk_elems:
            raise ValueError(f"shard_elems={shard_elems} must be a multiple of chunk_elems = {chunk_elems}: "
                             "every shard is whole records")
        self.shard = shard_elems
        self.n = world * shard_elems
        self.R = shard_elems // chunk_elems
        if self.R > max_records(world):
            raise ValueError(f"R={self.R} records per shard: the shared receive CQ would need "
                             f"{_pow2(2 * (world - 1) * self.R)} entries, above {MAX_QUEUE_DEPTH}; at world={world} R "
                             f"may be at most {max_records(world)}")
        # the unpack's counters from the bottom of the plan's scratch slot, the scatter pack's at its top
        if L.counter_bytes(self.R + 3) + L.counter_bytes(world * self.R + 1) + 24 * (world - 1) > L.SLOT_BYTES:
            raise ValueError(f"{self.R} records per shard need more counters than a scratch slot holds")
        # result records: 0 receive, 1-2 the scatter pack, 3.. compute
        self._allocate(world * self.R, (world - 1) * self.R, world + 3)
        dev = ctx.device
        self.staging = torch.zeros(world * self.R * self.rec, dtype=torch.uint8, device=f"cuda:{dev}")
        self.staging_mr = ctx.reg_mr(self.staging)
        order = [s * self.R + r for s in arrival_slots(self.rank, world) for r in range(self.R)]
        self.a_order = torch.tensor(order, dtype=torch.int32, device=f"cuda:{dev}")   # K7's walk: every record, as it lands
        self.compute_stream = torch.cuda.Stream(device=dev)
        self._done = torch.cuda.Event()
        self.send_qps = self.recv_qps = self.remote_landings = None
        self._backlogs = [0] * world    # receive WQEs a failed run left posted, per source
        with torch.cuda.stream(self.consumer_stream):
            self.words.zero_()              # loads the fill kernel now: a first load later would wait for the engine
        self._cleared.record(self.consumer_stream)
        torch.cuda.synchronize(dev)

    def _streams(self):
        return (self.consumer_stream, self.main_stream, self.compute_stream)

    def records(self) -> torch.Tensor:
        """The landed records, slot s (rank s's records of its shard ``rank``) at record s * R: after a run that ended
        OK, every source's K3 records."""
        return self.landing

    # ---------------------------------------------------------------- links
    def _attach_mesh(self, send_qps, recv_qps, remote_landings, scratch_slot: int, grid: int, in_process: bool):
        """``send_qps[d]`` / ``recv_qps[s]``: the queue pairs to rank d / from rank s; ``remote_landings[d]`` rank d's
        landing region (entry ``rank`` of each is None)."""
        q, N = self.rank, self.world
        peers = [d for d in range(N) if d != q]
        rcq = recv_qps[peers[0]].rcq
        if any(recv_qps[s].rcq is not rcq for s in peers):
            raise ValueError("a rank's receive queue pairs share one receive CQ")
        if rcq.depth < 2 * self.n_recv or any(recv_qps[s].rq_depth < 2 * self.R for s in peers):
            raise ValueError(f"the receive CQ ({rcq.depth}) must hold 2 * {self.n_recv} entries and each receive queue "
                             f"2 * {self.R}: one run's receives, and those a failed run leaves behind")
        if any(remote_landings[d].length < self.landing.numel() for d in peers):
            raise ValueError("a peer's landing region is smaller than this plan's")
        self.send_qps, self.recv_qps, self.remote_landings = list(send_qps), list(recv_qps), list(remote_landings)
        # the base class's single queue pairs: its link check, and the drain of stale completions on the shared CQ
        self.send_qp, self.recv_qp = send_qps[(q + 1) % N], recv_qps[(q - 1) % N]
        self.remote_landing = remote_landings[(q + 1) % N]
        self.scratch_slot, self.grid, self.in_process = scratch_slot, grid, in_process

    def connect(self, group=None, sq_depth: int = 256):
        """One process per GPU: create a send queue pair to every peer and a receive queue pair from every peer (the
        receive ones sharing one CQ), and connect them through ``parallel.peer.connect_mesh``.  Collective."""
        import torch.distributed as dist
        from .peer import connect_mesh
        if dist.get_rank(group) != self.rank or dist.get_world_size(group) != self.world:
            raise ValueError("the process group's rank and world size differ from the plan's")
        grid = self.grid or _default_grid(self.ctx, self.engine_ctas, 1, self.WAITERS)
        _check_budget(self.ctx, self.engine_ctas, 1, grid, self.WAITERS)
        send, recv = _mesh_qps(self.ctx, self.rank, self.world, self.n_recv, self.R, sq_depth)
        remote = connect_mesh(self.ctx, send, recv, [self.landing_mr], group)
        landings = [None if d == self.rank else next(iter(remote[d].values())) for d in range(self.world)]
        self._attach_mesh(send, recv, landings, 0, grid, in_process=False)

    # ---------------------------------------------------------------- consumer and failure accounting
    def _receive(self, views, kw):
        peers = [s for s in range(self.world) if s != self.rank]
        prepost = [self.R - self._backlogs[s] for s in peers]
        views.append(("receive", "recv", ops.recv_consume_qps([self.recv_qps[s] for s in peers], self.n_recv, prepost,
                                                              self.landing_mr, self.n_ids, self.words,
                                                              scratch_off=self._res(0), **kw)[0]))
        self._backlogs = [0] * self.world

    def _reap(self, res: List[RingResult]):
        self._stale_cqes, self._backlogs = reap(self.rank, self.R, [r.posted_to for r in res], res[self.rank].received)
        self._rq_backlog = sum(self._backlogs)

    def result(self) -> RingResult:
        res = super().result()
        view = next((v for name, kind, v in self._views if kind == "scatter"), None)
        res.posted_to = ops.parse_scatter(view)[1][:self.world] if view is not None else [0] * self.world
        return res

    # ---------------------------------------------------------------- run
    def _enqueue_scatter(self, x_flat: torch.Tensor):
        """Main stream: the scatter pack, behind the clear and the previous run's compute; the compute stream waits for
        the clear."""
        q = self.rank
        ms = self.main_stream
        ms.wait_event(self._cleared)
        ms.wait_event(self._done)           # the previous run's compute has read the own slot
        own, own_words = self._slot(q)
        v, _ = ops.pack_fp8_scatter(self.ctx, x_flat, q, self.world, self.staging_mr, own, own_words, self.send_qps,
                                    self.remote_landings, self.chunk, signal_every=self.signal_every, grid=self.grid,
                                    timeout_ms=self.timeout_ms, stream=ms, sync=False, scratch_slot=self.scratch_slot,
                                    result_off=self._res(1))
        self._views.append(("pack", "scatter", v))
        self.compute_stream.wait_event(self._cleared)

    def _check_run(self, x, out):
        L.tensor_ptr(x, torch.bfloat16, self.ctx.device, "x", self.n, exact=True, align=32)
        L.tensor_ptr(out, torch.bfloat16, self.ctx.device, "out", self.n, exact=True, align=32)
        _no_overlap(out, x, "x")

    def _check_gemm(self, x, b, c):
        if x.dim() != 2:
            raise ValueError(f"x must be [world * rows, K], not {tuple(x.shape)}")
        M, K = x.shape
        if M % self.world or (M // self.world) * K != self.shard:
            raise ValueError(f"x holds {M} x {K} elements: {self.world} shards of {self.shard} are needed")
        if self.chunk % (PANEL_ROWS * K):
            raise ValueError(f"chunk_elems={self.chunk}: the GEMM needs whole 128-row blocks per record, a multiple of "
                             f"128 * K = {PANEL_ROWS * K}")
        if b.K != K:
            raise ValueError(f"b has K={b.K}; x has K={K}")
        L.tensor_ptr(x, torch.bfloat16, self.ctx.device, "x", self.n, exact=True, align=32)
        if c.dtype != torch.bfloat16 or tuple(c.shape) != (M, b.rows) or not c.is_contiguous():
            raise ValueError(f"c must be a contiguous bf16 [{M}, {b.rows}] tensor")

    def enqueue_main(self, x: torch.Tensor, out: torch.Tensor):
        """Enqueue this rank's main and compute streams of :meth:`run` (after :meth:`start_consumer`)."""
        self._check_run(x, out)
        self._enqueue_scatter(x)
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
        M, K = x.shape
        self._enqueue_scatter(x.reshape(-1))
        a = MxOperand.from_chunk_records(self.landing, M, K, self.chunk)
        v, _ = ops.gemm_mxfp8(self.ctx, a, b, c, grid=self.grid, stream=self.compute_stream, sync=False,
                              scratch_slot=self.scratch_slot, cta_group=1, a_ready=self.words, a_order=self.a_order,
                              timeout_ms=self.timeout_ms, result_off=self._res(3))
        self._views.append(("gemm", "gemm", v))
        self._done.record(self.compute_stream)

    def run(self, x: torch.Tensor, out: torch.Tensor, sync: bool = True):
        """All-to-all: ``out[shard s]`` (bf16, ``world * shard_elems`` in all) = the dequantisation of rank s's K3
        records of its ``x[shard rank]``, the layout ``torch.distributed.all_to_all_single`` gives with equal splits.
        ``out`` may not overlap ``x``: the compute stream writes ``out`` while the pack still reads ``x``.  With ``sync``
        waits and returns a :class:`~rocnrdma_b200.parallel.ring_fp8.RingResult`.  Ranks simulated in one process must
        all be enqueued before any is waited for: use :func:`run_in_process`."""
        self._check_run(x, out)
        return self._run(lambda: self.enqueue_main(x, out), sync)

    def run_gemm(self, x: torch.Tensor, b: MxOperand, c: torch.Tensor, sync: bool = True):
        """The all-to-all GEMM of expert parallelism: ``x`` is bf16 ``[world * rows, K]``, rows ``[d * rows, (d + 1) *
        rows)`` going to rank d, and ``c[world * rows, Nb] = dequant(all-to-all of x) @ dequant(b).T``, rows in source
        order -- one expert's tokens from every rank times that expert's weights.  K7 starts on each record as it lands,
        the own shard first.  ``chunk_elems`` must be a multiple of ``128 * K``.  The landed records stay in
        :meth:`records`."""
        self._check_gemm(x, b, c)
        return self._run(lambda: self.enqueue_gemm(x, b, c), sync)


def _mesh_qps(ctx, rank: int, world: int, n_recv: int, R: int, sq_depth: int):
    """One rank's queue pairs: a send QP to every peer (each with its own send CQ) and a receive QP from every peer, the
    receive QPs sharing one receive CQ of ``_pow2(2 n_recv)`` entries.  Neither kind completes anything on its other CQ,
    so one small CQ serves both."""
    idle = ctx.create_cq(64)
    rcq = ctx.create_cq(_pow2(2 * n_recv))
    depth = max(16, _pow2(2 * R))
    send = [None if d == rank else ctx.create_qp(ctx.create_cq(2 * sq_depth), idle, sq_depth, 16) for d in range(world)]
    recv = [None if s == rank else ctx.create_qp(idle, rcq, 16, depth) for s in range(world)]
    return send, recv


def link_in_process(plans: List[AllToAllFp8], sq_depth: int = 256):
    """Simulate N ranks in one context: build N(N-1) send and N(N-1) receive queue pairs, connect rank s's send QP for d
    to rank d's receive QP for s, and give rank q device-scratch slot q.  Call before the engine starts."""
    N = len(plans)
    if N < 2 or any(p.world != N or p.rank != i for i, p in enumerate(plans)):
        raise ValueError("plans must be ranks 0..N-1 of one world of N >= 2")
    ctx = plans[0].ctx
    if any(not isinstance(p, AllToAllFp8) or p.ctx is not ctx or (p.shard, p.chunk) != (plans[0].shard, plans[0].chunk)
           for p in plans):
        raise ValueError("in-process plans are all-to-all plans that share one context, shard_elems and chunk_elems")
    if N > MAX_IN_PROCESS:
        raise ValueError(f"{N} in-process ranks: the device scratch has {MAX_IN_PROCESS} slots, one per rank")
    grid = plans[0].grid or _default_grid(ctx, plans[0].engine_ctas, N, plans[0].WAITERS)
    _check_budget(ctx, plans[0].engine_ctas, N, grid, plans[0].WAITERS)
    qps = [_mesh_qps(ctx, q, N, plans[q].n_recv, plans[q].R, sq_depth) for q in range(N)]
    for s in range(N):
        for d in range(N):
            if s != d:
                qps[s][0][d].connect(qps[d][1][s])
    for q, p in enumerate(plans):
        p._attach_mesh(qps[q][0], qps[q][1], [None if d == q else plans[d].landing_mr for d in range(N)], q, grid,
                       in_process=True)
    return plans


def run_in_process(plans: List[AllToAllFp8], xs, outs, sync: bool = True, skip=()):
    """Run the in-process all-to-all: every consumer, then every main and compute stream.  ``skip``: ranks whose main and
    compute streams are not enqueued (a rank that never contributes; its receives are still posted).  Returns one
    :class:`~rocnrdma_b200.parallel.ring_fp8.RingResult` per rank with ``sync``."""
    return _run_ranks(plans, [lambda p=p, x=x, o=o: p.enqueue_main(x, o) for p, x, o in zip(plans, xs, outs)], sync, skip)


def run_gemm_in_process(plans: List[AllToAllFp8], xs, bs, cs, sync: bool = True, skip=()):
    """:func:`run_in_process` for :meth:`AllToAllFp8.run_gemm`: rank q multiplies by ``bs[q]`` into ``cs[q]``."""
    return _run_ranks(plans, [lambda p=p, x=x, b=b, c=c: p.enqueue_gemm(x, b, c) for p, x, b, c in zip(plans, xs, bs, cs)],
                      sync, skip)
