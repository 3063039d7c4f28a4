"""fp8-compressed ring all-reduce of bf16 tensors, every hop started on the device as records land.

Each rank owns one shard of ``n / N`` elements (shard s is ``[s * n / N, (s + 1) * n / N)``) and moves it as K3 chunk
records of R = n / (N * chunk) records.  Rank q:

* consumer stream: clears its arrival words and runs one ``recv_consume`` for all 2(N-1)R records it will receive this
  run (it posts its own zero-length receive WQEs: RDMA_WRITE_IMM ignores the buffer);
* main stream, with no host step in between:
  1. ``pack_fp8_write`` packs ``x[shard q]`` into the next rank's landing slot 0;
  2. reduce hop k = 0..N-2 (``reduce_fp8``) waits on slot k's words, adds ``x[shard (q-1-k) mod N]`` and posts the sum to
     the next rank's slot k+1; hop N-2 holds the full sum of shard (q+1) mod N and posts it to slot N-1, the first
     all-gather slot;
  3. for j = 0..N-2, ``unpack_fp8`` unpacks slot N-1+j into ``out[shard (q-j) mod N]`` and, for j <= N-3, forwards the
     slot unchanged to the next rank's slot N+j as each record lands;
  4. this rank's own final records are unpacked from the send staging into ``out[shard (q+1) mod N]``.

Record r of landing slot m has the global id m * R + r: it is the record's immediate and the index of its arrival word,
so records of different hops that reach one queue pair never stamp the same word.  Every rank's output is the
dequantisation of the same final records, so every rank holds the same bits (``ops.ref_allreduce_fp8``).  Every read of
``x`` precedes the first write of ``out`` on one stream, so ``out=None`` (in place) is safe; the send staging is reused
from hop to hop because every posting launch waits for its flush.  DESIGN.md 3.4 has the details.

Error feedback (``error_feedback=True``): rank q quantises every shard exactly once per run -- shard q in the pack and
shard (q-1-k) mod N in reduce hop k -- so one fp32 residual of n elements holds, in shard s, the error rank q made on
shard s.  The pack and each hop quantise ``value + residual`` and write back what the records lost, in the same pass;
summed over runs the output then equals the exact sum up to the last residual, while no add saturates.  Every add
of those steps saturates at +-FLT_MAX, so finite inputs give a finite output and finite residuals on every run.
Nothing on the wire changes.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import torch

from .. import ops
from ..ops import gemm as G, launch as L, pack as P
from ..ops.rdma import RECV_WORDS

GUARD = 8                       # zero words behind the arrival words
MAX_IN_PROCESS = L.N_SLOTS      # one device-scratch slot per simulated rank
MAX_QUEUE_DEPTH = 16384         # the deepest queue create_qp builds (a power of two; the doorbell index is 16 bits)


def max_records(world: int) -> int:
    """The most records per shard a plan of ``world`` ranks can have: its receive queue and CQ hold
    ``_pow2(2 * 2(N-1)R)`` entries, at most ``MAX_QUEUE_DEPTH``."""
    return MAX_QUEUE_DEPTH // (4 * (int(world) - 1))


@dataclass(frozen=True)
class Step:
    """One launch of a rank's main stream.  ``kind``: ``pack`` (K3 of ``x[shard]``), ``reduce`` (landing slot
    ``read_slot`` plus ``x[shard]``) or ``unpack`` (``read_slot``, or the send staging when it is None, into
    ``out[shard]``).  ``send_slot``: the next rank's landing slot the launch posts to (immediates and words from
    ``send_slot * R``), None when it posts nothing."""
    kind: str
    read_slot: Optional[int]
    shard: int
    send_slot: Optional[int]


def schedule(rank: int, world: int) -> List[Step]:
    """Rank ``rank``'s main stream, in order (the module docstring's steps 1-4)."""
    N, q = world, rank
    steps = [Step("pack", None, q, 0)]
    steps += [Step("reduce", k, (q - 1 - k) % N, k + 1) for k in range(N - 1)]
    steps += [Step("unpack", N - 1 + j, (q - j) % N, N + j if j <= N - 3 else None) for j in range(N - 1)]
    steps.append(Step("unpack", None, (q + 1) % N, None))
    return steps


# the words of each kind of launch's result record, after the header
_WORDS = {"pack": P.PACK_WORDS, "reduce": P.REDUCE_WORDS, "unpack": P.UNPACK_WORDS, "recv": RECV_WORDS,
          "relay": P.RELAY_WORDS, "gemm": (), "gemm_rs": G.RS_WORDS, "scatter": P.SCATTER_WORDS}


def _pow2(n: int) -> int:
    return 1 << max(0, int(n) - 1).bit_length()


@dataclass
class LaunchResult:
    name: str
    status: str
    t_start_ns: int
    t_end_ns: int

    @property
    def device_ns(self) -> int:
        return self.t_end_ns - self.t_start_ns


@dataclass
class RingResult:
    """What one rank's run did: ``status`` is ``OK`` or the status of the first launch that did not end OK, which
    ``failed`` names; ``launches`` holds each launch's status and device time; ``total_ns`` runs from the first start
    to the last end."""
    rank: int
    status: str
    failed: Optional[str]
    launches: List[LaunchResult] = field(default_factory=list)
    total_ns: int = 0
    received: int = 0           # arrivals the consumer saw
    posted: int = 0             # records this rank posted to the next one
    posted_to: List[int] = field(default_factory=list)    # an all-to-all's: records posted to each rank

    @property
    def ok(self) -> bool:
        return self.status == "OK"

    def hop_ns(self) -> List[int]:
        """Device time of each launch of the main stream, in launch order."""
        return [l.device_ns for l in self.launches if l.name != "receive"]


class _RingPlan:
    """What the GPU-driven ring plans share: the arguments both check, the landing region, its arrival words and the
    streams, linking (the receive queue and the next rank's landing region), the consumer stream that receives and
    stamps every record a run brings, recovery after a failed run, and the result.  A plan calls
    ``_RingPlan.__init__``, sets ``shard`` and ``R``, then calls :meth:`_allocate`."""
    WAITERS = 1                 # waiting launches of a rank beside its compute grid: the consumer

    def __init__(self, ctx, chunk_elems: int, rank: int, world: int, grid: int, timeout_ms: int, signal_every: int,
                 engine_ctas: int):
        chunk_elems, rank, world = int(chunk_elems), int(rank), int(world)
        if world < 2:
            raise ValueError(f"world={world}: a ring needs at least 2 ranks")
        if not 0 <= rank < world:
            raise ValueError(f"rank={rank} outside [0, {world})")
        if chunk_elems <= 0 or chunk_elems % P.TILE_ELEMS:
            raise ValueError(f"chunk_elems={chunk_elems}: a positive multiple of {P.TILE_ELEMS}")
        self.ctx, self.chunk, self.rank, self.world = ctx, chunk_elems, rank, world
        self.grid, self.timeout_ms, self.signal_every, self.engine_ctas = int(grid), int(timeout_ms), int(signal_every), int(engine_ctas)
        self.rec = P.record_bytes(chunk_elems)

    def _allocate(self, n_ids: int, n_recv: int, n_results: int):
        """Check the result records, then allocate and register the landing region of ``n_ids`` records, its arrival
        words with guard words behind them, and the consumer and main streams.  ``n_recv``: records received per run;
        ``n_results``: result records of a run before the two a failed run's recovery takes."""
        if n_results + 2 > L.RING_SLOT_BYTES // L.RECORD_BYTES:
            raise ValueError(f"world={self.world}: {n_results + 2} result records do not fit {L.RING_SLOT_BYTES} bytes")
        self._DRAIN = n_results         # result records of the drain and of the backlog's receive
        self.n_ids, self.n_recv = n_ids, n_recv
        dev = self.ctx.device
        self.landing = torch.zeros(n_ids * self.rec, dtype=torch.uint8, device=f"cuda:{dev}")
        self.words_full = torch.zeros(n_ids + GUARD, dtype=torch.int64, device=f"cuda:{dev}")
        self.words = self.words_full[:n_ids]
        self.landing_mr = self.ctx.reg_mr(self.landing)
        self.consumer_stream = torch.cuda.Stream(device=dev)
        self.main_stream = torch.cuda.Stream(device=dev)
        self._cleared = torch.cuda.Event()
        self.send_qp = self.recv_qp = self.remote_landing = None
        self.scratch_slot = None
        self.in_process = False
        self._views = []
        self._stale_cqes = 0            # receive completions a failed run left unreaped (in-process accounting)
        self._rq_backlog = 0            # receive WQEs a failed run left posted
        self._failed = False

    def _slot(self, m):
        """Landing slot ``m``: its R records and their arrival words."""
        return self.landing[m * self.R * self.rec:(m + 1) * self.R * self.rec], self.words[m * self.R:(m + 1) * self.R]

    # ---------------------------------------------------------------- links
    def _attach(self, send_qp, recv_qp, remote_landing, scratch_slot: int, grid: int, in_process: bool):
        depth = recv_qp.rq_depth
        cq_depth = recv_qp.rcq.depth
        if depth < 2 * self.n_recv or cq_depth < 2 * self.n_recv:
            raise ValueError(f"the receive queue ({depth}) and its CQ ({cq_depth}) must hold 2 * {self.n_recv} entries: "
                             f"{self.n_recv} receives per run, and those a failed run leaves behind")
        if remote_landing.length < self.landing.numel():
            raise ValueError("the next rank's landing region is smaller than this plan's")
        self.send_qp, self.recv_qp, self.remote_landing = send_qp, recv_qp, remote_landing
        self.scratch_slot, self.grid, self.in_process = scratch_slot, grid, in_process

    def connect(self, group=None, sq_depth: int = 256):
        """One process per GPU: create this rank's queue pair and connect it through ``parallel.peer.connect_ring``.
        Its send queue goes to the next rank, its receive queue takes the previous rank's records.  Collective."""
        import torch.distributed as dist
        from .peer import connect_ring
        if dist.get_rank(group) != self.rank or dist.get_world_size(group) != self.world:
            raise ValueError("the process group's rank and world size differ from the plan's")
        grid = self.grid or _default_grid(self.ctx, self.engine_ctas, 1, self.WAITERS)
        _check_budget(self.ctx, self.engine_ctas, 1, grid, self.WAITERS)
        depth = _pow2(2 * self.n_recv)
        scq = self.ctx.create_cq(2 * sq_depth)
        rcq = self.ctx.create_cq(depth)
        qp = self.ctx.create_qp(scq, rcq, sq_depth, depth)
        _, remote = connect_ring(self.ctx, qp, [self.landing_mr], group)
        self._attach(qp, qp, next(iter(remote.values())), 0, grid, in_process=False)

    # ---------------------------------------------------------------- run
    def _res(self, i: int) -> int:
        return L.ring_result_offset(self.scratch_slot, i)

    def _shard(self, t, s):
        s %= self.world
        return t[s * self.shard:(s + 1) * self.shard]

    def start_consumer(self):
        """Enqueue the consumer stream: clear the words, then receive and stamp this run's ``n_recv`` records."""
        if self.send_qp is None:
            raise RuntimeError("link the plan first: link_in_process(plans) or plan.connect()")
        if self._failed and not self.in_process:
            raise RuntimeError("a failed run leaves receive completions behind that only a new connection clears: "
                               "build new plans and connect them")
        if self._rq_backlog > self.n_recv:
            raise RuntimeError(f"{self._rq_backlog} receive WQEs are left from failed runs: link new plans")
        cs = self.consumer_stream
        kw = dict(timeout_ms=self.timeout_ms, stream=cs, sync=False)
        views = []
        if self._stale_cqes:
            # completions of a failed run's late records: reap them before this run's words are cleared
            views.append(("drain", "recv", ops.recv_consume(self.recv_qp, self._stale_cqes, 0, None, scratch_off=self._res(self._DRAIN), **kw)[0]))
        with torch.cuda.stream(cs):
            self.words.zero_()
        self._cleared.record(cs)
        self._receive(views, kw)
        self._stale_cqes = self._rq_backlog = 0
        self._views = views

    def _receive(self, views, kw):
        """Enqueue the receives of this run's ``n_recv`` records, the backlog's WQEs included."""
        fresh = self.n_recv - self._rq_backlog
        views.append(("receive", "recv", ops.recv_consume(self.recv_qp, fresh, self.n_ids, self.words, scratch_off=self._res(0),
                                                  prepost_mr=self.landing_mr, prepost_bytes=0, **kw)[0]))
        if self._rq_backlog:
            # the receive WQEs a failed run left posted take the rest of this run's records
            views.append(("receive", "recv", ops.recv_consume(self.recv_qp, self._rq_backlog, self.n_ids, self.words,
                                                      scratch_off=self._res(self._DRAIN + 1), **kw)[0]))

    def _reap(self, res: List[RingResult]):
        """After a run of every rank in one process: record what the run left in this rank's receive queue for the next
        run to reap -- completions nobody reaped, and receive WQEs no record took."""
        arrivals = res[(self.rank - 1) % self.world].posted
        self._stale_cqes = max(0, arrivals - res[self.rank].received)
        self._rq_backlog = max(0, self.n_recv - arrivals)

    def _streams(self):
        return (self.consumer_stream, self.main_stream)

    def _run(self, enqueue, sync: bool):
        """Start the consumer, ``enqueue()`` this rank's other streams, and with ``sync`` wait and return the result."""
        self.start_consumer()
        enqueue()
        if not sync:
            return None
        self.synchronize()
        return self.result()

    def synchronize(self):
        for s in self._streams():
            s.synchronize()

    def result(self) -> RingResult:
        """Decode the last run's result records (after :meth:`synchronize`)."""
        launches, received, posted = [], 0, 0
        for name, kind, view in self._views:
            w = L.decode(view, _WORDS[kind])
            launches.append(LaunchResult(name, w["status"], w["t_start_ns"], w["t_end_ns"]))
            posted += w.get("wqes", 0) + w.get("records_posted", 0) + w.get("records_forwarded", 0)
            received += w["seen"] if name == "receive" else 0
        bad = next((l for l in launches if l.status != "OK"), None)
        starts = [l.t_start_ns for l in launches if l.t_start_ns > 0]
        ends = [l.t_end_ns for l in launches if l.t_end_ns > 0]
        total = max(ends) - min(starts) if starts and ends else 0
        if bad is not None:
            self._failed = True
        return RingResult(self.rank, bad.status if bad else "OK", bad.name if bad else None, launches, total, received,
                          posted)


class RingAllreduceFp8(_RingPlan):
    """One rank's plan of the fp8 ring all-reduce of ``n_elems`` bf16 elements over ``world`` ranks.

    Everything is allocated and registered here, before any engine runs (DESIGN.md 3.2): the send staging (R records),
    the landing region (2(N-1) slots of R records), the arrival words with guard words behind them, and the streams.
    Link the plans with :func:`link_in_process` (N simulated ranks in one context) or :meth:`connect` (one process per
    GPU, through ``parallel.peer.connect_ring``), start the engine (``ctx.engine_start(ctas=engine_ctas)`` on the
    software HCA), then call :meth:`run`.

    ``grid`` is the CTAs of every launch (0: as many as the SM budget allows).  Every kernel that waits must be resident
    as a whole beside the engine and the other waiters, so ``engine_ctas + ranks on the GPU * (grid + 1)`` may not
    exceed the device's SMs.  ``timeout_ms`` bounds every wait; a rank whose input never comes ends ``TIMEOUT``.

    ``error_feedback``: carry this rank's quantisation error from run to run in ``residual`` (fp32, ``n_elems``, zero at
    first), so that the bias of the fp8 rounding does not accumulate over the steps of a training loop.  ``residual`` is
    a public tensor: copy it out and back in between runs to checkpoint it, and :meth:`reset_residual` zeroes it.  After
    a run that did not end OK it is undefined, as ``out`` is; reset it before the next run.  With error feedback every
    fp32 add of the pack and the hops saturates at +-FLT_MAX, so finite inputs always give a finite output and a finite
    residual, also at the top of the range (``ops.ref_allreduce_fp8`` with ``residuals=``)."""

    def __init__(self, ctx, n_elems: int, chunk_elems: int, rank: int, world: int, *, grid: int = 0,
                 timeout_ms: int = 2000, signal_every: int = 1, engine_ctas: int = 16, error_feedback: bool = False):
        super().__init__(ctx, chunk_elems, rank, world, grid, timeout_ms, signal_every, engine_ctas)
        n_elems, world, chunk_elems = int(n_elems), self.world, self.chunk
        if n_elems <= 0 or n_elems % (world * chunk_elems):
            raise ValueError(f"n_elems={n_elems} must be a multiple of world * chunk_elems = {world * chunk_elems}: "
                             "every shard is whole records")
        self.n = n_elems
        self.shard = n_elems // world
        self.R = self.shard // chunk_elems
        counter_bytes = L.counter_bytes(self.R + 3)       # the reduce's and the unpack's: R records and 3 words
        if counter_bytes > L.SLOT_BYTES:
            raise ValueError(f"{self.R} records per shard need {counter_bytes} bytes of counters; a scratch slot holds 256 KiB")
        if self.R > max_records(world):
            raise ValueError(f"R={self.R} records per shard: the receive queue would need {_pow2(4 * (world - 1) * self.R)} "
                             f"entries, above {MAX_QUEUE_DEPTH}; at world={world} R may be at most {max_records(world)}")
        # result records: 0 receive, 1.. the 2N launches of schedule()
        self._allocate(2 * (world - 1) * self.R, 2 * (world - 1) * self.R, 2 * world + 1)
        dev = ctx.device
        self.staging = torch.zeros(self.R * self.rec, dtype=torch.uint8, device=f"cuda:{dev}")
        self.residual = torch.zeros(n_elems, dtype=torch.float32, device=f"cuda:{dev}") if error_feedback else None
        self.staging_mr = ctx.reg_mr(self.staging)
        with torch.cuda.stream(self.consumer_stream):
            self.words.zero_()              # loads the fill kernel now: a first load later would wait for the engine
            if self.residual is not None:
                self.residual.zero_()       # and reset_residual()'s
        self._cleared.record(self.consumer_stream)
        torch.cuda.synchronize(dev)

    # ---------------------------------------------------------------- run
    @property
    def error_feedback(self) -> bool:
        return self.residual is not None

    def reset_residual(self):
        """Zero the error-feedback residual, on the main stream (ordered after the runs already enqueued)."""
        if self.residual is None:
            raise RuntimeError("this plan has no residual: build it with error_feedback=True")
        with torch.cuda.stream(self.main_stream):
            self.residual.zero_()

    def enqueue_main(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, steps=None):
        """Enqueue this rank's main stream (after :meth:`start_consumer`): K3, the N-1 reduce hops and the N unpacks.
        ``steps``: only these indices of :func:`schedule` (a caller that steps the ring from the host)."""
        out = x if out is None else out
        for t, what in ((x, "x"), (out, "out")):
            L.tensor_ptr(t, torch.bfloat16, self.ctx.device, what, self.n, exact=True, align=32)
        N, q, R, rec = self.world, self.rank, self.R, self.rec  # noqa: F841
        ms = self.main_stream
        if steps is None or 0 in steps:
            ms.wait_event(self._cleared)
        common = dict(grid=self.grid, timeout_ms=self.timeout_ms, stream=ms, sync=False, scratch_slot=self.scratch_slot)
        post = dict(with_imm=True, signal_every=self.signal_every)
        views = self._views
        ef = lambda s: {} if self.residual is None else dict(residual=self._shard(self.residual, s))  # noqa: E731
        for i, st in enumerate(schedule(q, N)):
            if steps is not None and i not in steps:
                continue
            res = self._res(1 + i)
            dst = {} if st.send_slot is None else dict(qp=self.send_qp, dst_mr=self.remote_landing, **post)
            if st.kind == "pack":
                v, _ = ops.pack_fp8_write(self.ctx, self._shard(x, st.shard), self.staging_mr, chunk_elems=self.chunk,
                                          result_off=res, **ef(st.shard), **dst, **common)
                views.append(("pack", "pack", v))
            elif st.kind == "reduce":
                land, words = self._slot(st.read_slot)
                v, _ = ops.reduce_fp8(self.ctx, land, 1, self.shard, self.chunk, local=self._shard(x, st.shard),
                                      out_mr=self.staging_mr, dst_off=st.send_slot * R * rec, ready=words,
                                      imm_base=st.send_slot * R, result_off=res, **ef(st.shard), **dst, **common)
                views.append((f"reduce hop {st.read_slot}", "reduce", v))
            elif st.read_slot is not None:
                land, words = self._slot(st.read_slot)
                fwd = {} if st.send_slot is None else dict(
                    fwd_qp=self.send_qp, fwd_src_mr=self.landing_mr, fwd_dst_mr=self.remote_landing,
                    fwd_dst_off=st.send_slot * R * rec, imm_base=st.send_slot * R, **post)
                v, _ = ops.unpack_fp8(self.ctx, land, self._shard(out, st.shard), self.chunk, ready=words, result_off=res,
                                      **fwd, **common)
                views.append((f"unpack slot {st.read_slot}" + (" + forward" if fwd else ""), "unpack", v))
            else:
                v, _ = ops.unpack_fp8(self.ctx, self.staging, self._shard(out, st.shard), self.chunk, result_off=res,
                                      **common)
                views.append(("unpack own", "unpack", v))

    def run(self, x: torch.Tensor, out: Optional[torch.Tensor] = None, sync: bool = True):
        """All-reduce ``x`` (bf16, ``n_elems``) over the ring into ``out``, or in place when ``out`` is None, as
        ``torch.distributed.all_reduce`` does.  Enqueues everything for this rank with no host step between hops; with
        ``sync`` waits and returns a :class:`RingResult`.  Ranks simulated in one process must all be enqueued before
        any is waited for: use :func:`run_in_process`.  After a run that did not end OK the contents of ``out`` are
        undefined, as with NCCL, and so is ``residual`` with error feedback."""
        return self._run(lambda: self.enqueue_main(x, out), sync)


def _sms(ctx) -> int:
    return torch.cuda.get_device_properties(ctx.device).multi_processor_count


def _default_grid(ctx, engine_ctas: int, ranks: int, waiters: int = 1) -> int:
    return max(1, min(64, (_sms(ctx) - engine_ctas) // ranks - waiters))


def _check_budget(ctx, engine_ctas: int, ranks: int, grid: int, waiters: int = 1):
    """``waiters``: the one-CTA waiting launches of a rank beside its grid (the consumer, and a plan's relay)."""
    need = engine_ctas + ranks * (grid + waiters)
    if need > _sms(ctx):
        others = "consumer 1" if waiters == 1 else f"consumer and relay {waiters}"
        raise ValueError(f"SM budget: engine {engine_ctas} + {ranks} ranks x (grid {grid} + {others}) = {need} CTAs, "
                         f"above the device's {_sms(ctx)} SMs; every waiting kernel must be resident as a whole")


def link_in_process(plans: List[_RingPlan], sq_depth: int = 256, rq_depth: Optional[int] = None):
    """Simulate N ranks in one context: connect the send QP of rank q to the receive QP of rank q+1 for every q, and
    give rank q device-scratch slot q.  Call before the engine starts."""
    N = len(plans)
    if N < 2 or any(p.world != N or p.rank != i for i, p in enumerate(plans)):
        raise ValueError("plans must be ranks 0..N-1 of one world of N >= 2")
    ctx = plans[0].ctx
    if any(type(p) is not type(plans[0]) or p.ctx is not ctx or (p.n, p.chunk) != (plans[0].n, plans[0].chunk) for p in plans):
        raise ValueError("in-process plans are of one kind and share one context, n_elems and chunk_elems")
    if N > MAX_IN_PROCESS:
        raise ValueError(f"{N} in-process ranks: the device scratch has {MAX_IN_PROCESS} slots, one per rank")
    waiters = plans[0].WAITERS
    grid = plans[0].grid or _default_grid(ctx, plans[0].engine_ctas, N, waiters)
    _check_budget(ctx, plans[0].engine_ctas, N, grid, waiters)
    depth = rq_depth if rq_depth is not None else _pow2(2 * plans[0].n_recv)
    if depth < 2 * plans[0].n_recv:
        raise ValueError(f"rq_depth={depth}: the receive queue and its CQ must hold 2 * {plans[0].n_recv} entries: "
                         f"{plans[0].n_recv} receives per run, and those a failed run leaves behind")
    send, recv = [], []
    for _ in range(N):
        send.append(ctx.create_qp(ctx.create_cq(2 * sq_depth), ctx.create_cq(64), sq_depth, 16))
        recv.append(ctx.create_qp(ctx.create_cq(64), ctx.create_cq(depth), 16, depth))
    for q in range(N):
        nxt = (q + 1) % N
        send[q].connect(recv[nxt])
        plans[q]._attach(send[q], recv[q], plans[nxt].landing_mr, q, grid, in_process=True)
    return plans


def run_in_process(plans: List[RingAllreduceFp8], xs, outs=None, sync: bool = True, skip=()):
    """Run the in-process ring: every consumer, then every main stream.  ``skip``: ranks whose main stream is not
    enqueued (a rank that never contributes; its receives are still posted).  Returns one :class:`RingResult` per rank
    with ``sync``."""
    outs = outs or [None] * len(plans)
    return _run_ranks(plans, [lambda p=p, x=x, o=o: p.enqueue_main(x, o) for p, x, o in zip(plans, xs, outs)], sync, skip)


def _run_ranks(plans: List[_RingPlan], enqueues, sync: bool, skip):
    """Every consumer, then ``enqueues[q]()`` for every rank q not in ``skip``; with ``sync`` wait, and record what a
    failed run leaves in each receive queue for the next run to reap.  Returns one :class:`RingResult` per rank."""
    for p in plans:
        p.start_consumer()
    for p, enqueue in zip(plans, enqueues):
        if p.rank not in skip:
            enqueue()
    if not sync:
        return None
    for p in plans:
        p.synchronize()
    res = [p.result() for p in plans]
    for p in plans:
        p._reap(res)
    return res
