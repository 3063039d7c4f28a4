"""The fp8 ring all-reduce on one GPU at the record geometries where its kernels' walks get hard, at the largest plans
the receive queue allows, at the benchmark's shapes, on the edge payload, and over repeated runs of one engine session.

* `UnpackSchedule` mirrors `pack_fp8.cu` as the ring launches the forwarding unpack (``unpack_fp8_kernel<true>`` with
  arrival words): the grid clamp to one slot's tile count, CTA b's steps T0 = b, b + grid * 4, ... with the tiles of a
  step at T0 + g * grid, and per step the records thread 0 waits on and may claim, in the order it visits them.  The
  reduce hops run ``test_gpu_reduce_schedule.ReduceSchedule`` with the addend and P = 1.  Every geometry case asserts
  the facts it is there for; test_ring_fp8_schedule.py checks the model against hand-counted walks on the CPU.
* Every rank must hold the same bits (NaN included: every rank unpacks the same records) and equal
  ``ops.ref_allreduce_fp8`` up to the sign of NaN; each rank posts and receives 2(N-1)R records, and its send queue
  grows by exactly those records plus 2N-2 flushes (K3, N-1 reduce hops and N-2 forwarding unpacks each post one).

The rules of test_gpu_ring_fp8.py hold: every wait is bounded by 5 s or less, nothing allocates or synchronises the
device while the engine runs, landing and staging buffers start as poison, the guard words behind the arrival words
stay zero, and each case writes out its SM budget (engine CTAs + N x (grid + 1) of 132).
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import ring_fp8 as RF
from test_gpu_numerics import H100_SMS
from test_gpu_receive_fusion import _check_arrival_words
from test_gpu_reduce import _bf16_equal_up_to_nan
from test_gpu_reduce_schedule import ReduceSchedule
from test_gpu_ring_fp8 import WAIT_MS, _poison
from test_ring_fp8_references import KINDS, _kind_blocks, assert_bits_equal, edge_payload, ring_blocks

pytestmark = pytest.mark.gpu

TILE = P.TILE_ELEMS
ENGINE_CTAS = 16


# ------------------------------------------------------------------ schedule model of the forwarding unpack
class UnpackSchedule:
    """One ``unpack_fp8(ready=, fwd_qp=)`` launch over one landing slot of R records of ``chunk``: ``steps[b]`` lists
    CTA b's steps, each as its tiles in the flattened record-major order (tile T belongs to record T // tpc)."""
    G = 4

    def __init__(self, chunk, R, grid=0, sms=H100_SMS):
        self.tpc, self.R = chunk // TILE, R
        self.total = R * self.tpc
        self.requested = grid if grid > 0 else sms
        self.grid = min(self.requested, self.total)
        G, g_, total = self.G, self.grid, self.total
        self.steps = [[[T0 + g * g_ for g in range(G) if T0 + g * g_ < total] for T0 in range(b, total, g_ * G)]
                      for b in range(g_)]

    def visits(self, tiles):
        """The records thread 0 waits on and may claim, in order (it skips a record equal to the one before)."""
        out = []
        for T in tiles:
            r = T // self.tpc
            if not out or out[-1] != r:
                out.append(r)
        return out

    def owners(self):
        own = {r: set() for r in range(self.R)}
        for b, steps in enumerate(self.steps):
            for tiles in steps:
                for T in tiles:
                    own[T // self.tpc].add(b)
        return own

    def sure_claims(self):
        """(CTA, step) -> the records that step claims whatever the timing: records only that CTA holds, at the first
        of its steps that visits them."""
        own, out = self.owners(), {}
        for b, steps in enumerate(self.steps):
            seen = set()
            for i, tiles in enumerate(steps):
                for r in self.visits(tiles):
                    if r not in seen and own[r] == {b}:
                        out.setdefault((b, i), set()).add(r)
                    seen.add(r)
        return out

    def facts(self):
        all_steps = [t for steps in self.steps for t in steps]
        return {
            "claims_two": any(len(rs) >= 2 for rs in self.sure_claims().values()),
            "record_raced": any(len(c) > 1 for c in self.owners().values()),
            "waits_on_a_later_record": any(len(self.visits(t)) > 1 for t in all_steps),
            "partial_last_step": any(len(t) < self.G for t in all_steps),
            "clamped_grid": self.requested > self.total,
        }


UNPACK_FACTS = ("claims_two", "record_raced", "waits_on_a_later_record", "partial_last_step", "clamped_grid")
REDUCE_FACTS = ("multi_tile_run", "boundary_in_step", "step_completes_two", "record_shared", "partial_last_step",
                "waits_on_a_later_record")


def ring_grid(N, grid, waiters=1):
    """The grid every launch of an in-process ring of N ranks gets (``link_in_process``): ``grid``, or the default
    beside ``waiters`` one-CTA waiting launches per rank (the consumer, and the all-gather's relay)."""
    return grid or max(1, min(64, (H100_SMS - ENGINE_CTAS) // N - waiters))


def case_facts(N, tpc, R, grid):
    """The facts of the forwarding unpack and of a reduce hop at one geometry, as the ring launches them."""
    g = ring_grid(N, grid)
    u = UnpackSchedule(tpc * TILE, R, g).facts()
    r = ReduceSchedule(tpc * TILE, R, 1, local=True, grid=g, ready=True).facts()
    return {k for k in UNPACK_FACTS if u[k]}, {k for k in REDUCE_FACTS if r[k]}


# (N, tiles per record, R, grid (0: default), signal_every), with the unpack facts and reduce facts each case claims
GEOMETRY_CASES = [
    ((2, 3, 5, 1, 3), {"claims_two", "partial_last_step", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "waits_on_a_later_record"}),
    ((3, 5, 4, 2, 1), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "record_shared", "waits_on_a_later_record"}),
    ((4, 8, 2, 3, 1), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((5, 1, 2, 7, 3), {"clamped_grid", "partial_last_step"},
     {"partial_last_step"}),
    ((5, 8, 5, 3, 1), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((6, 5, 5, 0, 3), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((6, 1, 4, 13, 1), {"clamped_grid", "partial_last_step"},
     {"partial_last_step"}),
    ((7, 3, 7, 2, 8), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((7, 5, 1, 1, 1), {"partial_last_step"},
     {"multi_tile_run", "partial_last_step"}),
    ((8, 128, 2, 0, 1), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((8, 3, 4, 7, 5), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((2, 128, 4, 0, 1), {"partial_last_step", "record_raced", "waits_on_a_later_record"},
     {"multi_tile_run", "partial_last_step", "record_shared", "waits_on_a_later_record"}),
    ((3, 1, 7, 1, 8), {"claims_two", "partial_last_step", "waits_on_a_later_record"},
     {"partial_last_step", "step_completes_two", "waits_on_a_later_record"}),
]
GEOMETRY_IDS = [f"N{n}-tpc{t}-R{r}-grid{g or 'default'}-sig{s}" for (n, t, r, g, s), _, _ in GEOMETRY_CASES]


# ------------------------------------------------------------------ running and checking
def _plans(ctx, N, chunk, R, grid=0, signal_every=1):
    plans = [RF.RingAllreduceFp8(ctx, N * R * chunk, chunk, q, N, grid=grid, timeout_ms=WAIT_MS,
                                 signal_every=signal_every, engine_ctas=ENGINE_CTAS) for q in range(N)]
    RF.link_in_process(plans)
    return plans


def _spread_gpu(N, n, seed, lo=-20, hi=20):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(n, generator=g, device="cuda") *
             torch.exp2(torch.randint(lo, hi + 1, (n // 32,), generator=g, device="cuda").float()).repeat_interleave(32)
             ).to(torch.bfloat16) for _ in range(N)]


def _run(ctx, plans, runs):
    """``runs``: [(inputs on the GPU, outputs or None)], run back to back in one engine session from poisoned landing
    and staging buffers.  Returns each run's results and each rank's send-queue WQE growth."""
    chunk = plans[0].chunk
    for p in plans:
        _poison(p.landing, chunk)
        _poison(p.staging, chunk)
    wqe0 = [p.send_qp.counters()["n_wqe"] for p in plans]
    torch.cuda.synchronize()
    results = []
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=WAIT_MS)
    try:
        for xs, outs in runs:
            results.append(RF.run_in_process(plans, xs, outs))
    finally:
        ctx.engine_stop()
    return results, [p.send_qp.counters()["n_wqe"] - w for p, w in zip(plans, wqe0)]


def _check(plans, results, wqe_growth, outs, wants):
    N, R = plans[0].world, plans[0].R
    for res in results:
        for r in res:
            assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
            assert r.posted == r.received == 2 * (N - 1) * R, (r.rank, r.posted, r.received)
    assert wqe_growth == [len(results) * (2 * (N - 1) * R + 2 * N - 2)] * N, wqe_growth
    for p in plans:
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0
    for got, want in zip(outs, wants):
        first = got[0].view(torch.int16)
        for q in range(N):
            assert torch.equal(got[q].view(torch.int16), first), f"rank {q} differs from rank 0"
        _bf16_equal_up_to_nan(got[0], want)


def _sm_budget(N, grid, waiters=1):
    need = ENGINE_CTAS + N * (ring_grid(N, grid, waiters) + waiters)
    assert need <= H100_SMS
    return need


# ------------------------------------------------------------------ 1. record geometries
@pytest.mark.parametrize("case,unpack_claims,reduce_claims", GEOMETRY_CASES, ids=GEOMETRY_IDS)
def test_ring_geometry(ctx, case, unpack_claims, reduce_claims):
    N, tpc, R, grid, sig = case
    u, r = case_facts(N, tpc, R, grid)
    assert u == unpack_claims and r == reduce_claims, (u, r)
    _sm_budget(N, grid)
    chunk = tpc * TILE
    plans = _plans(ctx, N, chunk, R, grid, sig)
    n = N * R * chunk
    xs = _spread_gpu(N, n, seed=1000 + 10 * N + tpc)
    want = ops.ref_allreduce_fp8(xs, chunk)
    outs = [torch.full_like(x, 7.0) for x in xs]
    results, growth = _run(ctx, plans, [(xs, outs)])
    _check(plans, results, growth, [outs], [want])


# ------------------------------------------------------------------ 2. the largest plans the receive queue allows
@pytest.mark.parametrize("N,R", [(2, 4096), (8, 585)])
def test_ring_largest_legal_plan(ctx, N, R):
    """N = 2, R = 4096: the receive queue at 16384, and each reduce hop posts 4096 records through a 256-deep send queue.
    N = 8, R = 585.  SMs: engine 16 + N x (default grid + 1) <= 132."""
    assert R == RF.max_records(N)
    _sm_budget(N, 0)
    chunk = 8192
    plans = _plans(ctx, N, chunk, R)
    assert plans[0].recv_qp.rq_depth == RF.MAX_QUEUE_DEPTH
    xs = _spread_gpu(N, N * R * chunk, seed=2000 + N)
    want = ops.ref_allreduce_fp8(xs, chunk)
    results, growth = _run(ctx, plans, [(xs, None)])
    _check(plans, results, growth, [xs], [want])


# ------------------------------------------------------------------ 3. the benchmark's shapes
def _edge_band(xs, chunk, seed):
    """The edge kinds of test_ring_fp8_references.py in the first 8 and last 8 blocks of every record: kind k of record
    j enters on rank (j + k) mod N at the head of the record and on rank (j + k + 1) mod N at its tail."""
    N = len(xs)
    g = torch.Generator().manual_seed(seed)
    n_rec = xs[0].numel() // chunk
    band = np.zeros((N, n_rec, 16, 32), np.float32)
    for j in range(n_rec):
        for k, kind in enumerate(KINDS):
            for slot, first in ((k, j + k), (8 + k, j + k + 1)):
                a, b, rest = _kind_blocks(kind, g)
                for q in range(N):
                    d = (q - first) % N
                    band[q, j, slot] = a if d == 0 else b if d == 1 else rest
    for q, x in enumerate(xs):
        rows = x.view(n_rec, -1, 32)
        t = torch.from_numpy(band[q]).to(torch.bfloat16).to(x.device)
        rows[:, :8] = t[:, :8]
        rows[:, -8:] = t[:, 8:]
    return xs


def test_reference_on_the_gpu_equals_the_reference_on_the_cpu():
    N, chunk = 4, 1 << 16
    xs = _edge_band(_spread_gpu(N, N * 2 * chunk, seed=3000), chunk, seed=3001)
    got = ops.ref_allreduce_fp8(xs, chunk).cpu()
    _bf16_equal_up_to_nan(got, ops.ref_allreduce_fp8([x.cpu() for x in xs], chunk))      # NaN signs may differ


@pytest.mark.parametrize("N", [2, 4, 8])
def test_ring_at_the_benchmark_shape(ctx, N):
    """2^26 elements, chunk 2^20 (R = 32, 16, 8), 16 engine CTAs, the default grid; spread exponents with an edge band.
    Every element against the GPU reference; the first and last block of every record and a seeded 1/256 of the rest
    against the independent model."""
    n, chunk = 1 << 26, 1 << 20
    _sm_budget(N, 0)
    plans = _plans(ctx, N, chunk, n // (N * chunk))
    xs = _edge_band(_spread_gpu(N, n, seed=4000 + N), chunk, seed=4100 + N)
    want = ops.ref_allreduce_fp8(xs, chunk)
    outs = [torch.full_like(x, 7.0) for x in xs]
    results, growth = _run(ctx, plans, [(xs, outs)])
    _check(plans, results, growth, [outs], [want])
    # the independent model on sampled blocks
    nb, bpr, m = n // 32, chunk // 32, n // N
    g = torch.Generator().manual_seed(4200 + N)
    pick = torch.zeros(nb, dtype=torch.bool)
    pick[::bpr] = True
    pick[bpr - 1::bpr] = True
    pick[torch.randint(0, nb, (nb // 256,), generator=g)] = True
    idx = pick.nonzero().flatten()
    xb = torch.stack([x.view(-1, 32)[idx.cuda()].cpu() for x in xs]).float().numpy()        # [rank, block, 32]
    got = outs[0].view(-1, 32)[idx.cuda()].cpu().reshape(-1)
    shard = (idx * 32 // m).numpy()
    want_bits = np.empty((len(idx), 32), np.uint16)
    for s in range(N):
        sel = shard == s
        want_bits[sel] = ring_blocks(xb[[(s + h) % N for h in range(N)]][:, sel])
    assert_bits_equal(got, want_bits.reshape(-1), f"N={N} sampled blocks")


# ------------------------------------------------------------------ 4. the edge payload through the ring
@pytest.mark.parametrize("N", [3, 8])
def test_ring_edge_payload(ctx, N):
    """Every edge kind enters every shard at every hop (records of two tiles); the finite top-of-range sums come out
    finite on every rank and within the bound."""
    xs_cpu, R = edge_payload(N, seed=5000 + N)
    chunk = 16384
    _sm_budget(N, 0)
    plans = _plans(ctx, N, chunk, R)
    want = ops.ref_allreduce_fp8(xs_cpu, chunk)
    xs = [x.cuda() for x in xs_cpu]
    outs = [torch.full_like(x, 7.0) for x in xs]
    results, growth = _run(ctx, plans, [(xs, outs)])
    _check(plans, results, growth, [outs], [want.cuda()])
    x = torch.stack(xs_cpu).double()
    exact = x.sum(0)
    top = (x.abs() >= 1e38).any(0) & torch.isfinite(x).all(0) & (x.abs() != 1.5 * 2.0 ** 127).all(0)
    got = outs[0].cpu().double()
    assert bool(top.any()) and bool(torch.isfinite(got[top]).all()), "a finite top-of-range sum came out non-finite"
    assert bool(((got[top] - exact[top]).abs() <= 2.0 ** -4 * N * x[:, top].abs().amax(0)).all())


# ------------------------------------------------------------------ 5. repeated runs in one engine session
def test_ring_repeated_runs_one_engine_session(ctx):
    """Three runs on one set of plans with the engine started once: different inputs, in place, into ``out``, in place.
    Scratch counters and claim flags shared by the pack, reduce and unpack launches of a rank's slot must clean
    themselves, the words must clear, and the receive queue's index wraps past its depth (3 x 2(N-1)R > 2 x 2(N-1)R)."""
    N, tpc, R = 4, 3, 5
    chunk = tpc * TILE
    _sm_budget(N, 3)
    plans = _plans(ctx, N, chunk, R, grid=3, signal_every=3)
    assert 3 * plans[0].n_ids > plans[0].recv_qp.rq_depth
    n = N * R * chunk
    runs, outs, wants = [], [], []
    for i in range(3):
        xs = _spread_gpu(N, n, seed=6000 + i)
        wants.append(ops.ref_allreduce_fp8(xs, chunk))
        o = None if i % 2 == 0 else [torch.full_like(x, 7.0) for x in xs]
        runs.append((xs, o))
        outs.append(xs if o is None else o)
    results, growth = _run(ctx, plans, runs)
    _check(plans, results, growth, outs, wants)
