"""K4 with a landed addend (``ops.gemm_reduce_send``) and the fp8 ring reduce-scatter (collective and fused with the
GEMM) on one GPU.

The rules of test_gpu_ring_fp8.py hold: every kernel that waits is resident with what it waits for, every wait is
bounded by 5 s or less, nothing allocates or synchronises the device while the engine runs, arrival words are the head
of a zeroed tensor whose guard words must stay zero, and landing buffers start as poison (e4m3 448 under scale 2^127)
before every run, so a record read before it has landed changes the result.  GEMM operands are small integers, so every
fp32 partial is exact whatever the order of the adds and the references are exact.
"""
import os
import subprocess
import sys
import time

import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel import reduce_scatter_fp8 as RS
from test_gpu_numerics import _gen
from test_gpu_receive_fusion import _check_arrival_words
from test_gpu_ring_fp8 import WAIT_MS, _poison

pytestmark = pytest.mark.gpu


def _ints(shape, lo, hi, g):
    return torch.randint(lo, hi + 1, shape, generator=g).to(torch.bfloat16)


def _landed(n, Nb, g):
    """n fp8 panel records of [128, Nb] halves of integers: what a previous rank's panels look like."""
    return ops.ref_fp8_panels((torch.randint(-96, 97, (128 * n, Nb), generator=g).float() * 0.5))


def _want(c, walk, add, send, land, Nb):
    """Staging records (by send id) and bf16 rows the op must produce: ``ref_reduce_fp8`` of each panel's exact fp32
    partial with its landed record, or ``ref_fp8_panels`` without one."""
    rec, chunk = ops.panel_record_bytes(Nb), 128 * Nb
    recs, rows = {}, []
    for p, m in enumerate(walk):
        part = c[128 * m:128 * (m + 1)]
        if add[p] >= 0:
            y, r = ops.ref_reduce_fp8(land[add[p] * rec:(add[p] + 1) * rec], 1, chunk, chunk, local=part.reshape(-1))
        else:
            y, r = part.reshape(-1).to(torch.bfloat16), ops.ref_fp8_panels(part)
        if send[p] >= 0:
            recs[send[p]] = r
        else:
            rows.append(y.reshape(128, Nb))
    return recs, (torch.cat(rows) if rows else None)


class _Op:
    """Operands and buffers of one gemm_reduce_send over a loopback QP, allocated before any engine runs."""

    def __init__(self, ctx, M, Nb, K, walk, add, send, n_land, seed):
        g = _gen(seed)
        self.ctx = ctx
        self.M, self.Nb, self.K, self.ids = M, Nb, K, [walk, add, send]
        self.rec = ops.panel_record_bytes(Nb)
        self.a_cpu, self.b_cpu = _ints((M, K), -2, 2, g), _ints((Nb, K), -2, 2, g)
        self.a, self.b = self.a_cpu.cuda(), self.b_cpu.cuda()
        self.c = self.a_cpu.float() @ self.b_cpu.float().T                          # exact
        self.land_cpu = _landed(max(n_land, 1), Nb, g)
        self.land = torch.zeros_like(self.land_cpu, device="cuda")
        self.words_full = torch.zeros(max(n_land, 1) + 8, dtype=torch.int64, device="cuda")
        self.ready = self.words_full[:max(n_land, 1)]
        n_send = sum(1 for s in send if s >= 0)
        self.staging = torch.zeros(max(n_send, 1) * self.rec, dtype=torch.uint8, device="cuda")
        self.dst = torch.zeros_like(self.staging)
        self.smr, self.dmr = ctx.reg_mr(self.staging), ctx.reg_mr(self.dst)
        n_out = len(send) - n_send
        self.out = torch.full((128 * n_out, Nb), 7.0, dtype=torch.bfloat16, device="cuda") if n_out else None
        self.walk, self.add, self.send = (torch.tensor(v, dtype=torch.int32, device="cuda") for v in self.ids)
        self.qp = ctx.loopback_qp(depth=64)

    def launch(self, **kw):
        kw.setdefault("ids_host", self.ids)                # checked from the host lists: no read-back during a session
        return ops.gemm_reduce_send(self.ctx, self.a, self.b, walk=self.walk, add_ids=self.add, send_ids=self.send,
                                    qp=self.qp, staging_mr=self.smr, dst_mr=self.dmr, landing=self.land, ready=self.ready,
                                    out=self.out, with_imm=False, **kw)

    def check(self, posted_ids=None):
        recs, rows = _want(self.c, *self.ids, self.land_cpu, self.Nb)
        st, ds = self.staging.cpu(), self.dst.cpu()
        for i, r in recs.items():
            if posted_ids is not None and i not in posted_ids:
                continue
            assert torch.equal(st[i * self.rec:(i + 1) * self.rec], r), f"staging record {i}"
            assert torch.equal(ds[i * self.rec:(i + 1) * self.rec], r), f"destination record {i}"
        if rows is not None and posted_ids is None:
            assert torch.equal(self.out.cpu().view(torch.int16), rows.view(torch.int16)), "bf16 rows"


@pytest.fixture
def op_factory(ctx):
    return lambda *args, **kw: _Op(ctx, *args, **kw)


# ------------------------------------------------------------------ 1. the op alone
def test_no_addend_walk_is_gemm_send_fp8(ctx, op_factory):
    """A walk without addends, each panel posted as the record of its own m-block: the same bytes as
    ``gemm_send(out_fp8=True)``, in staging and at the destination, and n_wqe == records + 1."""
    M, Nb, K = 512, 512, 256
    walk = [2, 0, 3, 1]
    o = op_factory(M, Nb, K, walk, [-1] * 4, walk, 0, seed=1)
    torch.cuda.synchronize()
    r = o.launch(post_only=True)
    assert r.ok and r.records_posted == 4 and r.records_added == 0, r
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    ref = torch.zeros(4 * o.rec, dtype=torch.uint8, device="cuda")
    assert ops.gemm_send(ctx, o.a, o.b, ref, out_fp8=True, cta_group=1).ok
    assert torch.equal(o.staging, ref) and torch.equal(o.dst, ref)
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 4 + 1, q


@pytest.mark.parametrize("Nb,K", [(512, 256), (320, 200)], ids=["tile-multiple", "ragged"])
def test_addends_set_late_and_out_of_order(ctx, op_factory, Nb, K):
    """Landed records and their words are set on another stream, in another order, after the launch; the GEMM adds
    them, posts three records and stores two bf16 row blocks, all bit-identical to the reference.  The ragged case has Nb
    a multiple of 64 but not of 256 and K not a multiple of 64."""
    walk, add, send = [3, 1, 4, 0, 2], [-1, 0, 2, 1, 3], [0, -1, 1, -1, 2]
    o = op_factory(640, Nb, K, walk, add, send, 4, seed=2 + Nb)
    s_set, s_g = ctx.streams(2)
    order = [2, 0, 3, 1]
    rec = o.rec
    src = o.land_cpu.cuda()
    # the setter runs once before the engine: a kernel's first load waits for every resident kernel (DESIGN.md 3.2)
    with torch.cuda.stream(s_set):
        for i in order:
            o.land[i * rec:(i + 1) * rec].copy_(src[i * rec:(i + 1) * rec])
            o.ready[i:i + 1].fill_(1)
    torch.cuda.synchronize()
    _poison(o.land, 128 * Nb)
    o.words_full.zero_()
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        v, _ = o.launch(timeout_ms=WAIT_MS, stream=s_g, sync=False)
        with torch.cuda.stream(s_set):
            for i in order:
                o.land[i * rec:(i + 1) * rec].copy_(src[i * rec:(i + 1) * rec])
                o.ready[i:i + 1].fill_(1)
        s_set.synchronize()
        s_g.synchronize()
    finally:
        ctx.engine_stop()
    r = ops.parse_reduce_send(v)
    assert r.ok and r.records_posted == 3 and r.records_added == 4 and r.t_first_post_ns > 0, r
    o.check()
    assert bool((o.words_full[4:] == 0).all()), "a guard word was written"
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 3 + 1, q


def test_withheld_word_times_out(ctx, op_factory):
    """One CTA walks [0, 1, 2, 3]; position 1's word is withheld, 2's and 3's are set.  Position 0 (no addend) is posted,
    then the launch ends TIMEOUT within the bound and no later record is posted."""
    walk, add, send = [0, 1, 2, 3], [-1, 0, 1, 2], [0, 1, 2, 3]
    o = op_factory(512, 256, 128, walk, add, send, 3, seed=3)
    o.land.copy_(o.land_cpu.cuda())
    o.ready[1:].fill_(1)
    torch.cuda.synchronize()
    t0 = time.monotonic()
    r = o.launch(grid=1, timeout_ms=300, post_only=True)
    dt = time.monotonic() - t0
    assert r.status == "TIMEOUT" and r.records_posted == 1 and r.records_added == 0, r
    assert dt < 3.0, f"the timeout took {dt:.2f} s"
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    o.check(posted_ids={0})
    assert bool((o.dst[o.rec:] == 0).all()), "a record after the withheld one reached the destination"
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 1 + 1, q


def test_partial_step_leaves_the_scratch_clean(ctx, op_factory):
    """Nb = 512 (two tiles per panel), group_m = 4, three CTAs: tile t is panel t % 4, n-block t // 4, and CTA u takes
    tiles u, u + 3, u + 6.  Panel 2's word is withheld, the others are set.  CTA 2 times out on panel 2 and drops its
    later tile of panel 1, whose other tile CTA 1 stores and counts: panels 0 and 3 are posted, panel 1 is left with
    one tile of two counted.  The failed launch must still leave its scratch slot clean, so that two later launches on
    it (every word set) post every panel after all its tiles, bit-identical to the reference; a stale count would post
    panel 1 early in the first of them and never in the second."""
    walk = [0, 1, 2, 3]
    o = op_factory(512, 512, 128, walk, walk, walk, 4, seed=5)
    o.land.copy_(o.land_cpu.cuda())
    o.ready.fill_(1)
    o.ready[2] = 0
    torch.cuda.synchronize()
    r = o.launch(grid=3, group_m=4, timeout_ms=300, post_only=True)
    assert r.status == "TIMEOUT" and r.records_posted == 2 and r.records_added == 2, r
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    o.check(posted_ids={0, 3})
    o.ready[2] = 1
    torch.cuda.synchronize()
    for _ in range(2):
        o.staging.zero_()
        o.dst.zero_()
        torch.cuda.synchronize()
        r = o.launch(grid=3, group_m=4, timeout_ms=WAIT_MS, post_only=True)
        assert r.ok and r.records_posted == 4 and r.records_added == 4, r
        ctx.engine_run_oneshot(ctas=8)
        torch.cuda.synchronize()
        o.check()
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == (2 + 1) + 2 * (4 + 1), q


def test_a_timed_out_gate_ends_every_other_gate(ctx, op_factory):
    """Two CTAs, one tile per panel: CTA 0 walks panels 0 and 2, CTA 1 panels 1 and 3.  Words 0, 2 and 3 are withheld;
    word 1 is set by another stream after a spin of about 0.2 s.  CTA 0 times out on panel 0 at timeout_ms; CTA 1 posts
    panel 1 late and then gates panel 3.  With the grid-wide flag CTA 1's second gate ends with CTA 0's timeout, so the
    launch lasts about one timeout; a gate that only ran out its own timeout would end about 0.2 s later."""
    walk = [0, 1, 2, 3]
    tmo_ms = 1000
    o = op_factory(512, 256, 128, walk, walk, walk, 4, seed=6)
    o.land.copy_(o.land_cpu.cuda())
    s_set, s_g = ctx.streams(2)
    # load the spin and the fill now: a kernel's first load waits for every resident kernel (DESIGN.md 3.2)
    with torch.cuda.stream(s_set):
        torch.cuda._sleep(1000)
        o.ready[1:2].fill_(1)
    torch.cuda.synchronize()
    o.words_full.zero_()
    torch.cuda.synchronize()
    v, _ = o.launch(grid=2, group_m=1, timeout_ms=tmo_ms, post_only=True, stream=s_g, sync=False)
    with torch.cuda.stream(s_set):
        torch.cuda._sleep(400_000_000)
        o.ready[1:2].fill_(1)
    s_set.synchronize()
    s_g.synchronize()
    r = ops.parse_reduce_send(v)
    assert r.status == "TIMEOUT" and r.records_posted == 1 and r.records_added == 1, r
    assert r.t_first_post_ns - r.t_start_ns > 100_000_000, "panel 1 was not gated behind the late word"
    assert r.device_ns < (tmo_ms + 120) * 1_000_000, f"the launch took {r.device_ns / 1e6:.0f} ms"
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    o.check(posted_ids={1})
    q = o.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 1 + 1, q


def test_host_rejections(ctx, op_factory):
    o = op_factory(256, 256, 64, [0, 1], [-1, 0], [0, -1], 1, seed=4)
    bad = [
        (dict(cta_group=2), "cta_group"), (dict(direct=True), "direct"), (dict(plain_stores=True), "plain_stores"),
        (dict(stream_k=True), "stream_k"), (dict(ids_host=[[0, 0], [-1, 0], [0, -1]]), "every m-block"),
        (dict(ids_host=[[0, 2], [-1, 0], [0, -1]]), "every m-block"), (dict(ids_host=[[0, 1], [-1, 1], [0, -1]]), "add_ids"),
        (dict(ids_host=[[0, 1], [-1, 0], [0, 1]]), "send_ids"), (dict(ids_host=[[0, 1], [-1, 0], [-2, -1]]), "send_ids"),
    ]
    for kw, what in bad:
        with pytest.raises(ValueError, match=what):
            o.launch(**kw)
    with pytest.raises(ValueError, match="Nb of 32"):
        ops.gemm_reduce_send(ctx, o.a, o.b[:48].contiguous(), walk=o.walk, add_ids=o.add, send_ids=o.send, qp=o.qp,
                             staging_mr=o.smr, dst_mr=o.dmr, landing=o.land, ready=o.ready, out=o.out, ids_host=o.ids)
    a2 = torch.zeros(512, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="overlap"):
        ops.gemm_reduce_send(ctx, a2[:256], o.b, walk=o.walk, add_ids=o.add, send_ids=o.send, qp=o.qp, staging_mr=o.smr,
                             dst_mr=o.dmr, landing=o.land, ready=o.ready, out=a2.view(128, 256), ids_host=o.ids)


# ------------------------------------------------------------------ 2. the reduce-scatter, N simulated ranks
def _plans(ctx, N, shard, chunk, timeout_ms=WAIT_MS):
    plans = [RS.RingReduceScatterFp8(ctx, shard, chunk, q, N, timeout_ms=timeout_ms) for q in range(N)]
    RS.link_in_process(plans)
    return plans


def _inputs(N, n, seed):
    g = _gen(seed)
    return [(torch.randn(n, generator=g) * 4 ** (q % 3)).to(torch.bfloat16) for q in range(N)]


def _check_run(plans, res, outs, want):
    for r in res:
        assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
        assert r.received == plans[0].n_recv and r.posted == plans[0].n_recv, (r.rank, r.received, r.posted)
    for q, p in enumerate(plans):
        assert torch.equal(outs[q].cpu().view(torch.int16), want[q].view(torch.int16)), f"rank {q} differs from the reference"
        _check_arrival_words(p.words_full, p.n_ids)
        assert p.send_qp.counters()["n_err"] == 0


def _run(ctx, plans, xs_cpu):
    N = len(plans)
    xs = [x.cuda() for x in xs_cpu]
    outs = [torch.full((plans[0].shard,), 7.0, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    for p in plans:
        _poison(p.landing, p.chunk)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = RS.run_in_process(plans, xs, outs)
    finally:
        ctx.engine_stop()
    _check_run(plans, res, outs, ops.ref_reduce_scatter_fp8(xs_cpu, plans[0].chunk))
    return outs


@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_reduce_scatter_matches_reference(ctx, N):
    chunk, R = 8192, 2
    plans = _plans(ctx, N, R * chunk, chunk)
    _run(ctx, plans, _inputs(N, N * R * chunk, seed=10 + N))


def _gemm_operands(N, M, Nb, K, g, select=False):
    a = [_ints((M, K), -4, 4, g) for _ in range(N)]
    if select:                              # b a 0/1 column selection: every partial is exact in bf16
        b = []
        for _ in range(N):
            t = torch.zeros(Nb, K)
            t[torch.arange(Nb), torch.randint(0, K, (Nb,), generator=g)] = 1
            b.append(t.to(torch.bfloat16))
    else:
        b = [_ints((Nb, K), -2, 2, g) for _ in range(N)]
    return a, b


def _run_gemm(ctx, plans, a_cpu, b_cpu, Nb):
    N, M = len(plans), a_cpu[0].shape[0]
    a, b = [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    outs = [torch.full((M // N, Nb), 7.0, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    for p in plans:
        _poison(p.landing, p.chunk)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = RS.run_gemm_in_process(plans, a, b, outs)
    finally:
        ctx.engine_stop()
    parts = [(x.float() @ y.float().T).reshape(-1) for x, y in zip(a_cpu, b_cpu)]
    want = [w.reshape(M // N, Nb) for w in ops.ref_reduce_scatter_fp8(parts, 128 * Nb)]
    _check_run(plans, res, outs, want)
    for r in res:
        g = [l for l in r.launches if l.name == "gemm"]
        assert len(g) == 1 and g[0].status == "OK"
    return outs


@pytest.mark.parametrize("N", [2, 4, 8])
def test_reduce_scatter_gemm(ctx, N):
    """K_l = 128, Nb = 256, two 128-row panels per shard: every rank bit-identical to the reference of its partials."""
    Nb, K, R = 256, 128, 2
    M = N * 128 * R
    plans = _plans(ctx, N, (M // N) * Nb, 128 * Nb)
    a, b = _gemm_operands(N, M, Nb, K, _gen(30 + N))
    _run_gemm(ctx, plans, a, b, Nb)


def test_reduce_scatter_gemm_equals_gemm_then_run(ctx):
    """With bf16-exact partials, run_gemm gives the bits of every rank's gemm_send (bf16 C) followed by run."""
    N, Nb, K, R = 4, 320, 200, 1
    M = N * 128 * R
    plans = _plans(ctx, N, (M // N) * Nb, 128 * Nb)
    a, b = _gemm_operands(N, M, Nb, K, _gen(40), select=True)
    fused = _run_gemm(ctx, plans, a, b, Nb)
    cs = []
    for x, y in zip(a, b):
        c = torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda")
        assert ops.gemm_send(ctx, x.cuda(), y.cuda(), c).ok
        cs.append(c.reshape(-1).cpu())
    assert all(torch.equal(c.float(), (x.float() @ y.float().T).reshape(-1)) for c, x, y in zip(cs, a, b))
    unfused = _run(ctx, plans, cs)
    for q in range(N):
        assert torch.equal(fused[q].reshape(-1).view(torch.int16), unfused[q].view(torch.int16)), q


def test_run_and_run_gemm_alternate_in_one_session(ctx):
    N, Nb, K = 3, 256, 64
    M = N * 128
    chunk = 128 * Nb
    plans = _plans(ctx, N, (M // N) * Nb, chunk)
    g = _gen(50)
    xs_cpu = _inputs(N, N * chunk, seed=51)
    a_cpu, b_cpu = _gemm_operands(N, M, Nb, K, g)
    xs, a, b = [x.cuda() for x in xs_cpu], [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    outs = [[torch.zeros(chunk, dtype=torch.bfloat16, device="cuda") for _ in range(N)] for _ in range(4)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = [RS.run_in_process(plans, xs, outs[0]), RS.run_gemm_in_process(plans, a, b, [o.view(128, Nb) for o in outs[1]]),
               RS.run_in_process(plans, xs, outs[2]), RS.run_gemm_in_process(plans, a, b, [o.view(128, Nb) for o in outs[3]])]
    finally:
        ctx.engine_stop()
    want_x = ops.ref_reduce_scatter_fp8(xs_cpu, chunk)
    want_g = ops.ref_reduce_scatter_fp8([(x.float() @ y.float().T).reshape(-1) for x, y in zip(a_cpu, b_cpu)], chunk)
    for i in range(4):
        _check_run(plans, res[i], outs[i], want_x if i % 2 == 0 else want_g)


def test_rank_that_never_contributes(ctx):
    """Rank 1 posts its receives but never runs its GEMM: the ranks downstream report TIMEOUT and the run ends within
    2N x timeout_ms.  The next run, with every rank, is clean."""
    N, Nb, K = 3, 256, 64
    M = N * 256
    plans = _plans(ctx, N, (M // N) * Nb, 128 * Nb, timeout_ms=300)
    a_cpu, b_cpu = _gemm_operands(N, M, Nb, K, _gen(60))
    a, b = [t.cuda() for t in a_cpu], [t.cuda() for t in b_cpu]
    outs = [torch.zeros(M // N, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        res = RS.run_gemm_in_process(plans, a, b, outs, skip={1})
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    assert res[2].status == "TIMEOUT", (res[2].status, res[2].failed)
    for r in res:
        for l in r.launches:
            assert l.status in ("OK", "TIMEOUT"), (r.rank, l)
    assert dt < 2 * N * 0.3 + 1.0, f"the failed run took {dt:.2f} s"
    _run_gemm(ctx, plans, a_cpu, b_cpu, Nb)


def test_plan_rejections(ctx):
    with pytest.raises(ValueError, match="SM budget"):
        RS.link_in_process([RS.RingReduceScatterFp8(ctx, 8192, 8192, q, 2, grid=58) for q in range(2)])
    plans = _plans(ctx, 2, 128 * 256, 128 * 256)
    x = torch.zeros(2 * 128 * 256, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="overlap"):
        plans[0].run(x, x[:128 * 256])
    a = torch.zeros(256, 64, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(256, 64, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="128 \\* Nb"):
        plans[0].run_gemm(a, b[:128].contiguous(), torch.zeros(128, 128, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(ValueError, match="world \\* 128"):
        plans[0].run_gemm(a[:128].contiguous(), b, torch.zeros(64, 256, dtype=torch.bfloat16, device="cuda"))


_FIRST_RUN = """
import sys
import torch
sys.path.insert(0, {root!r})
import rocnrdma_b200 as rn
from rocnrdma_b200 import ops
from rocnrdma_b200.parallel import reduce_scatter_fp8 as RS
ctx = rn.Context(device=0)
N, Nb, K = {N}, 256, 64
M = N * 128 * {R}
plans = [RS.RingReduceScatterFp8(ctx, (M // N) * Nb, 128 * Nb, q, N, timeout_ms=2000) for q in range(N)]
RS.link_in_process(plans)
g = torch.Generator().manual_seed(7)
a = [torch.randint(-2, 3, (M, K), generator=g).to(torch.bfloat16) for _ in range(N)]
b = [torch.randint(-2, 3, (Nb, K), generator=g).to(torch.bfloat16) for _ in range(N)]
outs = [torch.zeros(M // N, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
ad, bd = [t.cuda() for t in a], [t.cuda() for t in b]
xs = [torch.randint(-64, 65, (M * Nb,), generator=g).to(torch.bfloat16) for _ in range(N)]
xd = [t.cuda() for t in xs]
torch.cuda.synchronize()
ctx.engine_start(ctas=16, idle_timeout_ms=5000)
try:
    if {kind!r} == "run":
        res = RS.run_in_process(plans, xd, [o.reshape(-1) for o in outs])
    else:
        res = RS.run_gemm_in_process(plans, ad, bd, outs)
finally:
    ctx.engine_stop()
if {kind!r} == "run":
    want = ops.ref_reduce_scatter_fp8(xs, 128 * Nb)
else:
    want = ops.ref_reduce_scatter_fp8([(x.float() @ y.float().T).reshape(-1) for x, y in zip(a, b)], 128 * Nb)
print("statuses", *[r.status for r in res])
print("exact", all(torch.equal(o.cpu().reshape(-1).view(torch.int16), w.view(torch.int16)) for o, w in zip(outs, want)))
ctx.close()
"""


@pytest.mark.parametrize("N,R,kind", [(2, 3, "run_gemm"), (3, 1, "run_gemm"), (2, 3, "run"), (3, 1, "run")],
                         ids=["2-3", "3-1", "run-2-3", "run-3-1"])
def test_first_run_of_a_fresh_process(N, R, kind):
    """The first run_gemm, or the first run, of a new process: every kernel a run uses is loaded before the engine
    starts."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", _FIRST_RUN.format(root=root, N=N, R=R, kind=kind)], capture_output=True,
                       text=True, timeout=300, cwd=root)
    assert p.returncode == 0, p.stderr[-3000:]
    assert f"statuses {' '.join(['OK'] * N)}" in p.stdout and "exact True" in p.stdout, p.stdout
