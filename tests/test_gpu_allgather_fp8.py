"""The record relay, K7's ordered walk and the fp8 ring all-gather (collective and fused with K7) on one GPU.

The rules of test_gpu_ring_fp8.py hold: every kernel that waits is resident with what it waits for, every wait is
bounded by 5 s or less, nothing allocates or synchronises the device while the engine runs, arrival words are the head
of a zeroed tensor whose guard words must stay zero, and landing buffers start as poison (e4m3 448 under scale 2^127)
before every run, so a record read or relayed before it has landed changes the result.
"""
import time

import pytest
import torch

from rocnrdma_b200 import _native as NAT, ops
from rocnrdma_b200.ops import gemm_mx as MX, pack as P
from rocnrdma_b200.parallel import allgather_fp8 as AG
from test_gpu_numerics import _bits_equal, _gen, _mx_exact_operand, _spread
from test_gpu_receive_fusion import _Records, _arrival_words, _check_arrival_words
from test_gpu_ring_fp8 import POISON_Q, WAIT_MS, _Fwd, _poison

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ 1. relay_records alone
@pytest.mark.parametrize("signal_every", [1, 3])
def test_relay_words_set_late_and_out_of_order(ctx, signal_every):
    """The relay is launched on poisoned records in one order; another stream lands and stamps them in another.  Each
    record is posted once, as WRITE_IMM with immediate r: the destination's words are exactly the relayed ids, the bytes
    are the records', and n_wqe == records + 1."""
    chunk, n_rec = 16384, 7
    f = _Fwd(ctx, chunk, n_rec, 0, seed=21)
    rec = P.record_bytes(chunk)
    ids = torch.randperm(n_rec, generator=_gen(22))[:6].to(torch.int32)
    land_order = torch.randperm(n_rec, generator=_gen(23)).tolist()
    ids_dev = ids.cuda()
    s_set, s_c, s_r = ctx.streams(3)
    # the setter runs once before the relay exists: a kernel's first load waits for every resident kernel (DESIGN.md 3.2)
    with torch.cuda.stream(s_set):
        for r in land_order:
            f.land[r * rec:(r + 1) * rec].copy_(f.src[r * rec:(r + 1) * rec])
            f.ready[r:r + 1].fill_(1)
    torch.cuda.synchronize()
    _poison(f.land[:f.nb], chunk)
    f.full.zero_()
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cv, _ = ops.recv_consume(f.qp, len(ids), n_rec, f.dready, timeout_ms=WAIT_MS, sync=False, stream=s_c,
                                 prepost_mr=f.dmr, prepost_bytes=0)
        rv, _ = ops.relay_records(f.qp, f.lmr, f.dmr, rec, ids_dev, ready=f.ready, signal_every=signal_every,
                                  timeout_ms=WAIT_MS, stream=s_r, sync=False)
        with torch.cuda.stream(s_set):
            for r in land_order:
                f.land[r * rec:(r + 1) * rec].copy_(f.src[r * rec:(r + 1) * rec])
                f.ready[r:r + 1].fill_(1)
        for s in (s_set, s_c, s_r):
            s.synchronize()
    finally:
        ctx.engine_stop()
    r = ops.parse_relay(rv)
    assert r["status"] == "OK" and r["records_posted"] == len(ids) and r["t_first_post_ns"] > 0, r
    c = ops.parse_recv(cv)
    assert c["status"] == "OK" and c["seen"] == len(ids), c
    relayed = set(ids.tolist())
    st = f.dfull.tolist()
    assert all((st[i] != 0) == (i in relayed) for i in range(n_rec)), st
    assert all(v == 0 for v in st[n_rec:]), "a guard word was written"
    f.check_bytes(relayed)
    q = f.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == len(ids) + 1, q


def test_relay_withheld_word_times_out(ctx):
    """ids [3, 0, 2, 1] with word 2 withheld: records 3 and 0 are posted, then TIMEOUT within the bound; record 1, whose
    word is set, comes after 2 and is never posted."""
    chunk, n_rec = 8192, 4
    f = _Fwd(ctx, chunk, n_rec, 0, seed=24)
    f.land[:f.nb].copy_(f.src)
    f.ready.fill_(1)
    f.ready[2] = 0
    ids = torch.tensor([3, 0, 2, 1], dtype=torch.int32, device="cuda")
    s_c, s_r = ctx.streams(2)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cv, _ = ops.recv_consume(f.qp, 2, n_rec, f.dready, timeout_ms=WAIT_MS, sync=False, stream=s_c,
                                 prepost_mr=f.dmr, prepost_bytes=0)
        t0 = time.monotonic()
        r = ops.relay_records(f.qp, f.lmr, f.dmr, f.nb // n_rec, ids, ready=f.ready, timeout_ms=300, stream=s_r)
        dt = time.monotonic() - t0
        s_c.synchronize()
    finally:
        ctx.engine_stop()
    assert r["status"] == "TIMEOUT" and r["records_posted"] == 2, r
    assert dt < 3.0, f"the timeout took {dt:.2f} s"
    st = f.dfull.tolist()
    assert [st[i] != 0 for i in range(n_rec)] == [True, False, False, True], st
    f.check_bytes({0, 3})
    q = f.qp.counters()
    assert q["n_err"] == 0 and q["n_wqe"] == 3, q                  # two records and the flush


def test_relay_id_outside_the_records(ctx):
    """An id past the records ends the relay with -22 before it posts anything for that id; the records before it go."""
    chunk, n_rec = 8192, 3
    f = _Fwd(ctx, chunk, n_rec, 0, seed=25)
    f.land[:f.nb].copy_(f.src)
    for _ in range(n_rec):
        f.qp.post_recv(f.dmr, 0)
    ids = torch.tensor([1, n_rec, 0], dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    r = ops.relay_records(f.qp, f.lmr, f.dmr, P.record_bytes(chunk), ids, post_only=True)
    assert r["status"] == "-22" and r["records_posted"] == 1, r
    ctx.engine_run_oneshot(ctas=8)
    torch.cuda.synchronize()
    f.check_bytes({1})


def test_relay_host_rejections(ctx):
    chunk, n_rec = 8192, 2
    f = _Fwd(ctx, chunk, n_rec, 0, seed=26)
    rec = P.record_bytes(chunk)
    ids = torch.zeros(2, dtype=torch.int32, device="cuda")
    bad = [
        (dict(rec_bytes=rec + 1), "multiple of 64"),
        (dict(rec_bytes=0), "multiple of 64"),
        (dict(rec_bytes=f.nb + 64), "must hold a record"),
        (dict(ids=ids.long()), "int32"),
        (dict(ids=ids.cpu()), "cuda"),
        (dict(ids=ids[:0]), "non-empty"),
        (dict(ready=f.ready[:1]), "at least 2"),
        (dict(ready=f.ready.int()), "int64"),
        (dict(scratch_slot=8), "scratch_slot"),
    ]
    torch.cuda.synchronize()
    for kw, what in bad:
        args = dict(rec_bytes=rec, ids=ids, ready=f.ready)
        args.update(kw)
        rb, i = args.pop("rec_bytes"), args.pop("ids")
        with pytest.raises(ValueError, match=what):
            ops.relay_records(f.qp, f.lmr, f.dmr, rb, i, **args)
    assert f.qp.counters()["n_wqe"] == 0


# ------------------------------------------------------------------ 2. gemm_mxfp8(a_order=)
@pytest.mark.parametrize("order", ["identity", "perm0", "perm1", "reverse"])
@pytest.mark.parametrize("M", [1024, 2048])
def test_ordered_k7_on_arrival_matches_unordered(ctx, M, order):
    """K3 records of 256 rows land through recv_consume while the ordered K7 waits on their words; C is bit-identical to
    K7 without an order run on the same records after they arrived."""
    K, Nb = 256, 392
    chunk = 256 * K
    L = _Records("chunk", M, K)
    g = _gen(M + len(order))
    x = _spread(M, K, g, 32).to(torch.bfloat16).cuda()
    bq, bs = _mx_exact_operand(Nb, K, g)
    ids = {"identity": list(range(L.n)), "reverse": list(range(L.n))[::-1]}.get(order)
    if ids is None:
        ids = torch.randperm(L.n, generator=_gen(int(order[-1]) + M)).tolist()
    a_order = torch.tensor(ids, dtype=torch.int32, device="cuda")
    nb = L.n * L.bytes
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    rcv = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L.poison(rcv)
    y = torch.full((M, Nb), 7.0, dtype=torch.bfloat16, device="cuda")
    y0 = torch.zeros_like(y)
    full, ready = _arrival_words(L.n)
    smr, rmr = ctx.reg_mr(stg), ctx.reg_mr(rcv)
    qp = ctx.loopback_qp(depth=64)
    a_op, b_op = L.operand(rcv), MX.MxOperand.from_tensors(bq, bs)
    _, s_recv, s_mm = ctx.streams(3)
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + GEMM 48 + pack 32 = 89 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, L.n, L.n, ready, timeout_ms=WAIT_MS, sync=False, stream=s_recv, prepost_mr=rmr,
                                    prepost_bytes=0)
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=48, cta_group=1, a_ready=ready, a_order=a_order,
                                  timeout_ms=WAIT_MS, sync=False, stream=s_mm)
        r = ops.pack_fp8_write(ctx, x.reshape(-1), smr, qp=qp, dst_mr=rmr, chunk_elems=chunk, with_imm=True, grid=32,
                               timeout_ms=WAIT_MS)
        s_recv.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.wqes == L.n, r
    assert ops.parse_recv(cview)["seen"] == L.n
    _check_arrival_words(full, L.n)
    assert torch.equal(rcv, ops.ref_pack_fp8(x.reshape(-1), chunk).cuda())
    g1 = MX._parse(gview, M, Nb, K)
    assert g1.ok and g1.variant == 1, g1
    r0 = ops.gemm_mxfp8(ctx, a_op, b_op, y0, cta_group=1)
    assert r0.ok
    assert torch.equal(y.view(torch.int16), y0.view(torch.int16)), f"ordered K7 ({order}) differs from K7 without an order"


def test_ordered_k7_refusals(ctx):
    K, M, Nb = 256, 512, 256
    L = _Records("chunk", M, K)
    buf = torch.zeros(L.n * L.bytes, dtype=torch.uint8, device="cuda")
    bq, bs = _mx_exact_operand(Nb, K, _gen(5))
    a_op, b_op = L.operand(buf), MX.MxOperand.from_tensors(bq, bs)
    y = torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda")
    order = torch.arange(L.n, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="cta_group=2"):
        ops.gemm_mxfp8(ctx, a_op, b_op, y, cta_group=2, a_order=order)
    with pytest.raises(ValueError, match="int32"):
        ops.gemm_mxfp8(ctx, a_op, b_op, y, cta_group=1, a_order=order.long())
    with pytest.raises(ValueError, match="elements"):
        ops.gemm_mxfp8(ctx, a_op, b_op, y, cta_group=1, a_order=order[:1])
    ragged = MX.MxOperand.from_tensors(torch.zeros(200, K, dtype=torch.uint8, device="cuda"),
                                       torch.zeros(200, K // 32, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="whole records"):
        ops.gemm_mxfp8(ctx, ragged, b_op, torch.zeros(200, Nb, dtype=torch.bfloat16, device="cuda"), a_order=order[:1])
    # the native entry point refuses the pair kernel itself, before it launches anything
    lib = NAT.load()
    done = ctx.dev_scratch(32, offset=3 * (256 << 10))
    out, _ = ctx.scratch(64, offset=4096 + 3 * 64)
    rc = lib.rn_k_gemm_mxfp8_ordered(int(torch.cuda.current_stream().cuda_stream), 0, a_op.q_ptr, a_op.s_ptr, a_op.rows_per_rec,
                                     a_op.rec_stride, b_op.q_ptr, b_op.s_ptr, 0, 0, y.data_ptr(), M, Nb, K, out, 2, done, 0,
                                     1000, order.data_ptr())
    assert rc == -22
    # an order that is a permutation gives C unchanged, plain A included
    y1, y2 = torch.zeros_like(y), torch.zeros_like(y)
    assert ops.gemm_mxfp8(ctx, a_op, b_op, y1, cta_group=1).ok
    assert ops.gemm_mxfp8(ctx, a_op, b_op, y2, a_order=order.flip(0).contiguous()).ok
    assert torch.equal(y1.view(torch.int16), y2.view(torch.int16))


# ------------------------------------------------------------------ 3. the all-gather, N simulated ranks
def _plans(ctx, N, chunk, R, timeout_ms=WAIT_MS):
    plans = [AG.RingAllgatherFp8(ctx, R * chunk, chunk, q, N, timeout_ms=timeout_ms) for q in range(N)]
    AG.link_in_process(plans)
    return plans


def _shards(N, n, seed):
    g = _gen(seed)
    return [(torch.randn(n, generator=g) * 4 ** (s % 3)).to(torch.bfloat16) for s in range(N)]


def _gather_checked(ctx, plans, xs_cpu, in_place):
    """One run from poisoned landing buffers; every output and every rank's records against the reference and rank 0."""
    N, chunk, n = len(plans), plans[0].chunk, plans[0].shard
    want, want_rec = ops.ref_allgather_fp8(xs_cpu, chunk)
    outs = [torch.full((N * n,), 7.0, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    if in_place:
        for q in range(N):
            outs[q][q * n:(q + 1) * n].copy_(xs_cpu[q])
        xs = [outs[q][q * n:(q + 1) * n] for q in range(N)]
    else:
        xs = [x.cuda() for x in xs_cpu]
    for p in plans:
        _poison(p.landing, chunk)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = AG.run_in_process(plans, xs, outs)
    finally:
        ctx.engine_stop()
    for r in res:
        assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
        assert r.received == plans[0].n_recv and r.posted == plans[0].n_recv
    for q in range(N):
        assert _bits_equal(outs[q].cpu(), want), f"rank {q} differs from the reference"
        assert torch.equal(outs[q].view(torch.int16), outs[0].view(torch.int16))
        assert torch.equal(plans[q].records().cpu(), want_rec), f"rank {q}'s gathered records"
        _check_arrival_words(plans[q].words_full, plans[q].n_ids)
        assert plans[q].send_qp.counters()["n_err"] == 0
    return res


@pytest.mark.parametrize("chunk", [8192, 1 << 20], ids=["8192", "1M"])
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_allgather_matches_reference(ctx, N, chunk):
    """In place, then into ``out`` with other inputs: every rank bit-identical to ``ref_allgather_fp8``."""
    R = 3 if chunk == 8192 else 1
    plans = _plans(ctx, N, chunk, R)
    _gather_checked(ctx, plans, _shards(N, R * chunk, seed=N * 3), in_place=True)
    _gather_checked(ctx, plans, _shards(N, R * chunk, seed=N * 3 + 1), in_place=False)


def test_allgather_rank_that_never_contributes(ctx):
    """Rank 1 posts its receives but never runs its main stream: the ranks that wait for its shard report TIMEOUT, no
    wait is longer than timeout_ms and the run ends within 2N x timeout_ms.  The next run, with all ranks, is clean."""
    N, chunk, R, tmo = 3, 8192, 2, 300
    plans = _plans(ctx, N, chunk, R, timeout_ms=tmo)
    n = R * chunk
    xs = [x.cuda() for x in _shards(N, n, seed=77)]
    outs = [torch.zeros(N * n, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        t0 = time.monotonic()
        res = AG.run_in_process(plans, xs, outs, skip={1})
        dt = time.monotonic() - t0
    finally:
        ctx.engine_stop()
    for q in (0, 2):
        assert res[q].status == "TIMEOUT", (q, res[q].status, res[q].failed)
    for r in res:
        for l in r.launches:
            assert l.status in ("OK", "TIMEOUT"), (r.rank, l)
    assert dt < 2 * N * tmo / 1000 + 1.0, f"the failed run took {dt:.2f} s"
    for p in plans:
        assert p.send_qp.counters()["n_err"] == 0
    _gather_checked(ctx, plans, _shards(N, n, seed=78), in_place=False)


def test_allgather_rejections(ctx):
    plans = [AG.RingAllgatherFp8(ctx, 8192, 8192, q, 2) for q in range(2)]
    with pytest.raises(ValueError, match="must hold"):
        AG.link_in_process(plans, rq_depth=1)
    with pytest.raises(ValueError, match="SM budget"):
        AG.link_in_process([AG.RingAllgatherFp8(ctx, 8192, 8192, q, 2, grid=57) for q in range(2)])
    AG.link_in_process([AG.RingAllgatherFp8(ctx, 8192, 8192, q, 2, grid=48) for q in range(2)])   # 16 + 2 x 50 fits
    plans = _plans(ctx, 2, 8192, 1)
    x = torch.zeros(8192, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="out"):
        plans[0].run(x, torch.zeros(8192, dtype=torch.bfloat16, device="cuda"))
    b = MX.MxOperand.from_tensors(torch.zeros(128, 128, dtype=torch.uint8, device="cuda"),
                                  torch.zeros(128, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="128 \\* K"):
        plans[0].run_gemm(x.view(64, 128), b, torch.zeros(128, 128, dtype=torch.bfloat16, device="cuda"))


# ------------------------------------------------------------------ 4. the all-gather GEMM
@pytest.mark.parametrize("N", [2, 4, 8])
def test_allgather_gemm(ctx, N):
    """K = 4096, 256 rows per record, Nb = 4096, two records per shard: the gathered records are the reference's, and C
    is bit-identical on every rank and to K7 run on the same records after the gather."""
    K, Nb, rows = 4096, 4096, 512
    chunk = 256 * K
    plans = [AG.RingAllgatherFp8(ctx, rows * K, chunk, q, N, timeout_ms=WAIT_MS) for q in range(N)]
    AG.link_in_process(plans)
    g = _gen(100 + N)
    xs_cpu = [_spread(rows, K, g, 16).to(torch.bfloat16) for _ in range(N)]
    xs = [x.cuda() for x in xs_cpu]
    bq, bs = _mx_exact_operand(Nb, K, g)
    b_op = MX.MxOperand.from_tensors(bq, bs)
    cs = [torch.full((N * rows, Nb), 7.0, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    _, want_rec = ops.ref_allgather_fp8([x.reshape(-1) for x in xs_cpu], chunk)
    for p in plans:
        _poison(p.landing, chunk)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=plans[0].engine_ctas, idle_timeout_ms=WAIT_MS)
    try:
        res = AG.run_gemm_in_process(plans, xs, [b_op] * N, cs)
    finally:
        ctx.engine_stop()
    for r in res:
        assert r.ok, (r.rank, r.status, r.failed, [(l.name, l.status) for l in r.launches])
        assert r.received == plans[0].n_recv and r.posted == plans[0].n_recv
    for q in range(N):
        assert torch.equal(plans[q].records().cpu(), want_rec), f"rank {q}'s gathered records"
        assert bool((plans[q].records() != POISON_Q).any())
        _check_arrival_words(plans[q].words_full, plans[q].n_ids)
    c_ref = torch.zeros_like(cs[0])
    a_op = MX.MxOperand.from_chunk_records(plans[0].records(), N * rows, K, chunk)
    assert ops.gemm_mxfp8(ctx, a_op, b_op, c_ref, cta_group=1).ok
    for q in range(N):
        assert torch.equal(cs[q].view(torch.int16), c_ref.view(torch.int16)), f"rank {q}'s C"
