"""Pulled records on one GPU: ``read_records`` posts RDMA READs from the device and stamps one arrival word per record as
it lands; ``unpack_fp8(ready=)`` and ``gemm_mxfp8(a_ready=)`` consume those words exactly as they consume the words
``recv_consume`` writes for pushed records.

Landing buffers start out as poison (e4m3 448 under scale 2^127, or 0x5A bytes), so a consumer that reads a record before
its word is set, or a record that lands in the wrong place, changes bits.  The rules of test_gpu_receive_fusion.py hold
here too: every kernel that waits on another is resident with it within the 132 SMs of an H100 SXM (each test writes
out its sum), the launch order is consumer, then the GEMM that runs on arrival, then the poster, every wait is bounded
by 5 s or less, nothing allocates or synchronises the device while the engine runs, and the arrival words are the head
of a zeroed tensor whose guard words must still be zero at the end.
"""
import ctypes as C
import time

import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, ops
from rocnrdma_b200.ops import gemm_mx as MX
from rocnrdma_b200.ops import pack as P
from test_gpu_numerics import _gen, _mx_exact_operand, _mx_exact_ref
from test_gpu_receive_fusion import GUARD, _arrival_words, _check_arrival_words, _check_on_arrival, _out_buffer, _Records

pytestmark = pytest.mark.gpu

WAIT_MS = 5000
POISON = 0x5A
CANARY = 0xC5


def _clamped(window, burst, signal_every):
    """The burst and CQ moderation the poster really uses (rn_stream_clamp)."""
    b, s = C.c_uint32(burst), C.c_uint32(signal_every)
    N.load().rn_stream_clamp(window, C.byref(b), C.byref(s))
    return b.value, s.value


def _indices(kind, n):
    """(int32 source indices, number of source records) for a pull of n records."""
    if kind == "none":
        return None, n
    if kind == "reversed":
        return torch.arange(n - 1, -1, -1, dtype=torch.int32), n
    if kind == "subset":                                   # every third of 3n records
        return torch.arange(0, 3 * n, 3, dtype=torch.int32), 3 * n
    g = _gen(n)                                            # repeats: n draws from n // 3 records
    return torch.randint(0, n // 3, (n,), generator=g, dtype=torch.int32), n // 3


def _check_stamps(ready, n, signal_every):
    """Words do not decrease with r, and the records one CQE completed (one signaled WQE every ``signal_every``
    records, and the last) share its stamp."""
    st = ready[:n].tolist()
    assert all(st[r] >= st[r - 1] for r in range(1, n)), f"stamps decrease: {st}"
    for g0 in range(0, n, signal_every):
        grp = st[g0:min(g0 + signal_every, n)]
        assert len(set(grp)) == 1, f"records {g0}..{g0 + len(grp) - 1} share one CQE but not one stamp: {grp}"


# ------------------------------------------------------------------ 1. pull only, software HCA loopback
KNOBS = [(w, s, b) for w in (1, 4, 16) for s in (1, 4) for b in (1, 8)]


@pytest.mark.parametrize("kind", ["none", "reversed", "subset", "repeats"])
@pytest.mark.parametrize("rec", [64, 4096 + 3, 1 << 20], ids=["64B", "4KiB+3", "1MiB"])
def test_pull_lands_and_stamps_every_record(ctx, rec, kind):
    """Every knob combination (window 1, 4, 16; signal_every 1, 4; burst 1, 8, as clamped) pulls n records: landing
    record r equals source record indices[r] byte for byte, the canary behind the last record is untouched, every word
    is set in order, the records of one CQE share a stamp, and the guard words stay zero."""
    n = 24
    idx, n_src = _indices(kind, n)
    src = torch.empty(n_src * rec, dtype=torch.uint8, device="cuda")
    ops.fill_random(src, seed=rec + n_src)
    dst_full = torch.empty(n * rec + 64, dtype=torch.uint8, device="cuda")
    dst = dst_full[:n * rec]
    sm, dm = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    idx_d = idx.cuda() if idx is not None else None
    j = idx.tolist() if idx is not None else list(range(n))
    want = src.view(n_src, rec)[torch.tensor(j, device="cuda")]
    for window, signal_every, burst in KNOBS:
        b, s = _clamped(window, burst, signal_every)
        dst_full[:n * rec].fill_(POISON)
        dst_full[n * rec:].fill_(CANARY)
        full, ready = _arrival_words(n)
        torch.cuda.synchronize()
        # SMs: engine 16 + poster 1 = 17 of 132
        ctx.engine_start(ctas=16, idle_timeout_ms=WAIT_MS)
        try:
            r = ops.read_records(qp, sm, dm, rec, n, indices=idx_d, ready=ready, window=window, burst=burst,
                                 signal_every=signal_every, timeout_ms=WAIT_MS)
        finally:
            ctx.engine_stop()
        knobs = f"window={window} signal_every={signal_every}->{s} burst={burst}->{b}"
        assert r["status"] == "OK" and r["done"] == n, (knobs, r)
        assert r["last_idx"] - r["first_idx"] == n - 1 and r["cons"] == r["last_idx"] + 1, (knobs, r)
        assert torch.equal(dst.view(n, rec), want), knobs
        assert bool((dst_full[n * rec:] == CANARY).all()), f"{knobs}: wrote past the last record"
        _check_arrival_words(full, n)
        _check_stamps(ready, n, s)
    assert qp.counters()["n_err"] == 0


# ------------------------------------------------------------------ 2. errors
@pytest.mark.parametrize("signal_every", [1, 4])
@pytest.mark.parametrize("case", ["index_past_region", "bad_rkey"])
def test_failed_read_stamps_only_what_landed(ctx, case, signal_every):
    """(a) index k points past the remote region; (b) the source key is not registered.  The status is CQE_ERROR and
    the QP is in ERR; the records before the failure have landed and are stamped (with CQ moderation their stamp comes
    from the error completion), the failing one and every later one are unstamped and still hold their poison."""
    rec, n, n_src, k = 4096, 16, 16, 10
    src = torch.empty(n_src * rec, dtype=torch.uint8, device="cuda")
    ops.fill_random(src, seed=7)
    dst = torch.full((n * rec,), POISON, dtype=torch.uint8, device="cuda")
    sm, dm = ctx.reg_mr(src), ctx.reg_mr(dst)
    idx = torch.arange(n, dtype=torch.int32)
    if case == "bad_rkey":
        sm = rn.api.MemoryRegion(ctx, sm.addr, sm.length, 0x5555, sm.access)
        k = 0
    else:
        idx[k] = n_src + 5
    idx_d = idx.cuda()
    full, ready = _arrival_words(n)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    # SMs: engine 8 + poster 1 = 9 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        r = ops.read_records(qp, sm, dm, rec, n, indices=idx_d, ready=ready, window=4, signal_every=signal_every,
                             timeout_ms=WAIT_MS)
    finally:
        ctx.engine_stop()
    assert r["status"] == "CQE_ERROR" and r["done"] == k, r
    assert qp.state == "ERR"
    assert torch.equal(dst[:k * rec], src[:k * rec]), "a record before the failure did not land"
    assert bool((dst[k * rec:] == POISON).all()), "the failing record or a later one changed the landing buffer"
    st = full.tolist()
    assert all(st[r_] != 0 for r_ in range(k)), f"records before the failure are unstamped: {st[:k]}"
    assert all(w == 0 for w in st[k:]), f"the failing record or a later one (or a guard word) was stamped: {st[k:]}"


# ------------------------------------------------------------------ 3. K5 gated on arrival words, no engine
CHUNK = 16384


def _k3_source(n_chunks, seed):
    """(bf16 payload, its K3 chunk records) on the GPU."""
    g = _gen(seed)
    x = (torch.randn(n_chunks * CHUNK, generator=g) * 2.0 ** torch.randint(-8, 9, (n_chunks * CHUNK // 32, 1), generator=g)
         .expand(-1, 32).reshape(-1)).to(torch.bfloat16).cuda()
    return x, P.ref_pack_fp8(x, CHUNK)


def _poison_records(buf, n_chunks):
    r = buf.view(n_chunks, -1)
    r.fill_(0xFE)
    r[:, :CHUNK] = 0x7E


def test_unpack_waits_for_each_arrival_word(ctx):
    """``unpack_fp8(ready=)`` is launched on poisoned records.  Another stream puts records 1..n-1 in place and sets their
    words, out of the order any poster sets them; 100 ms later K5's end-time word is still 0.  Then record 0 lands and
    its word is set, and the output equals ref_unpack_fp8 bit for bit.  The workers that read record 0 read record 4 in
    the same step, whose word is set long before: each of them must wait for every record it reads."""
    n_chunks = 8
    rec = P.record_bytes(CHUNK)
    _, recs = _k3_source(n_chunks, 11)
    want = P.ref_unpack_fp8(recs, n_chunks * CHUNK, CHUNK)
    land = torch.empty_like(recs)
    out = torch.full((n_chunks * CHUNK,), float("nan"), dtype=torch.bfloat16, device="cuda")
    full, ready = _arrival_words(n_chunks)
    s_set, s_k5 = ctx.streams(2)

    def set_rest():
        land[rec:].copy_(recs[rec:])
        ready[1:].fill_(1)

    def set_first():
        land[:rec].copy_(recs[:rec])
        ready[:1].fill_(1)

    # The setter runs once before K5 exists: a kernel's first load waits for every resident kernel (DESIGN.md 3.2), and
    # torch picks its fill kernel by the alignment of the slice, so only these very calls load what the setter needs.
    with torch.cuda.stream(s_set):
        set_rest()
        set_first()
    torch.cuda.synchronize()
    _poison_records(land, n_chunks)
    full.zero_()
    torch.cuda.synchronize()
    # SMs: K5 8 CTAs; the setter's copies and fills wait on nothing
    uview, _ = P.unpack_fp8(ctx, land, out, CHUNK, ready=ready, grid=8, timeout_ms=WAIT_MS, sync=False, stream=s_k5)
    with torch.cuda.stream(s_set):
        set_rest()
    s_set.synchronize()
    time.sleep(0.1)
    early = list((C.c_int64 * 8).from_buffer(uview))
    with torch.cuda.stream(s_set):
        set_first()
    s_k5.synchronize()
    s_set.synchronize()
    assert early[2] == 0, f"K5 finished (status word {early[0]}) before record 0 was in place"
    u = P.parse_unpack(uview)
    assert u["status"] == "OK" and u["records_seen"] == n_chunks, u
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    assert bool((full[n_chunks:] == 0).all())


def test_unpack_times_out_on_a_word_never_set(ctx):
    n_chunks = 4
    _, recs = _k3_source(n_chunks, 12)
    out = torch.zeros(n_chunks * CHUNK, dtype=torch.bfloat16, device="cuda")
    full, ready = _arrival_words(n_chunks)
    ready[:n_chunks - 1] = 1                             # the last record never arrives
    torch.cuda.synchronize()
    t0 = time.monotonic()
    u = P.unpack_fp8(ctx, recs, out, CHUNK, ready=ready, grid=4, timeout_ms=300)
    dt = time.monotonic() - t0
    assert u["status"] == "TIMEOUT", u
    assert dt < 3.0, f"the timeout took {dt:.2f} s"
    # the scratch the kernel cleans up after itself is clean: the next call runs normally
    ready[n_chunks - 1] = 1
    u = P.unpack_fp8(ctx, recs, out, CHUNK, ready=ready, grid=4, timeout_ms=WAIT_MS)
    assert u["status"] == "OK" and u["records_seen"] == n_chunks, u
    assert torch.equal(out, P.ref_unpack_fp8(recs, n_chunks * CHUNK, CHUNK))


# ------------------------------------------------------------------ 4. pull -> K5 on arrival
@pytest.mark.parametrize("window,signal_every", [(16, 1), (8, 4)])
def test_pull_then_unpack_on_arrival(ctx, window, signal_every):
    """K3 records of seeded bf16, pulled through a permutation into a poisoned landing buffer; K5, launched first,
    unpacks each record once its word is set.  The output equals ref_unpack_fp8 of the gathered records bit for bit."""
    n_chunks = 12
    rec = P.record_bytes(CHUNK)
    _, recs = _k3_source(n_chunks, 21 + window)
    perm = torch.randperm(n_chunks, generator=_gen(3 + window)).to(torch.int32)
    gathered = recs.view(n_chunks, rec)[perm.long().cuda()].reshape(-1)
    want = P.ref_unpack_fp8(gathered, n_chunks * CHUNK, CHUNK)
    land = torch.empty_like(recs)
    _poison_records(land, n_chunks)
    out = torch.full((n_chunks * CHUNK,), float("nan"), dtype=torch.bfloat16, device="cuda")
    full, ready = _arrival_words(n_chunks)
    sm, lm = ctx.reg_mr(recs), ctx.reg_mr(land)
    qp = ctx.loopback_qp(depth=64)
    perm_d = perm.cuda()
    s_pull, s_k5 = ctx.streams(2)
    torch.cuda.synchronize()
    # SMs: engine 16 + K5 8 + poster 1 = 25 of 132
    ctx.engine_start(ctas=16, idle_timeout_ms=WAIT_MS)
    try:
        uview, _ = P.unpack_fp8(ctx, land, out, CHUNK, ready=ready, grid=8, timeout_ms=WAIT_MS, sync=False, stream=s_k5)
        pview, _ = ops.read_records(qp, sm, lm, rec, n_chunks, indices=perm_d, ready=ready, window=window,
                                    signal_every=signal_every, timeout_ms=WAIT_MS, sync=False, stream=s_pull)
        s_pull.synchronize()
        s_k5.synchronize()
    finally:
        ctx.engine_stop()
    r = ops.parse_read_records(pview)
    assert r["status"] == "OK" and r["done"] == n_chunks, r
    u = P.parse_unpack(uview)
    assert u["status"] == "OK" and u["records_seen"] == n_chunks, u
    _check_arrival_words(full, n_chunks)
    assert torch.equal(land, gathered)
    bad = (out.view(torch.int16) != want.view(torch.int16)).nonzero().flatten()
    assert bad.numel() == 0, f"{bad.numel()} unpacked values differ, first at {bad[0].item()}"


# ------------------------------------------------------------------ 5. pull -> K7 on arrival
PULL_GEMM_CASES = [("panel", 512), ("chunk", 768)]


@pytest.mark.parametrize("gather", [False, True], ids=["whole", "gathered"])
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("kind,M", PULL_GEMM_CASES, ids=[k for k, _ in PULL_GEMM_CASES])
def test_pull_then_gemm_on_arrival(ctx, kind, M, cta_group, gather):
    """K4 panel records or K3 chunk records of an exact MX operand, pulled whole or gathered in reverse order into a
    poisoned landing buffer; ``gemm_mxfp8(a_ready=)``, launched before the pull, multiplies them as they land.  The
    result equals the same call after arrival bit for bit, and that equals the exact product of the gathered operand."""
    K, N_ = 256, 264
    L = _Records(kind, M, K)
    g = _gen(M + 10 * cta_group + gather)
    aq, as_ = _mx_exact_operand(M, K, g)
    bq, bs = _mx_exact_operand(N_, K, g)
    src = L.build(aq, as_)
    idx = torch.arange(L.n - 1, -1, -1, dtype=torch.int32) if gather else None
    gathered = src.view(L.n, L.bytes)[idx.long().cuda()].reshape(-1) if gather else src
    exact = _mx_exact_ref(*L.parts(gathered), bq, bs)
    land = torch.empty_like(src)
    L.poison(land)
    pad, y = _out_buffer(M, N_)
    full, ready = _arrival_words(L.n)
    sm, lm = ctx.reg_mr(src), ctx.reg_mr(land)
    qp = ctx.loopback_qp(depth=64)
    idx_d = idx.cuda() if gather else None
    a_op, b_op = L.operand(land), MX.MxOperand.from_tensors(bq, bs)
    s_pull, s_mm = ctx.streams(2)
    torch.cuda.synchronize()
    # SMs: engine 8 + GEMM 64 + poster 1 = 73 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=64, cta_group=cta_group, a_ready=ready, timeout_ms=WAIT_MS,
                                  sync=False, stream=s_mm)
        pview, _ = ops.read_records(qp, sm, lm, L.bytes, L.n, indices=idx_d, ready=ready, window=4, timeout_ms=WAIT_MS,
                                    sync=False, stream=s_pull)
        s_pull.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    r = ops.parse_read_records(pview)
    assert r["status"] == "OK" and r["done"] == L.n, r
    _check_arrival_words(full, L.n)
    assert torch.equal(land, gathered)
    _check_on_arrival(ctx, y, gview, a_op, b_op, cta_group, exact=exact)
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


def test_pull_then_gemm_on_arrival_many_tiles_per_cta(ctx):
    """The benchmark's record size: K4 panel records at K = 4096 (528 KiB each), 16 of them, gathered in reverse, and a
    GEMM of only 8 single CTAs, so every CTA works through 8 tiles and waits on several records.  Scale bytes of 127
    keep the fp32 accumulation exact, so the on-arrival result equals the exact product of the gathered operand."""
    M, K, N_ = 2048, 4096, 512
    L = _Records("panel", M, K)
    g = _gen(4096)
    aq, as_ = _mx_exact_operand(M, K, g, scale_lo=127, scale_hi=127)
    bq, bs = _mx_exact_operand(N_, K, g, scale_lo=127, scale_hi=127)
    src = L.build(aq, as_)
    idx = torch.arange(L.n - 1, -1, -1, dtype=torch.int32)
    gathered = src.view(L.n, L.bytes)[idx.long().cuda()].reshape(-1)
    exact = _mx_exact_ref(*L.parts(gathered), bq, bs)
    land = torch.empty_like(src)
    L.poison(land)
    pad, y = _out_buffer(M, N_)
    full, ready = _arrival_words(L.n)
    sm, lm = ctx.reg_mr(src), ctx.reg_mr(land)
    qp = ctx.loopback_qp(depth=64)
    idx_d = idx.cuda()
    a_op, b_op = L.operand(land), MX.MxOperand.from_tensors(bq, bs)
    s_pull, s_mm = ctx.streams(2)
    torch.cuda.synchronize()
    # SMs: engine 16 + GEMM 8 + poster 1 = 25 of 132
    ctx.engine_start(ctas=16, idle_timeout_ms=WAIT_MS)
    try:
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=8, cta_group=1, a_ready=ready, timeout_ms=WAIT_MS, sync=False,
                                  stream=s_mm)
        pview, _ = ops.read_records(qp, sm, lm, L.bytes, L.n, indices=idx_d, ready=ready, window=16, timeout_ms=WAIT_MS,
                                    sync=False, stream=s_pull)
        s_pull.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    r = ops.parse_read_records(pview)
    assert r["status"] == "OK" and r["done"] == L.n, r
    _check_arrival_words(full, L.n)
    assert torch.equal(land, gathered)
    _check_on_arrival(ctx, y, gview, a_op, b_op, 1, exact=exact)
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


# ------------------------------------------------------------------ 6. the verbs wire, adopted mlx5dv queues
def test_pull_then_unpack_on_the_mock_connectx():
    """read_records posts into the mock ConnectX's send queue mapped to the GPU and polls its CQ; K5 unpacks on the
    words.  Exact end to end, no error completion and no doorbell out of order."""
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        n_chunks = 8
        rec = P.record_bytes(CHUNK)
        _, recs = _k3_source(n_chunks, 31)
        perm = torch.randperm(n_chunks, generator=_gen(31)).to(torch.int32)
        gathered = recs.view(n_chunks, rec)[perm.long().cuda()].reshape(-1)
        want = P.ref_unpack_fp8(gathered, n_chunks * CHUNK, CHUNK)
        land = torch.empty_like(recs)
        _poison_records(land, n_chunks)
        out = torch.full((n_chunks * CHUNK,), float("nan"), dtype=torch.bfloat16, device="cuda")
        full, ready = _arrival_words(n_chunks)
        sm, lm = vctx.reg_mr(recs), vctx.reg_mr(land)
        qp = vctx.loopback_qp(depth=64)
        assert qp.on_gpu
        perm_d = perm.cuda()
        s_pull, s_k5 = vctx.streams(2)
        torch.cuda.synchronize()
        # SMs: K5 8 + poster 1 = 9 of 132 (the NIC is a host thread)
        uview, _ = P.unpack_fp8(vctx, land, out, CHUNK, ready=ready, grid=8, timeout_ms=WAIT_MS, sync=False, stream=s_k5)
        pview, _ = ops.read_records(qp, sm, lm, rec, n_chunks, indices=perm_d, ready=ready, window=4, timeout_ms=WAIT_MS,
                                    sync=False, stream=s_pull)
        s_pull.synchronize()
        s_k5.synchronize()
        r = ops.parse_read_records(pview)
        assert r["status"] == "OK" and r["done"] == n_chunks, r
        u = P.parse_unpack(uview)
        assert u["status"] == "OK" and u["records_seen"] == n_chunks, u
        _check_arrival_words(full, n_chunks)
        assert torch.equal(land, gathered)
        assert torch.equal(out.view(torch.int16), want.view(torch.int16))
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_db_order_violations"] == 0, c
    finally:
        vctx.close()


# ------------------------------------------------------------------ 7. host-side rejections
def test_pull_host_side_rejections(ctx):
    src = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    sm, dm = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=16)
    words = torch.zeros(16 + GUARD, dtype=torch.int64, device="cuda")
    idx = torch.zeros(16, dtype=torch.int32, device="cuda")
    bad = [
        (dict(rec_bytes=0, n=4), "rec_bytes"),
        (dict(rec_bytes=ctx.max_msg_bytes + 1, n=1), "rec_bytes"),
        (dict(rec_bytes=4096, n=17), "do not fit"),
        (dict(rec_bytes=4096, n=4, dst_off=(1 << 16) - 4096 * 3), "do not fit"),
        (dict(rec_bytes=64, n=4, ready=words.to(torch.int32)), "ready"),
        (dict(rec_bytes=64, n=4, ready=words.cpu()), "ready"),
        (dict(rec_bytes=64, n=4, ready=words[:3]), "ready"),
        (dict(rec_bytes=64, n=4, indices=idx.to(torch.int64)), "indices"),
        (dict(rec_bytes=64, n=4, indices=idx.cpu()), "indices"),
        (dict(rec_bytes=64, n=4, indices=idx[:3]), "indices"),
    ]
    for kw, what in bad:
        with pytest.raises(ValueError, match=what):
            ops.read_records(qp, sm, dm, **kw)
    # K5: a receive CQ or arrival words, not both; one int64 word per record
    n_chunks = 2
    recs = torch.zeros(n_chunks * P.record_bytes(CHUNK), dtype=torch.uint8, device="cuda")
    out = torch.zeros(n_chunks * CHUNK, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError, match="not both"):
        P.unpack_fp8(ctx, recs, out, CHUNK, qp=qp, ready=words)
    with pytest.raises(ValueError, match="ready"):
        P.unpack_fp8(ctx, recs, out, CHUNK, ready=words[:1])
    with pytest.raises(ValueError, match="ready"):
        P.unpack_fp8(ctx, recs, out, CHUNK, ready=words.to(torch.int32))
    assert int(words.count_nonzero()) == 0, "a rejected call launched something"
