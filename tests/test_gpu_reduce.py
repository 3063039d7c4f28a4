"""``reduce_fp8`` on one GPU: the sum of several sources of K3 records (plus a bf16 addend) as they land, re-packed and
forwarded from the same kernel, against ``ref_reduce_fp8`` bit for bit.

The one allowed difference is a NaN's sign and payload: the hardware conversions produce one canonical NaN where the
reference keeps what the input had, so NaN must sit at the same positions and every other value must match exactly.

The rules of test_gpu_receive_fusion.py hold here too: every kernel that waits on another is launched first and is
resident with it within the 132 SMs of an H100 SXM (each test writes out its sum), every wait is bounded by 5 s or less,
nothing allocates or synchronises the device while the engine runs, the arrival words are the head of a zeroed tensor
whose guard words must still be zero at the end, and landing buffers start as poison (e4m3 448 under scale 2^127, codes
0x7E under scale byte 0xFE), so a record read before it has landed changes the result.
"""
import time

import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from test_gpu_numerics import _bits_equal, _gen, _records_equal_up_to_nan_sign
from test_gpu_receive_fusion import GUARD, _arrival_words, _check_arrival_words

pytestmark = pytest.mark.gpu

WAIT_MS = 5000
POISON_Q, POISON_S = 0x7E, 0xFE
CANARY = 0xC5


def _source_records(n_src, n, chunk, seed, edges=False):
    """Source-major K3 records (CPU uint8) of seeded bf16 data spread over 2^+-20.  With ``edges`` the first record of
    each source also holds NaN codes, scale bytes 0x00 and 0xFF, fp32 subnormals (scale byte 0x00 / 0x01 under small
    codes) and, in sources 0 and 1, a block whose finite sum overflows (1.5 * 2^127 twice)."""
    rec = P.record_bytes(chunk)
    out = []
    for s in range(n_src):
        g = _gen(seed * 16 + s)
        x = (torch.randn(n, generator=g) * torch.exp2(torch.randint(-20, 21, (n // 32,), generator=g).float())
             .repeat_interleave(32)).to(torch.bfloat16)
        r = P.ref_pack_fp8(x, chunk).view(n // chunk, rec)
        if edges:
            q, sc = r[0, :chunk], r[0, chunk:chunk + chunk // 32]
            q[5 + s] = 0x7F                                    # NaN code
            q[32 * 2 + s] = 0xFF                               # -NaN code
            sc[3], sc[4] = 0x00, 0x01                          # fp32 subnormals (2^-127, 2^-126 times small codes)
            q[32 * 3:32 * 5] = torch.randint(0, 0x30, (64,), generator=g).to(torch.uint8)
            sc[6] = 0xFF                                       # Inf (nonzero codes) and NaN (zero codes)
            q[32 * 6 + 1] = 0
            if s < 2:
                sc[8] = 254
                q[32 * 8] = 0x3C                               # 1.5 * 2^127 in both: the fp32 sum overflows
                q[32 * 8 + 1] = 0x30 if s == 0 else 0xB0       # 0.5 * 2^127 and its negation: a finite neighbour of 0
        out.append(r.reshape(-1))
    return torch.cat(out)


def _bf16_equal_up_to_nan(got, want):
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), "NaN at different positions"
    assert _bits_equal(got[~nan], want[~nan]), f"{int((got[~nan].view(torch.int16) != want[~nan].view(torch.int16)).sum())} values differ"


def _poison(buf, chunk):
    r = buf.view(-1, P.record_bytes(chunk))
    r.fill_(POISON_S)
    r[:, :chunk] = POISON_Q


# ------------------------------------------------------------------ 1. numerics, no waits
CHUNKS = {8192: 5, 16384: 3, 1 << 20: 2}                # chunk -> records per source
SOURCES = [1, 2, 3, 4, 5, 7, 8]                          # every variant at full and partial width (test_reduce_references.py)


@pytest.mark.parametrize("outputs", ["bf16", "records", "both"])
@pytest.mark.parametrize("local", [False, True], ids=["no_local", "local"])
@pytest.mark.parametrize("n_src", SOURCES)
@pytest.mark.parametrize("chunk", list(CHUNKS), ids=[str(c) for c in CHUNKS])
def test_reduce_matches_reference(ctx, chunk, n_src, local, outputs):
    """Every output at grids 1, 8 and the default, bit for bit (NaN up to its sign and payload), with canaries behind
    the bf16 output and behind the last output record.  Grid 1 walks every tile from one CTA, grid 8 many steps each."""
    n = chunk * CHUNKS[chunk]
    nb = P.staging_bytes(n, chunk)
    recs_cpu = _source_records(n_src, n, chunk, seed=chunk + 10 * n_src + local, edges=True)
    loc_cpu = (torch.randn(n, generator=_gen(n_src + 100)) * 64).to(torch.bfloat16) if local else None
    want_y, want_r = P.ref_reduce_fp8(recs_cpu, n_src, n, chunk, local=loc_cpu)
    recs = recs_cpu.cuda()
    loc = loc_cpu.cuda() if local else None
    ybuf = torch.empty(n + 64, dtype=torch.bfloat16, device="cuda")
    rbuf = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    mr = ctx.reg_mr(rbuf[:nb]) if outputs != "bf16" else None
    for grid in (1, 8, 0):
        ybuf.fill_(7.0)
        rbuf.fill_(CANARY)
        r = ops.reduce_fp8(ctx, recs, n_src, n, chunk, local=loc, out=ybuf[:n] if outputs != "records" else None,
                           out_mr=mr, grid=grid)
        assert r.ok and r.records_reduced == n // chunk and r.records_posted == 0, (grid, r)
        if outputs != "records":
            _bf16_equal_up_to_nan(ybuf[:n].cpu(), want_y)
        if outputs != "bf16":
            _records_equal_up_to_nan_sign(rbuf[:nb].cpu(), want_r, chunk)
        assert bool((ybuf[n:] == 7.0).all()), f"grid {grid}: stored past the bf16 output"
        assert bool((rbuf[nb:] == CANARY).all()), f"grid {grid}: stored past the last output record"
        if outputs == "records":
            assert bool((ybuf == 7.0).all())


def test_reduce_edge_payload_covers_every_case(ctx):
    """The payload of the numerics cases does hold what they claim: NaN, +-Inf, fp32 subnormals, scale bytes 0x00 and
    0xFF in the inputs, and a finite sum that overflows (scale byte 254 in the records of the sum)."""
    chunk, n = 8192, 8192
    recs = _source_records(2, n, chunk, seed=1, edges=True)
    y, out = P.ref_reduce_fp8(recs, 2, n, chunk)
    d = P._decode_records(recs, 2, n, chunk)
    assert bool(torch.isnan(d).any()) and bool(torch.isinf(d).any())
    sub = (d != 0) & (d.abs() < torch.finfo(torch.float32).tiny)
    assert bool(sub.any()), "no fp32 subnormal among the decoded inputs"
    assert bool(torch.isfinite(d[:, 256]).all()) and torch.isinf(y[256].float()), "no finite sum that overflows"
    assert out[chunk + 8].item() == 254 and (out[256].item() & 0x7F) == 0x7F and out[257].item() in (0x00, 0x80)
    sc = recs.view(2, -1)[:, chunk:chunk + chunk // 32]
    assert bool((sc == 0).any()) and bool((sc == 0xFF).any())


# ------------------------------------------------------------------ 2. each wait is honoured
def test_reduce_waits_for_every_word_it_reads(ctx):
    """P = 3, launched on poisoned records.  Another stream lands and stamps every record except (source 2, record 0),
    in reverse order; 100 ms later the end-time word is still 0.  Then that record lands and is stamped, and the result
    is exact.  With P = 3 a step holds two tiles ``grid`` apart: the step that reads record 0 also reads record 4, whose
    words are set long before, so each worker must wait on every word it reads."""
    chunk, n_rec, n_src, grid = 16384, 8, 3, 8
    n = chunk * n_rec
    rec = P.record_bytes(chunk)
    recs_cpu = _source_records(n_src, n, chunk, seed=2)
    want_y, want_r = P.ref_reduce_fp8(recs_cpu, n_src, n, chunk)
    recs = recs_cpu.cuda()
    land = torch.empty_like(recs)
    y = torch.full((n,), float("nan"), dtype=torch.bfloat16, device="cuda")
    stg = torch.zeros(P.staging_bytes(n, chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(stg)
    full, ready = _arrival_words(n_src * n_rec)
    last = 2 * n_rec + 0
    order = [i for i in reversed(range(n_src * n_rec)) if i != last]
    s_set, s_red = ctx.streams(2)

    def land_one(i):
        land[i * rec:(i + 1) * rec].copy_(recs[i * rec:(i + 1) * rec])
        ready[i:i + 1].fill_(1)

    # The setter runs once before the reduce exists: a kernel's first load waits for every resident kernel (DESIGN.md
    # 3.2), so only these very calls load what the setter needs.
    with torch.cuda.stream(s_set):
        for i in order + [last]:
            land_one(i)
    torch.cuda.synchronize()
    _poison(land, chunk)
    full.zero_()
    torch.cuda.synchronize()
    # SMs: the reduce 8 CTAs; the setter's copies and fills wait on nothing
    view, _ = ops.reduce_fp8(ctx, land, n_src, n, chunk, out=y, out_mr=smr, ready=ready, grid=grid, timeout_ms=WAIT_MS,
                             sync=False, stream=s_red)
    with torch.cuda.stream(s_set):
        for i in order:
            land_one(i)
    s_set.synchronize()
    time.sleep(0.1)
    early = ops.parse_reduce(view)
    with torch.cuda.stream(s_set):
        land_one(last)
    s_red.synchronize()
    s_set.synchronize()
    assert early.t_end_ns == 0, f"the reduce finished ({early.status}) before record (2, 0) was in place"
    r = ops.parse_reduce(view)
    assert r.ok and r.records_reduced == n_rec, r
    _check_arrival_words(full, n_src * n_rec)
    _bf16_equal_up_to_nan(y.cpu(), want_y)
    assert torch.equal(stg.cpu(), want_r)


# ------------------------------------------------------------------ 3. timeout
def test_reduce_times_out_and_never_posts_an_unseen_record(ctx):
    """One word, (source 1, record 2), is never set, with posting on.  The status is TIMEOUT within the bound; record 2
    is never posted (its destination bytes are still poison and no downstream word is set); no record is posted twice
    and ``records_posted`` equals the records that landed downstream; the flush completes."""
    chunk, n_rec, n_src = 8192, 4, 2
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    rec = P.record_bytes(chunk)
    recs = _source_records(n_src, n, chunk, seed=3).cuda()
    _, want_r = P.ref_reduce_fp8(recs.cpu(), n_src, n, chunk)
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nb, dtype=torch.uint8, device="cuda")
    _poison(dst, chunk)
    smr, dmr = ctx.reg_mr(stg), ctx.reg_mr(dst)
    full, ready = _arrival_words(n_src * n_rec)
    ready.fill_(1)
    ready[1 * n_rec + 2] = 0
    full2, ready2 = _arrival_words(n_rec)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(n_rec):
        qp.post_recv(dmr, 0)
    s_recv, s_red = ctx.streams(2)
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + reduce 4 = 13 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, n_rec - 1, n_rec, ready2, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        t0 = time.monotonic()
        r = ops.reduce_fp8(ctx, recs, n_src, n, chunk, out_mr=smr, qp=qp, dst_mr=dmr, with_imm=True, ready=ready, grid=4,
                           timeout_ms=300, stream=s_red)
        dt = time.monotonic() - t0
        s_recv.synchronize()
    finally:
        ctx.engine_stop()
    assert r.status == "TIMEOUT", r
    assert dt < 3.0, f"the timeout took {dt:.2f} s"
    assert r.records_reduced == n_rec - 1 and r.records_posted == n_rec - 1, r
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == n_rec - 1, cons
    st = full2.tolist()
    assert st[2] == 0 and all(st[i] != 0 for i in (0, 1, 3)), f"downstream words: {st[:n_rec]}"
    assert all(w == 0 for w in st[n_rec:])
    d, w = dst.view(n_rec, rec), want_r.view(n_rec, rec)
    for i in (0, 1, 3):
        assert torch.equal(d[i].cpu(), w[i]), f"record {i} at the destination"
    assert bool((d[2, :chunk] == POISON_Q).all()) and bool((d[2, chunk:] == POISON_S).all()), "record 2 was posted"
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == (n_rec - 1) + 1, c          # three records and the flush, each once
    # the scratch the kernel cleans up after itself is clean: the next call runs normally
    ready[1 * n_rec + 2] = 1
    r2 = ops.reduce_fp8(ctx, recs, n_src, n, chunk, out_mr=smr, ready=ready, grid=4, timeout_ms=WAIT_MS)
    assert r2.ok and r2.records_reduced == n_rec, r2
    assert torch.equal(stg.cpu(), want_r)


# ------------------------------------------------------------------ 4. a two-hop ring on the software HCA, pushed
@pytest.mark.parametrize("signal_every", [1, 4])
def test_two_hop_ring_pushed(ctx, signal_every):
    """K3 packs x0 and WRITE_IMMs it to hop 1; ``recv_consume`` stamps hop 1's words; ``reduce_fp8(local=x1)`` re-packs
    the sum and WRITE_IMMs it to hop 2; a second ``recv_consume`` stamps; ``reduce_fp8(local=x2, out=y)`` finishes.
    Distinct loopback QPs, streams and scratch slots; consumers are launched first, then K3.  y and the records that
    landed at hop 2 equal the reference chain bit for bit."""
    chunk, n_rec = 16384, 6
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    g = _gen(40 + signal_every)
    xs = [(torch.randn(n, generator=g) * 8).to(torch.bfloat16) for _ in range(3)]
    r0 = P.ref_pack_fp8(xs[0], chunk)                                  # what lands at hop 1
    _, r1 = P.ref_reduce_fp8(r0, 1, n, chunk, local=xs[1])            # what hop 1 forwards, and lands at hop 2
    want_y, _ = P.ref_reduce_fp8(r1, 1, n, chunk, local=xs[2])
    x0, x1, x2 = (x.cuda() for x in xs)
    stg0, stg1 = (torch.zeros(nb, dtype=torch.uint8, device="cuda") for _ in range(2))
    land1, land2 = (torch.empty(nb + 256, dtype=torch.uint8, device="cuda") for _ in range(2))
    for land in (land1, land2):
        _poison(land[:nb], chunk)
        land[nb:].fill_(CANARY)
    ybuf = torch.full((n + 64,), 7.0, dtype=torch.bfloat16, device="cuda")
    m0, m1 = ctx.reg_mr(stg0), ctx.reg_mr(stg1)
    l1, l2 = ctx.reg_mr(land1[:nb]), ctx.reg_mr(land2[:nb])
    full1, ready1 = _arrival_words(n_rec)
    full2, ready2 = _arrival_words(n_rec)
    qp1, qp2 = ctx.loopback_qp(depth=64), ctx.loopback_qp(depth=64)
    for _ in range(n_rec):
        qp1.post_recv(l1, 0)
        qp2.post_recv(l2, 0)
    _, s_c1, s_c2, s_a, s_b = ctx.streams(5)       # K3 runs on ctx.stream
    torch.cuda.synchronize()
    # SMs: engine 8 + consumers 2 + reduce 8 + reduce 8 + K3 16 = 42 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        c1, _ = ops.recv_consume(qp1, n_rec, n_rec, ready1, timeout_ms=WAIT_MS, sync=False, stream=s_c1, scratch_off=8192)
        c2, _ = ops.recv_consume(qp2, n_rec, n_rec, ready2, timeout_ms=WAIT_MS, sync=False, stream=s_c2, scratch_off=8256)
        va, _ = ops.reduce_fp8(ctx, land1, 1, n, chunk, local=x1, out_mr=m1, qp=qp2, dst_mr=l2, with_imm=True,
                               signal_every=signal_every, ready=ready1, grid=8, timeout_ms=WAIT_MS, sync=False, stream=s_a,
                               scratch_slot=4)
        vb, _ = ops.reduce_fp8(ctx, land2, 1, n, chunk, local=x2, out=ybuf[:n], ready=ready2, grid=8, timeout_ms=WAIT_MS,
                               sync=False, stream=s_b, scratch_slot=5)
        pr = ops.pack_fp8_write(ctx, x0, m0, qp=qp1, dst_mr=l1, chunk_elems=chunk, with_imm=True, signal_every=signal_every,
                                grid=16, timeout_ms=WAIT_MS)
        for s in (s_c1, s_c2, s_a, s_b):
            s.synchronize()
    finally:
        ctx.engine_stop()
    assert pr.ok and pr.wqes == n_rec, pr
    ra, rb = ops.parse_reduce(va), ops.parse_reduce(vb)
    assert ra.ok and ra.records_reduced == n_rec and ra.records_posted == n_rec, ra
    assert ra.t_first_post_ns >= ra.t_start_ns > 0
    assert rb.ok and rb.records_reduced == n_rec and rb.records_posted == 0, rb
    for cv in (c1, c2):
        cons = ops.parse_recv(cv)
        assert cons["status"] == "OK" and cons["seen"] == n_rec, cons
    _check_arrival_words(full1, n_rec)
    _check_arrival_words(full2, n_rec)
    for q in (qp1, qp2):
        c = q.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == n_rec + 1, c
    assert torch.equal(land1[:nb].cpu(), r0) and torch.equal(stg1.cpu(), r1)
    assert torch.equal(land2[:nb].cpu(), r1), "the records that landed at hop 2 differ from the reference chain"
    assert bool((land1[nb:] == CANARY).all()) and bool((land2[nb:] == CANARY).all())
    assert _bits_equal(ybuf[:n].cpu(), want_y)
    assert bool((ybuf[n:] == 7.0).all())


# ------------------------------------------------------------------ 5. pull, P = 4
def test_pull_four_sources_and_reduce_on_arrival(ctx):
    """Four ``read_records`` posters on four loopback QPs fill the four source slices and their word slices, source 1
    through a permutation; the reduce, launched first, sums each record once all four of its words are set."""
    chunk, n_rec, n_src = 16384, 6, 4
    n = chunk * n_rec
    rec = P.record_bytes(chunk)
    nb = n_rec * rec
    srcs_cpu = _source_records(n_src, n, chunk, seed=5).view(n_src, nb)
    perm = torch.randperm(n_rec, generator=_gen(55)).to(torch.int32)
    landed = srcs_cpu.clone()
    landed[1] = srcs_cpu[1].view(n_rec, rec)[perm.long()].reshape(-1)
    loc_cpu = (torch.randn(n, generator=_gen(56)) * 4).to(torch.bfloat16)
    want_y, want_r = P.ref_reduce_fp8(landed.reshape(-1), n_src, n, chunk, local=loc_cpu)
    srcs = [srcs_cpu[s].cuda() for s in range(n_src)]
    loc = loc_cpu.cuda()
    land = torch.empty(n_src * nb, dtype=torch.uint8, device="cuda")
    _poison(land, chunk)
    y = torch.full((n,), float("nan"), dtype=torch.bfloat16, device="cuda")
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    smr, lm = ctx.reg_mr(stg), ctx.reg_mr(land)
    src_mrs = [ctx.reg_mr(t) for t in srcs]
    full, ready = _arrival_words(n_src * n_rec)
    qps = [ctx.loopback_qp(depth=64) for _ in range(n_src)]
    perm_d = perm.cuda()
    streams = ctx.streams(n_src + 1)
    torch.cuda.synchronize()
    # SMs: engine 16 + reduce 8 + posters 4 = 28 of 132
    ctx.engine_start(ctas=16, idle_timeout_ms=WAIT_MS)
    try:
        rv, _ = ops.reduce_fp8(ctx, land, n_src, n, chunk, local=loc, out=y, out_mr=smr, ready=ready, grid=8,
                               timeout_ms=WAIT_MS, sync=False, stream=streams[0])
        pviews = []
        for s in range(n_src):
            pv, _ = ops.read_records(qps[s], src_mrs[s], lm, rec, n_rec, indices=perm_d if s == 1 else None, dst_off=s * nb,
                                     ready=ready[s * n_rec:(s + 1) * n_rec], window=4, timeout_ms=WAIT_MS, sync=False,
                                     stream=streams[s + 1], scratch_off=40960 + 64 * s)
            pviews.append(pv)
        for st in streams:
            st.synchronize()
    finally:
        ctx.engine_stop()
    for pv in pviews:
        p = ops.parse_read_records(pv)
        assert p["status"] == "OK" and p["done"] == n_rec, p
    r = ops.parse_reduce(rv)
    assert r.ok and r.records_reduced == n_rec, r
    _check_arrival_words(full, n_src * n_rec)
    assert torch.equal(land.cpu(), landed.reshape(-1))
    assert _bits_equal(y.cpu(), want_y)
    assert torch.equal(stg.cpu(), want_r)


# ------------------------------------------------------------------ 6. the mock ConnectX through adopted queues
def test_reduce_posts_to_the_mock_connectx():
    """The reduce posts its records into the mock ConnectX's send queue mapped to the GPU.  Exact end to end, no error
    completion and no doorbell out of order."""
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        chunk, n_rec, n_src = 1 << 16, 4, 3
        n = chunk * n_rec
        nb = P.staging_bytes(n, chunk)
        recs_cpu = _source_records(n_src, n, chunk, seed=6)
        want_y, want_r = P.ref_reduce_fp8(recs_cpu, n_src, n, chunk)
        recs = recs_cpu.cuda()
        stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        dst = torch.empty(nb, dtype=torch.uint8, device="cuda")
        _poison(dst, chunk)
        y = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
        smr, dmr = vctx.reg_mr(stg), vctx.reg_mr(dst)
        qp = vctx.loopback_qp(depth=64)
        assert qp.on_gpu
        torch.cuda.synchronize()
        r = ops.reduce_fp8(vctx, recs, n_src, n, chunk, out=y, out_mr=smr, qp=qp, dst_mr=dmr, signal_every=2,
                           timeout_ms=WAIT_MS)
        assert r.ok and r.records_posted == n_rec and r.records_reduced == n_rec, r
        assert torch.equal(dst.cpu(), want_r)
        assert _bits_equal(y.cpu(), want_y)
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_db_order_violations"] == 0, c
    finally:
        vctx.close()


# ------------------------------------------------------------------ 7. host-side rejections
def test_reduce_host_side_rejections(ctx):
    chunk, n_rec, n_src = 8192, 2, 2
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    recs = torch.zeros(n_src * nb + 64, dtype=torch.uint8, device="cuda")
    y = torch.zeros(n + 16, dtype=torch.bfloat16, device="cuda")
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    small = torch.zeros(nb - 64, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    smr, small_mr, dmr = ctx.reg_mr(stg), ctx.reg_mr(small), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=16)
    words = torch.zeros(n_src * n_rec + GUARD, dtype=torch.int64, device="cuda")
    loc = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    out = y[:n]
    bad = [
        (dict(n_src=0), "n_src"),
        (dict(n_src=9), "n_src"),
        (dict(n_elems=n + 4096), "multiples"),
        (dict(chunk_elems=12288, n_elems=3 * 12288), "multiples"),
        (dict(n_elems=3 * chunk, chunk_elems=2 * chunk), "multiples"),
        (dict(records=recs[:n_src * nb - 1]), "records hold"),
        (dict(records=recs[1:n_src * nb + 1]), "aligned"),
        (dict(records=recs.cpu()), "records"),
        (dict(local=loc.float()), "local"),
        (dict(local=loc[:n - 32]), "local"),
        (dict(local=loc.cpu()), "local"),
        (dict(local=torch.zeros(2 * n, dtype=torch.bfloat16, device="cuda")[::2]), "local"),
        (dict(out=y[:n].float()), "out"),
        (dict(out=y[1:n + 1]), "out"),
        (dict(out=y[:n].cpu()), "out"),
        (dict(out=None), "needs an output"),
        (dict(out=None, out_mr=small_mr), "out_mr"),
        (dict(qp=qp), "posting"),
        (dict(qp=qp, out_mr=smr), "posting"),
        (dict(dst_mr=dmr, out_mr=smr), "dst_mr without qp"),
        (dict(qp=qp, out_mr=smr, dst_mr=dmr, dst_off=64), "do not fit"),
        (dict(ready=words.to(torch.int32)), "ready"),
        (dict(ready=words.cpu()), "ready"),
        (dict(ready=words[:n_src * n_rec - 1]), "ready"),
        (dict(scratch_slot=-1), "scratch_slot"),
        (dict(scratch_slot=8), "scratch_slot"),
    ]
    for kw, what in bad:
        args = dict(records=recs, n_src=n_src, n_elems=n, chunk_elems=chunk, out=out)
        args.update(kw)
        with pytest.raises(ValueError, match=what):
            ops.reduce_fp8(ctx, **args)
    torch.cuda.synchronize()
    assert bool((y == 0).all()) and bool((stg == 0).all()) and bool((dst == 0).all()), "a rejected call launched something"
    assert qp.counters()["n_wqe"] == 0
