"""Receive-side fusion on one GPU, against exact references.

``gemm_mxfp8(..., a_ready=words)`` starts each tile once the record it reads has landed; ``recv_consume`` turns every
receive completion into a nonzero arrival word (word = immediate = panel or chunk id).  K7 computes each tile in one CTA
or one 2-CTA cluster, in a fixed k-block order, so its result depends neither on the grid nor on when a tile starts.
Every GEMM that runs on arrival here is therefore checked twice:

  (a) bit for bit against the same call (same ``cta_group``) run after every record is in place, without ``a_ready``;
  (b) that sequential result against fp64: the round-to-nearest-even product bit for bit when the operands keep the
      fp32 accumulation exact, else the per-element bound of test_gpu_numerics.py with K7's gamma.

Every receive buffer starts out as poison that decodes nothing like a record (e4m3 448 under scale 2^127, or NaN codes),
so a tile that reads a record before it has landed, or half of one, changes bits in (a).  Direct mode -- the producer's
own stores carry the data and the queue pair only announces it -- is checked the same way, with a local destination.

Rules the tests keep (DESIGN.md 3.2):
* every kernel that waits on another is resident with it, one GEMM CTA per SM, within the 132 SMs of an H100 SXM (each
  test writes out its sum), and the launch order is consumer, then the GEMM that runs on arrival, then the producer;
* every wait is bounded by 5 s or less;
* nothing allocates, works on the default stream or synchronises the device while the engine runs;
* the arrival words are the head of a larger zeroed tensor, and the words behind them must still be zero at the end:
  a kernel that reads past them reads zeros, so it fails the same way every time instead of on leftover bytes.
"""
import ctypes as C
import time

import pytest
import torch

from rocnrdma_b200 import ops, wire as W
from rocnrdma_b200.ops import gemm_mx as MX
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.ops.rdma import WAIT_STATUS
from test_gpu_numerics import (_bits_equal, _bound_check, _chunk_records, _deq64, _edge_payload, _exact_operands, _gen,
                               _mismatch, _mx_exact_operand, _mx_exact_ref, _panel_records, _spread)

pytestmark = pytest.mark.gpu

H = W.MEM_HOST_PINNED
WAIT_MS = 5000
GUARD = 8                      # zero words behind the arrival words
POISON_Q, POISON_S = 0x7E, 0xFE  # e4m3 448 under 2^127: every product with it overflows fp32


def _k7_gamma(K):
    """K7's error bound per unit of S (DESIGN.md, fp8 numerics)."""
    return (K / 32) * 2.0 ** -23 + 32 * 2.0 ** -11


class _Records:
    """An fp8 operand [M, K] as the records it travels in: K4 panel records (128 rows each, the last one whole) or K3
    chunk records of 256 rows (``pack_fp8_write`` of a [M, K] bf16 matrix with ``chunk_elems = 256 * K``)."""

    def __init__(self, kind, M, K):
        self.kind, self.M, self.K = kind, M, K
        self.rows = 128 if kind == "panel" else 256
        self.n = -(-M // self.rows)
        self.q_bytes = self.rows * K
        self.bytes = ops.panel_record_bytes(K) if kind == "panel" else P.record_bytes(self.q_bytes)
        assert kind == "panel" or M % self.rows == 0

    def build(self, q, s):
        return _panel_records(q, s) if self.kind == "panel" else _chunk_records(q, s, self.q_bytes)

    def operand(self, buf):
        if self.kind == "panel":
            return MX.MxOperand.from_panel_records(buf, self.M, self.K)
        return MX.MxOperand.from_chunk_records(buf, self.M, self.K, self.q_bytes)

    def poison(self, buf):
        r = buf[:self.n * self.bytes].view(self.n, self.bytes)
        r.fill_(POISON_S)
        r[:, :self.q_bytes] = POISON_Q

    def parts(self, buf):
        """(e4m3 codes [M, K], scale bytes [M, K/32]) of the first M rows."""
        r = buf[:self.n * self.bytes].view(self.n, self.bytes)
        q = r[:, :self.q_bytes].reshape(self.n * self.rows, self.K)[:self.M].contiguous()
        s = r[:, self.q_bytes:self.q_bytes + self.q_bytes // 32].reshape(self.n * self.rows, self.K // 32)[:self.M].contiguous()
        return q, s


def _arrival_words(n):
    full = torch.zeros(n + GUARD, dtype=torch.int64, device="cuda")
    return full, full[:n]


def _check_arrival_words(full, n):
    missing = (full[:n] == 0).nonzero().flatten().tolist()
    assert not missing, f"records without an arrival stamp: {missing}"
    assert bool((full[n:] == 0).all()), "a word past the records was written"


def _words(view):
    return list((C.c_int64 * 8).from_buffer(view))


def _out_buffer(M, N):
    """bf16 [M, N] with a canary row behind it."""
    pad = torch.full((M + 1, N), 7.0, device="cuda", dtype=torch.bfloat16)
    return pad, pad[:M]


def _check_on_arrival(ctx, y, view, a_op, b_op, cta_group, exact=None, parts=None, label=""):
    """(a) and (b) for the on-arrival result ``y`` whose result words are ``view``: read them before the sequential call,
    which reuses the same result slot.  ``exact``: the RNE bf16 reference; else ``parts`` = (aq, as, bq, bs) for the
    fp64 bound."""
    w = _words(view)
    assert w[0] == 0, f"on-arrival GEMM: {WAIT_STATUS.get(w[0], w[0])}"
    assert w[6] == cta_group, f"ran variant {w[6]}, asked for cta_group {cta_group}"
    seq = torch.full_like(y, 7.0)
    r = ops.gemm_mxfp8(ctx, a_op, b_op, seq, cta_group=cta_group)
    assert r.ok and r.variant == cta_group, (r.status, r.variant)
    assert _bits_equal(y, seq), "on arrival vs after arrival: " + _mismatch(y, seq)
    if exact is not None:
        assert _bits_equal(seq, exact), _mismatch(seq, exact)
    else:
        aq, as_, bq, bs = parts
        A, B = _deq64(aq, as_), _deq64(bq, bs)
        _bound_check(seq, A @ B.T, A.abs() @ B.abs().T, _k7_gamma(aq.shape[1]), label)


# ------------------------------------------------------------------ host-delivered records gate their tiles
GATE_CASES = [("panel", 384), ("panel", 300), ("chunk", 512), ("chunk", 768)]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("kind,M", GATE_CASES, ids=[f"{k}-{m}" for k, m in GATE_CASES])
def test_host_delivered_records_gate_their_tiles(ctx, kind, M, cta_group):
    """The GEMM is launched before any record exists.  The host RDMA_WRITE_IMMs the records in reverse order from a
    buffer that already holds them; all but record 0 land, and 100 ms later the GEMM must still be running (its
    end-time word, zeroed at launch, is 0).  Then record 0 lands and the result is checked exactly.
    M = 384 and 300 give the pair kernel an odd number of 128-row blocks (a last tile past row M); chunk records hold
    two 128-row blocks each, so the GEMM must wait on one word per record, not one per block."""
    K, N = 256, 264
    L = _Records(kind, M, K)
    g = _gen(M * 3 + cta_group + (kind == "chunk"))
    aq, as_ = _mx_exact_operand(M, K, g)
    bq, bs = _mx_exact_operand(N, K, g)
    exact = _mx_exact_ref(aq, as_, bq, bs)
    src = L.build(aq, as_)
    rcv = torch.empty_like(src)
    L.poison(rcv)
    pad, y = _out_buffer(M, N)
    full, ready = _arrival_words(L.n)
    sm, rm = ctx.reg_mr(src), ctx.reg_mr(rcv)
    scq, rcq = ctx.create_cq(64, H), ctx.create_cq(64)        # host-posted QP; its receive CQ is polled on the GPU
    qp = ctx.create_qp(scq, rcq, 16, 16, H).connect()
    for _ in range(L.n):
        qp.post_recv(rm, 0)
    a_op, b_op = L.operand(rcv), MX.MxOperand.from_tensors(bq, bs)
    _, s_recv, s_mm = ctx.streams(3)
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + GEMM 64 = 73 of 132; the host is the producer
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, L.n, L.n, ready, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=64, cta_group=cta_group, a_ready=ready, timeout_ms=WAIT_MS,
                                  sync=False, stream=s_mm)
        for i in reversed(range(1, L.n)):
            qp.post_write(sm, rm, L.bytes, src_off=i * L.bytes, dst_off=i * L.bytes, imm=i)
        time.sleep(0.1)
        early = _words(gview)
        qp.post_write(sm, rm, L.bytes, imm=0)
        s_recv.synchronize()
        s_mm.synchronize()
        wcs = scq.wait(L.n, timeout_s=5.0)
    finally:
        ctx.engine_stop()
    assert early[2] == 0, f"the GEMM finished (status {WAIT_STATUS.get(early[0], early[0])}) before record 0 was posted"
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == L.n and cons["bytes"] == L.n * L.bytes, cons
    assert not any(w.is_error for w in wcs) and qp.counters()["n_err"] == 0
    _check_arrival_words(full, L.n)
    st = ready.tolist()
    assert all(st[i] <= st[i - 1] for i in range(1, L.n)), f"records consumed out of posting order: {st}"
    assert torch.equal(rcv, src)
    _check_on_arrival(ctx, y, gview, a_op, b_op, cta_group, exact=exact)
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


# ------------------------------------------------------------------ K4 -> wire -> K7, engine-moved
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("M", [1024, 1152, 1100])
def test_k4_wire_k7_chain_on_arrival(ctx, M, cta_group):
    """GEMM 1 (exact integer operands) emits fp8 panel records and RDMA_WRITE_IMMs each one (immediate = panel id); a
    consumer stamps each arrival; GEMM 2, launched before anything has arrived, multiplies the records as they land.
    The records equal the reference byte for byte at both ends.  M = 1152 has 9 panels (odd), M = 1100 9 with a short
    last one."""
    K1, N1, N2 = 256, 512, 264
    p, q, exact = _exact_operands(M, N1, K1, seed=M + cta_group)
    g = _gen(M * 5 + cta_group)
    wq, ws = _mx_exact_operand(N2, N1, g)
    L = _Records("panel", M, N1)
    nb = L.n * L.bytes
    ref = ops.ref_fp8_panels(exact.float())
    snd = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda")
    rcv = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L.poison(rcv)
    pad, y = _out_buffer(M, N2)
    full, ready = _arrival_words(L.n)
    sm, rm = ctx.reg_mr(snd[:nb]), ctx.reg_mr(rcv)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(L.n):
        qp.post_recv(rm, 0)
    a_op, b_op = L.operand(rcv), MX.MxOperand.from_tensors(wq, ws)
    _, s_recv, s_mm = ctx.streams(3)           # GEMM 1 runs on ctx.stream
    torch.cuda.synchronize()
    # SMs: engine 8 + GEMM 1 48 + consumer 1 + GEMM 2 64 = 121 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, L.n, L.n, ready, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=64, cta_group=cta_group, a_ready=ready, timeout_ms=WAIT_MS,
                                  sync=False, stream=s_mm)
        r1 = ops.gemm_send(ctx, p, q, snd, c_mr=sm, qp=qp, dst_mr=rm, out_fp8=True, with_imm=True, grid=48, timeout_ms=WAIT_MS)
        s_recv.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    assert r1.ok and r1.panels_posted == L.n, (r1.status, r1.panels_posted)
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == L.n and cons["bytes"] == nb, cons
    assert qp.counters()["n_err"] == 0
    _check_arrival_words(full, L.n)
    assert torch.equal(snd[:nb], ref), "GEMM 1's records differ from the reference"
    assert torch.all(snd[nb:] == 0xAB), "GEMM 1 stored beyond the last record"
    assert torch.equal(rcv, ref), "the delivered records differ from the reference"
    xq, xs = L.parts(ref)
    _check_on_arrival(ctx, y, gview, a_op, b_op, cta_group, parts=(xq, xs, wq, ws), label=f"K4->K7 M={M} cta_group={cta_group}")
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


# ------------------------------------------------------------------ K3 -> wire -> K7, engine-moved
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("M", [512, 768])
def test_k3_wire_k7_chain_on_arrival(ctx, M, cta_group):
    """A bf16 [M, K] matrix packed into chunk records of 256 rows and RDMA_WRITE_IMM'd one by one (immediate = chunk id);
    GEMM 2 uses the records as they land, waiting on one word per record."""
    K, N = 256, 264
    chunk = 256 * K
    L = _Records("chunk", M, K)
    g = _gen(M * 7 + cta_group)
    x = _spread(M, K, g, 32).to(torch.bfloat16).cuda()
    bq, bs = _mx_exact_operand(N, K, g)
    nb = L.n * L.bytes
    ref = ops.ref_pack_fp8(x.reshape(-1), chunk)
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    rcv = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L.poison(rcv)
    pad, y = _out_buffer(M, N)
    full, ready = _arrival_words(L.n)
    smr, rmr = ctx.reg_mr(stg), ctx.reg_mr(rcv)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(L.n):
        qp.post_recv(rmr, 0)
    a_op, b_op = L.operand(rcv), MX.MxOperand.from_tensors(bq, bs)
    _, s_recv, s_mm = ctx.streams(3)
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + GEMM 2 64 + pack 32 = 105 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, L.n, L.n, ready, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=64, cta_group=cta_group, a_ready=ready, timeout_ms=WAIT_MS,
                                  sync=False, stream=s_mm)
        r = ops.pack_fp8_write(ctx, x.reshape(-1), smr, qp=qp, dst_mr=rmr, chunk_elems=chunk, with_imm=True, grid=32,
                               timeout_ms=WAIT_MS)
        s_recv.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.wqes == L.n, r
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == L.n and cons["bytes"] == nb, cons
    assert qp.counters()["n_err"] == 0
    _check_arrival_words(full, L.n)
    assert torch.equal(stg, ref), "packed records differ from the reference"
    assert torch.equal(rcv, ref), "the delivered records differ from the reference"
    xq, xs = L.parts(ref)
    _check_on_arrival(ctx, y, gview, a_op, b_op, cta_group, parts=(xq, xs, bq, bs), label=f"K3->K7 M={M} cta_group={cta_group}")
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


# ------------------------------------------------------------------ direct mode, K4
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("out_fp8", [False, True], ids=["bf16", "fp8"])
def test_k4_direct_mode_local_destination(ctx, out_fp8, cta_group):
    """``gemm_send(direct=True)`` into a local registered buffer: the epilogue's stores are the transfer and each panel
    is announced by a zero-length RDMA_WRITE_IMM.  The destination is exact, nothing moved on the wire (0 bytes), and
    with fp8 records a GEMM that runs on the announcements reads exactly what the epilogue stored."""
    M, N, K, N2 = 512, 512, 256, 264
    a, b, exact = _exact_operands(M, N, K, seed=41 + 2 * cta_group + int(out_fp8))
    panels = M // 128
    if out_fp8:
        L = _Records("panel", M, N)
        nb = L.n * L.bytes
        buf = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda")
        d = buf[:nb]
        L.poison(d)
        want, canary = ops.ref_fp8_panels(exact.float()), 0xAB
    else:
        buf = torch.full((M * N + 64,), 7.0, dtype=torch.bfloat16, device="cuda")
        d = buf[:M * N].view(M, N)
        d.fill_(float("nan"))
        want, canary = exact.to(torch.bfloat16), 7.0
    dm = ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(panels):
        qp.post_recv(dm, 0)
    full, ready = _arrival_words(panels)
    if out_fp8:
        wq, ws = _mx_exact_operand(N2, N, _gen(43 + cta_group))
        pad, y = _out_buffer(M, N2)
        a_op, b_op = L.operand(d), MX.MxOperand.from_tensors(wq, ws)
    _, s_recv, s_mm = ctx.streams(3)
    torch.cuda.synchronize()
    # SMs: engine 8 + GEMM 1 48 + consumer 1 (+ GEMM 2 64 with fp8 records) = 121 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, panels, panels, ready, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        if out_fp8:
            gview, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y, grid=64, cta_group=cta_group, a_ready=ready, timeout_ms=WAIT_MS,
                                      sync=False, stream=s_mm)
        r1 = ops.gemm_send(ctx, a, b, d, c_mr=dm, qp=qp, dst_mr=dm, direct=True, with_imm=True, out_fp8=out_fp8,
                           cta_group=cta_group, grid=48, timeout_ms=WAIT_MS)
        s_recv.synchronize()
        s_mm.synchronize()
    finally:
        ctx.engine_stop()
    assert r1.ok and r1.panels_posted == panels and r1.variant == cta_group, (r1.status, r1.panels_posted, r1.variant)
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == panels and cons["bytes"] == 0, cons
    assert qp.counters()["n_err"] == 0
    _check_arrival_words(full, panels)
    if out_fp8:
        diff = (d != want).nonzero()
        assert diff.numel() == 0, f"{diff.numel()} record bytes differ, first at {diff[0].item()}"
        assert torch.all(buf[nb:] == canary), "stored beyond the last record"
        xq, xs = L.parts(want)
        _check_on_arrival(ctx, y, gview, a_op, b_op, cta_group, parts=(xq, xs, wq, ws), label=f"direct K4->K7 cta_group={cta_group}")
        assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"
    else:
        assert _bits_equal(d, want), _mismatch(d, want)
        assert torch.all(buf[M * N:] == canary), "stored beyond the destination"


# ------------------------------------------------------------------ direct mode, K3
@pytest.mark.parametrize("pack_grid", [1, 3, 0])
def test_k3_direct_pack_unpacked_on_arrival(ctx, pack_grid):
    """``pack_fp8_write(direct=True)`` stores the records into the destination itself and announces each with a
    zero-length RDMA_WRITE_IMM; ``unpack_fp8`` waits for each announcement before reading the record.  The destination
    starts as NaN codes, so an unpack that ran ahead of a record leaves NaN in the output."""
    chunk, n_chunks = 16384, 6
    n = chunk * n_chunks
    x = torch.nan_to_num(_edge_payload(n).float(), nan=1.0, posinf=2.0, neginf=-2.0).to(torch.bfloat16).cuda()
    nb = P.staging_bytes(n, chunk)
    ref = P.ref_pack_fp8(x, chunk)
    want = P.ref_unpack_fp8(ref, n, chunk)
    assert not bool(torch.isnan(want).any())
    remote = torch.full((nb,), 0x7F, dtype=torch.uint8, device="cuda")
    out = torch.full((n,), float("nan"), dtype=torch.bfloat16, device="cuda")
    rmr = ctx.reg_mr(remote)
    cq_a, cq_b = ctx.create_cq(256), ctx.create_cq(256)
    qa = ctx.create_qp(cq_a, cq_a, 64, 64)
    qb = ctx.create_qp(cq_b, cq_b, 64, 64)
    qa.connect(qb)
    for _ in range(n_chunks):
        qb.post_recv(rmr, 0)
    torch.cuda.synchronize()
    # SMs: engine 16 + unpack 4 (the CQ poller and 3 workers, which wait for arrivals) = 20 of 132; the pack's CTAs wait
    # for nothing but the engine
    ctx.engine_start(ctas=16, idle_timeout_ms=WAIT_MS)
    try:
        uview, ust = P.unpack_fp8(ctx, remote, out, chunk, qp=qb, grid=3, timeout_ms=WAIT_MS, sync=False, stream=ctx.aux_stream)
        r = P.pack_fp8_write(ctx, x, rmr, qp=qa, dst_mr=rmr, chunk_elems=chunk, with_imm=True, direct=True, grid=pack_grid,
                             timeout_ms=WAIT_MS)
        ust.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.wqes == n_chunks, r
    u = P.parse_unpack(uview)
    assert u["status"] == "OK" and u["records_seen"] == n_chunks, u
    assert qa.counters()["n_err"] == 0
    assert torch.equal(remote, ref), "records differ from the reference"
    bad = (out.view(torch.int16) != want.view(torch.int16)).nonzero().flatten()
    assert bad.numel() == 0, f"{bad.numel()} unpacked values differ, first at {bad[0].item()}: got {out[bad[0]].item()}"


# ------------------------------------------------------------------ host-side checks
def test_a_ready_takes_one_word_per_record(ctx):
    """One arrival word per record of A: a plain matrix is one record, chunk records of 256 rows need M / 256 words.
    All words are set, so nothing waits; the result equals the same call without ``a_ready``."""
    K, N = 256, 136
    g = _gen(77)
    bq, bs = _mx_exact_operand(N, K, g)
    b_op = MX.MxOperand.from_tensors(bq, bs)
    for kind, M in (("plain", 300), ("chunk", 512)):
        aq, as_ = _mx_exact_operand(M, K, g)
        if kind == "plain":
            a_op, n_rec = MX.MxOperand.from_tensors(aq, as_), 1
        else:
            L = _Records(kind, M, K)
            a_op, n_rec = L.operand(L.build(aq, as_)), L.n
        ready = torch.ones(n_rec, dtype=torch.int64, device="cuda")
        y, y0 = (torch.zeros(M, N, device="cuda", dtype=torch.bfloat16) for _ in range(2))
        assert ops.gemm_mxfp8(ctx, a_op, b_op, y, a_ready=ready).ok
        assert ops.gemm_mxfp8(ctx, a_op, b_op, y0).ok
        assert _bits_equal(y, y0), (kind, _mismatch(y, y0))


def test_receive_fusion_host_side_rejections(ctx):
    # direct K4: whole tiles only
    a = torch.zeros(300, 256, dtype=torch.bfloat16, device="cuda")
    b = torch.zeros(256, 256, dtype=torch.bfloat16, device="cuda")
    c = torch.zeros(300, 256, dtype=torch.bfloat16, device="cuda")
    cm = ctx.reg_mr(c)
    qp = ctx.loopback_qp(depth=16)
    with pytest.raises(ValueError, match="direct"):
        ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=cm, direct=True, with_imm=True)
    # direct K3: records are announced by RDMA_WRITE_IMM
    x = torch.zeros(2 * P.TILE_ELEMS, dtype=torch.bfloat16, device="cuda")
    stg = torch.zeros(P.staging_bytes(x.numel(), P.TILE_ELEMS), dtype=torch.uint8, device="cuda")
    sm = ctx.reg_mr(stg)
    with pytest.raises(ValueError, match="with_imm"):
        P.pack_fp8_write(ctx, x, sm, qp=qp, dst_mr=sm, chunk_elems=P.TILE_ELEMS, direct=True)
    # K7: fewer arrival words than records
    K = 64
    b_op = MX.MxOperand.from_tensors(*_mx_exact_operand(8, K, _gen(5)))
    for kind, M, words in (("panel", 300, 2), ("chunk", 512, 1)):
        L = _Records(kind, M, K)
        a_op = L.operand(torch.zeros(L.n * L.bytes, dtype=torch.uint8, device="cuda"))
        y = torch.zeros(M, 8, device="cuda", dtype=torch.bfloat16)
        with pytest.raises(ValueError, match="one word per record"):
            ops.gemm_mxfp8(ctx, a_op, b_op, y, a_ready=torch.ones(words, dtype=torch.int64, device="cuda"))
