"""``reduce_fp8`` where its schedule gets hard: steps that hold several tiles of one record, ``post_only``, and every
e4m3 code under every scale byte against a decoder that shares nothing with the package's references.

* `ReduceSchedule` mirrors `pack_fp8.cu` as the host launches the reduce and its workers walk it: the variant rule (P and
  the addend give G tiles per step and PMAX sources), the grid clamp, the step walk (CTA b takes steps T0 = b,
  b + grid * G, ...; the tiles of a step are T0 + g * grid), and per step the runs of tiles by record -- thread 0 adds
  each run's length to its record's counter and the CTA that brings it to tiles-per-record posts the record -- and the
  records the step waits on.  Every case below asserts the facts it exercises; test_reduce_references.py checks the
  model against hand-counted walks on the CPU.
* test_gpu_reduce.test_reduce_matches_reference runs P = 1..5, 7 and 8, with and without the addend: every variant
  at P = PMAX, and at P < PMAX wherever the variant rule sends a smaller P to it (test_reduce_references.py checks it).
* Posting cases run with WRITE_IMM on a loopback QP, the engine resident, and a ``recv_consume`` launched first that
  stamps one word per record landed downstream: every record must be posted exactly once, and what lands must equal
  ``ref_reduce_fp8`` byte for byte.
* The sweep decodes e4m3 from its bit fields and UE8M0 as 2^(byte - 127) in fp64, rounds fp32 to bf16 from the bits,
  and sums with numpy fp32 adds in source order: no ``torch.float8_e4m3fn`` and no ``ops.pack.ue8m0``.

The rules of test_gpu_receive_fusion.py hold: every kernel that waits on another is launched first and is resident with
it (each launch writes out its SM budget), every wait is bounded by 5 s or less, nothing allocates or synchronises the
device while the engine runs, and landing buffers start as poison with canaries behind them.
"""
import time

import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops, wire as W
from rocnrdma_b200.ops import pack as P
from test_gpu_numerics import H100_SMS, _gen, _records_equal_up_to_nan_sign
from test_gpu_receive_fusion import _arrival_words, _check_arrival_words
from test_gpu_reduce import CANARY, POISON_Q, POISON_S, WAIT_MS, _bf16_equal_up_to_nan, _poison, _source_records

pytestmark = pytest.mark.gpu

TILE = P.TILE_ELEMS
# (G tiles per step, PMAX sources, addend): pack_fp8.cu RN_REDUCE_VARIANTS, the entries with EF = false
VARIANTS = ((4, 1, False), (4, 2, False), (2, 4, False), (1, 8, False), (2, 2, True), (1, 8, True))
# ... and the entries with EF = true (a residual): P = 1 without the addend, P <= 2 with it, one tile per step
EF_VARIANTS = ((1, 1, False), (1, 2, True))


# ------------------------------------------------------------------ schedule model
def variant_of(n_src, local, ef=False):
    """The variant rn_k_reduce_fp8 launches for P = ``n_src`` sources, with or without the addend, and with or without
    a residual (``ef``; the host refuses other P with one)."""
    if local:
        pmax = 2 if n_src <= 2 else 8
    else:
        pmax = 1 if n_src == 1 else 2 if n_src <= 2 else 4 if n_src <= 4 else 8
    return next(v for v in (EF_VARIANTS if ef else VARIANTS) if v[1:] == (pmax, bool(local)))


class ReduceSchedule:
    """One launch of ``reduce_fp8``: ``steps[b]`` lists CTA b's steps in order, each as the list of its tiles in the
    flattened record-major order (tile T belongs to record T // tpc)."""

    def __init__(self, chunk, n_rec, n_src, local=False, grid=0, ready=False, sms=H100_SMS, ef=False):
        self.tpc, self.n_rec, self.n_src = chunk // TILE, n_rec, n_src
        self.variant = variant_of(n_src, local, ef)
        self.G, self.pmax = self.variant[0], self.variant[1]
        self.total = n_rec * self.tpc
        if grid <= 0:
            grid = sms if ready else 4 * sms
        self.requested = grid
        self.grid = min(grid, self.total)
        G, g_, total = self.G, self.grid, self.total
        self.steps = [[[T0 + g * g_ for g in range(G) if T0 + g * g_ < total] for T0 in range(b, total, g_ * G)]
                      for b in range(g_)]

    def runs(self, tiles):
        """(record, n) per run of a step's tiles, in the order thread 0 counts them."""
        out = []
        for T in tiles:
            r = T // self.tpc
            if out and out[-1][0] == r:
                out[-1][1] += 1
            else:
                out.append([r, 1])
        return [tuple(x) for x in out]

    def waits(self, tiles):
        """The records whose words (one per source) a gated step waits on before it reads anything."""
        return [r for r, _ in self.runs(tiles)]

    def owners(self):
        """Record -> the CTAs that hold its tiles."""
        own = {r: set() for r in range(self.n_rec)}
        for b, steps in enumerate(self.steps):
            for tiles in steps:
                for T in tiles:
                    own[T // self.tpc].add(b)
        return own

    def completing_steps(self):
        """(CTA, step) -> the records that step completes whatever the timing: records whose tiles all belong to that CTA
        and whose last tile is in that step."""
        own, out = self.owners(), {}
        for b, steps in enumerate(self.steps):
            for i, tiles in enumerate(steps):
                for T in tiles:
                    if T % self.tpc == self.tpc - 1 and own[T // self.tpc] == {b}:
                        out.setdefault((b, i), set()).add(T // self.tpc)
        return out

    def facts(self):
        all_steps = [tiles for steps in self.steps for tiles in steps]
        runs = [self.runs(t) for t in all_steps]
        own = self.owners()
        return {
            "multi_tile_run": any(n > 1 for rs in runs for _, n in rs),
            "boundary_in_step": any(len(rs) > 1 and any(n > 1 for _, n in rs) for rs in runs),
            "step_completes_two": any(len(rs) >= 2 for rs in self.completing_steps().values()),
            "record_owned_by_one_cta": any(len(c) == 1 for c in own.values()),
            "record_shared": any(len(c) > 1 for c in own.values()),
            "partial_last_step": any(len(t) < self.G for t in all_steps),
            "waits_on_a_later_record": any(len(self.waits(t)) > 1 for t in all_steps),
            "variant": self.variant,
            "full_width": self.n_src == self.pmax,
        }


FACTS = ("multi_tile_run", "boundary_in_step", "step_completes_two", "record_owned_by_one_cta", "record_shared",
         "partial_last_step", "waits_on_a_later_record")

# (chunk, records, P, addend, grid, dst_off): tiles per record 3, 5, 6 and 128; G 4, 2, 2, 1 and 4
POST_CASES = [
    (24576, 5, 2, False, 1, 0),        # tpc 3, G 4, one CTA: runs (r0 x3, r1 x1), (r1 x2, r2 x2), (r2 x1, r3 x3), (r4 x3)
    (40960, 6, 1, True, 2, 0),         # tpc 5, G 2: records shared by two CTAs, steps that straddle two records
    (49152, 7, 3, False, 3, 4160),     # tpc 6, G 2 at partial width (PMAX 4), records land 4160 bytes into the region
    (1 << 20, 5, 8, True, 4, 0),       # tpc 128, G 1 at full width with the addend: 32 steps per CTA per record
    (1 << 20, 5, 1, False, 3, 0),      # tpc 128, G 4, grid 3: runs of 4 and a short last step
]
POST_IDS = [f"tpc{c // TILE}-rec{n}-P{p}{'-local' if l else ''}-grid{g}{f'-off{o}' if o else ''}"
            for c, n, p, l, g, o in POST_CASES]


def _local(n, seed):
    return (torch.randn(n, generator=_gen(seed)) * 64).to(torch.bfloat16)


# ------------------------------------------------------------------ independent decoder and sum
def e4m3_fp64(codes):
    """e4m3 codes (uint8 array) -> fp64 from the bit fields: sign, 4-bit exponent (bias 7), 3-bit mantissa, subnormals
    at exponent 0, NaN for 0x7F / 0xFF and no Inf."""
    c = np.asarray(codes, dtype=np.int64)
    e, m = (c >> 3) & 0xF, c & 7
    mag = np.where(e == 0, m * 2.0 ** -9, (8 + m) * np.exp2(e - 10.0))
    v = np.where(c & 0x80, -mag, mag)
    return np.where((c & 0x7F) == 0x7F, np.nan, v)


def ue8m0_fp64(scale_bytes):
    """UE8M0 scale bytes -> fp64: 2^(byte - 127), byte 0x00 = 2^-127, byte 0xFF = Inf."""
    b = np.asarray(scale_bytes, dtype=np.int64)
    return np.where(b == 0xFF, np.inf, np.exp2(b - 127.0))


def decode_fp32(records, n_src, n_elems, chunk):
    """fp32 [n_src, n_elems] of source-major records: the fp64 product of code and scale, rounded once to fp32 (exact
    unless it reaches 2^128, which is Inf in both)."""
    rec = P.record_bytes(chunk)
    n_rec = n_elems // chunk
    r = np.asarray(records.reshape(-1)[:n_src * n_rec * rec].numpy()).reshape(n_src * n_rec, rec)
    q = e4m3_fp64(r[:, :chunk]).reshape(-1, 32)
    s = ue8m0_fp64(r[:, chunk:chunk + chunk // 32]).reshape(-1, 1)
    with np.errstate(over="ignore", invalid="ignore"):
        return (q * s).astype(np.float32).reshape(n_src, n_elems)


def bf16_rne_bits(x):
    """fp32 -> bf16 bits, round to nearest even on the bit pattern; NaN stays NaN (quiet, with its sign)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    out = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(x)
    out[nan] = (0x7FC0 | ((u[nan] >> 16) & 0x8000)).astype(np.uint16)
    return out


def independent_sum_bits(records, n_src, n_elems, chunk, local=None):
    """bf16 bits of the reduce's sum: from ``local`` (bf16 bits widened) or from source 0, then the other sources in
    source order, one numpy fp32 add each."""
    d = decode_fp32(records, n_src, n_elems, chunk)
    if local is not None:
        acc = (local.view(torch.int16).numpy().astype(np.uint16).astype(np.uint32) << 16).view(np.float32)
        first = 0
    else:
        acc, first = d[0], 1
    with np.errstate(over="ignore", invalid="ignore"):
        for s in range(first, n_src):
            acc = acc + d[s]
    return bf16_rne_bits(acc)


SWEEP = 1 << 16        # one record: 256 codes x 256 scale bytes, 8 blocks of 32 per scale byte


def sweep_records(n_src, seed):
    """``n_src`` sources of one 65536-element record each.  Every source holds every (code, scale byte) pair once:
    scale byte b's 256 codes fill 8 blocks.  Source s permutes the codes within each scale byte and then the 2048
    blocks, each with its own permutation, so a pair sits beside different partners in every source position."""
    g = _gen(seed)
    rec = P.record_bytes(SWEEP)
    out = torch.zeros(n_src, rec, dtype=torch.uint8)
    for s in range(n_src):
        codes = torch.argsort(torch.rand(256, 256, generator=g), dim=1).to(torch.uint8)       # row b: scale byte b
        scales = torch.arange(256, dtype=torch.int32).repeat_interleave(8).to(torch.uint8)     # 2048 blocks
        perm = torch.randperm(2048, generator=g)
        out[s, :SWEEP] = codes.reshape(2048, 32)[perm].reshape(-1)
        out[s, SWEEP:SWEEP + SWEEP // 32] = scales[perm]
    return out.reshape(-1)


def sweep_addend(seed):
    """A bf16 addend for the sweep: zero in every other block, so the smallest decoded values still reach the sum, and
    spread over 2^-40..2^40 in the others."""
    g = _gen(seed)
    x = torch.randn(SWEEP, generator=g) * torch.exp2(torch.randint(-40, 41, (SWEEP // 32,), generator=g).float()).repeat_interleave(32)
    x.view(-1, 64)[:, :32] = 0.0
    return x.to(torch.bfloat16)


def _u16(t):
    return t.view(torch.int16).numpy().astype(np.uint16)


def _assert_bf16_bits(got, want_bits, label=""):
    """bf16 tensor against reference bits: NaN at the same positions, every other value identical."""
    g = _u16(got)
    gn, wn = (g & 0x7FFF) > 0x7F80, (want_bits & 0x7FFF) > 0x7F80
    assert np.array_equal(gn, wn), f"{label}: NaN at {int((gn != wn).sum())} different positions"
    bad = np.flatnonzero(g[~wn] != want_bits[~wn])
    assert bad.size == 0, f"{label}: {bad.size} values differ, first got 0x{g[~wn][bad[0]]:04x} want 0x{want_bits[~wn][bad[0]]:04x}"


# ------------------------------------------------------------------ B. posting where steps share records
@pytest.mark.parametrize("gated", [False, True], ids=["posted", "words_set"])
@pytest.mark.parametrize("signal_every", [1, 4])
@pytest.mark.parametrize("case", POST_CASES, ids=POST_IDS)
def test_reduce_posts_every_record_once(ctx, case, signal_every, gated):
    """Every record completed by runs of several tiles, across record boundaries inside a step, or two at once, is
    posted exactly once: ``records_posted == n_rec``, one WQE per record plus the flush, one arrival stamp per record
    downstream, and the landed records, the local records and the bf16 sum equal the reference.  ``words_set`` runs the
    same walk through the gated path (every arrival word already nonzero)."""
    chunk, n_rec, n_src, local, grid, dst_off = case
    sch = ReduceSchedule(chunk, n_rec, n_src, local, grid, ready=gated)
    assert sch.grid == grid
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    recs_cpu = _source_records(n_src, n, chunk, seed=chunk // TILE + 7 * n_src, edges=True)
    loc_cpu = _local(n, n_rec + 200) if local else None
    want_y, want_r = P.ref_reduce_fp8(recs_cpu, n_src, n, chunk, local=loc_cpu)
    recs = recs_cpu.cuda()
    loc = loc_cpu.cuda() if local else None
    ybuf = torch.full((n + 64,), 7.0, dtype=torch.bfloat16, device="cuda")
    rbuf = torch.full((nb + 256,), CANARY, dtype=torch.uint8, device="cuda")
    _poison(rbuf[:nb], chunk)
    dbuf = torch.full((dst_off + nb + 256,), CANARY, dtype=torch.uint8, device="cuda")
    _poison(dbuf[dst_off:dst_off + nb], chunk)
    smr, dmr = ctx.reg_mr(rbuf[:nb]), ctx.reg_mr(dbuf)
    ready = None
    if gated:
        full_in, ready = _arrival_words(n_src * n_rec)
        ready.fill_(1)
    full, stamps = _arrival_words(n_rec)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(n_rec):
        qp.post_recv(dmr, 0)
    s_recv, s_red = ctx.streams(2)
    torch.cuda.synchronize()
    # SMs: engine 8 + consumer 1 + reduce <= 4 = 13 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        cview, _ = ops.recv_consume(qp, n_rec, n_rec, stamps, timeout_ms=WAIT_MS, sync=False, stream=s_recv)
        r = ops.reduce_fp8(ctx, recs, n_src, n, chunk, local=loc, out=ybuf[:n], out_mr=smr, qp=qp, dst_mr=dmr,
                           dst_off=dst_off, with_imm=True, signal_every=signal_every, ready=ready, grid=grid,
                           timeout_ms=WAIT_MS, stream=s_red)
        s_recv.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.records_reduced == n_rec and r.records_posted == n_rec, r
    cons = ops.parse_recv(cview)
    assert cons["status"] == "OK" and cons["seen"] == n_rec, cons
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == n_rec + 1, c
    _check_arrival_words(full, n_rec)
    if gated:
        _check_arrival_words(full_in, n_src * n_rec)
    _records_equal_up_to_nan_sign(dbuf[dst_off:dst_off + nb].cpu(), want_r, chunk)
    _records_equal_up_to_nan_sign(rbuf[:nb].cpu(), want_r, chunk)
    _bf16_equal_up_to_nan(ybuf[:n].cpu(), want_y)
    assert bool((dbuf[:dst_off] == CANARY).all()) and bool((dbuf[dst_off + nb:] == CANARY).all()), "stored outside the records"
    assert bool((rbuf[nb:] == CANARY).all()), "stored past the last output record"
    assert bool((ybuf[n:] == 7.0).all()), "stored past the bf16 output"


WAIT_CASE = (24576, 5, 2, 1)          # (chunk, records, P, grid): tpc 3, G 4, one CTA


def test_reduce_waits_on_the_second_record_of_a_step(ctx):
    """tpc 3, grid 1, G 4: step 0 reads tiles 0-3, so records 0 and 1.  Launched on poisoned records; another stream
    lands and stamps every record except (source 1, record 1); 100 ms later the end-time word is still 0.  Then that
    record lands, and the sum is exact.  A worker that waited only on the first record of a step would read record 1
    of source 1 as poison in step 0."""
    chunk, n_rec, n_src, grid = WAIT_CASE
    sch = ReduceSchedule(chunk, n_rec, n_src, False, grid, ready=True)
    assert sch.G == 4 and sch.waits(sch.steps[0][0]) == [0, 1]
    n = chunk * n_rec
    rec = P.record_bytes(chunk)
    recs_cpu = _source_records(n_src, n, chunk, seed=21)
    want_y, want_r = P.ref_reduce_fp8(recs_cpu, n_src, n, chunk)
    recs = recs_cpu.cuda()
    land = torch.empty_like(recs)
    y = torch.full((n,), float("nan"), dtype=torch.bfloat16, device="cuda")
    stg = torch.zeros(P.staging_bytes(n, chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(stg)
    full, ready = _arrival_words(n_src * n_rec)
    last = 1 * n_rec + 1
    order = [i for i in range(n_src * n_rec) if i != last]
    s_set, s_red = ctx.streams(2)

    def land_one(i):
        land[i * rec:(i + 1) * rec].copy_(recs[i * rec:(i + 1) * rec])
        ready[i:i + 1].fill_(1)

    # the setter runs once before the reduce exists, so that only these calls load what it needs (DESIGN.md 3.2)
    with torch.cuda.stream(s_set):
        for i in order + [last]:
            land_one(i)
    torch.cuda.synchronize()
    _poison(land, chunk)
    full.zero_()
    torch.cuda.synchronize()
    # SMs: the reduce 1 CTA; the setter's copies and fills wait on nothing
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
    assert early.t_end_ns == 0, f"the reduce finished ({early.status}) before record (1, 1) was in place"
    r = ops.parse_reduce(view)
    assert r.ok and r.records_reduced == n_rec, r
    _check_arrival_words(full, n_src * n_rec)
    _bf16_equal_up_to_nan(y.cpu(), want_y)
    assert torch.equal(stg.cpu(), want_r)


# ------------------------------------------------------------------ D. post_only, delivered by a later engine run
def _send_cqes(qp):
    wc = qp.scq.poll(64)
    assert not any(w.is_error for w in wc) and all(w.opcode == W.CQE_REQ for w in wc), wc
    return [w.wqe_counter for w in wc]


@pytest.mark.parametrize("kernel", ["reduce", "pack"])
def test_post_only_then_engine_run(ctx, kernel):
    """The kernel posts every record and the flush with no engine resident and returns; nothing has landed yet.  A
    one-shot engine run then delivers them: the records at the destination are exact, one WQE per record plus the flush,
    and the send CQ holds exactly the signaled WQEs (every second one) and the flush, none in error.  The next ordinary
    call on the same QP and scratch slot runs clean."""
    chunk, n_rec, n_src, grid, sig = 24576, 5, 2, 1, 2
    n = chunk * n_rec
    nb = P.staging_bytes(n, chunk)
    if kernel == "reduce":
        recs = _source_records(n_src, n, chunk, seed=31, edges=True)
        _, want = P.ref_reduce_fp8(recs, n_src, n, chunk)
        recs = recs.cuda()
    else:
        x_cpu = (torch.randn(n, generator=_gen(32)) * 16).to(torch.bfloat16)
        want = P.ref_pack_fp8(x_cpu, chunk)
        x = x_cpu.cuda()
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nb, dtype=torch.uint8, device="cuda")
    smr, dmr = ctx.reg_mr(stg), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)

    def run(post_only):
        if kernel == "reduce":
            r = ops.reduce_fp8(ctx, recs, n_src, n, chunk, out_mr=smr, qp=qp, dst_mr=dmr, signal_every=sig,
                               post_only=post_only, grid=grid, timeout_ms=WAIT_MS)
            assert r.ok and r.records_reduced == n_rec and r.records_posted == n_rec, r
        else:
            r = ops.pack_fp8_write(ctx, x, smr, qp=qp, dst_mr=dmr, chunk_elems=chunk, signal_every=sig, grid=grid,
                                   post_only=post_only, timeout_ms=WAIT_MS)
            assert r.ok and r.wqes == n_rec, r

    _poison(dst, chunk)
    torch.cuda.synchronize()
    run(post_only=True)
    assert bool((dst[:chunk] == POISON_Q).all()) and bool((dst[chunk:P.record_bytes(chunk)] == POISON_S).all()), \
        "a record landed with no engine resident"
    ctx.engine_run_oneshot(ctas=8)
    assert ctx.last_engine_fatal == 0
    _records_equal_up_to_nan_sign(dst.cpu(), want, chunk)
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == n_rec + 1, c
    # records at WQE indices 0..4 signal every second slot (1 and 3); the flush at index 5 is always signaled
    assert _send_cqes(qp) == [1, 3, n_rec], "send completions"
    # the same QP and scratch slot, waited on as usual
    _poison(dst, chunk)
    stg.zero_()
    torch.cuda.synchronize()
    # SMs: engine 8 + the kernel 1 of 132
    ctx.engine_start(ctas=8, idle_timeout_ms=WAIT_MS)
    try:
        run(post_only=False)
    finally:
        ctx.engine_stop()
    _records_equal_up_to_nan_sign(dst.cpu(), want, chunk)
    assert torch.equal(stg.cpu(), dst.cpu())
    c = qp.counters()
    assert c["n_err"] == 0 and c["n_wqe"] == 2 * (n_rec + 1), c


# ------------------------------------------------------------------ E. every code under every scale byte
SWEEP_CASES = [(1, False), (2, False), (2, True), (3, False), (3, True)]


@pytest.mark.parametrize("n_src,local", SWEEP_CASES, ids=[f"P{p}{'-local' if l else ''}" for p, l in SWEEP_CASES])
def test_reduce_every_code_under_every_scale(ctx, n_src, local):
    """Each source holds all 65536 (e4m3 code, scale byte) pairs, permuted differently: the bf16 sum equals the
    independent fp64-decoded, numpy-summed reference bit for bit (NaN at the same positions), and the records of the
    sum equal ``ref_reduce_fp8``.  P = 1 without an addend is the decode alone."""
    recs_cpu = sweep_records(n_src, seed=500 + 2 * n_src + local)
    loc_cpu = sweep_addend(600 + n_src) if local else None
    want_bits = independent_sum_bits(recs_cpu, n_src, SWEEP, SWEEP, local=loc_cpu)
    _, want_r = P.ref_reduce_fp8(recs_cpu, n_src, SWEEP, SWEEP, local=loc_cpu)
    nb = P.record_bytes(SWEEP)
    recs = recs_cpu.cuda()
    loc = loc_cpu.cuda() if local else None
    y = torch.empty(SWEEP, dtype=torch.bfloat16, device="cuda")
    stg = torch.empty(nb, dtype=torch.uint8, device="cuda")
    mr = ctx.reg_mr(stg)
    for grid in (1, 0):
        y.fill_(7.0)
        stg.fill_(CANARY)
        r = ops.reduce_fp8(ctx, recs, n_src, SWEEP, SWEEP, local=loc, out=y, out_mr=mr, grid=grid)
        assert r.ok and r.records_reduced == 1, r
        _assert_bf16_bits(y.cpu(), want_bits, f"grid {grid}")
        _records_equal_up_to_nan_sign(stg.cpu(), want_r, SWEEP)
