"""Both GEMMs bit for bit at the benchmark's shapes with many tiles per CTA, and the K4 epilogues at their edges.

* Scale: the exact-integer construction of test_gpu_numerics.py (sparse A, at most 128 nonzeros per row, entries in
  [-1, 4], so S = |A| @ |B|^T <= 2^11 at any K) at 4096^3, 8192 x 8192 x 2048, 16384 x 4096 x 1024 and 8192^3, on the
  default grid, on the grid the GEMM gets next to a 32-CTA engine, and on a small odd grid where one unit runs dozens
  of tiles.  The reference is fp64 on the GPU; the bf16 output must equal its round-to-nearest-even bit for bit.  The
  schedule model below (`Schedule`) mirrors both kernels' launch rule and tile loop; every case asserts what it
  exercises: tiles per unit, a tile that enters the operand ring at a nonzero stage, panels whose completion order the
  schedule leaves to run time.  test_numerics_references.py checks the model on the CPU.
* Edges: operands built so that every output is the exact fp32 sum of at most two chosen products (B holds powers of two
  at k positions no other column uses), filling the output's 32-column MX blocks with the quantiser's edge classes
  (zero blocks, 448 * 2^k and the next fp32 above it, e4m3 ties and the same ties nudged below bf16 precision, e4m3
  subnormals, values that round to signed zero, bf16 ties, values near fp32 max), and with the classes whose value rests
  on how wgmma accumulates (+-Inf, Inf - Inf, a NaN row of A, fp32 subnormal accumulators, -0): those are checked
  against the behaviour observed on an H100, which DESIGN.md records, and both epilogues must round and quantise
  whatever the accumulator holds exactly as the references do."""
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import gemm_mx as MX
from test_gpu_numerics import (H100_SMS, StreamK, _bits_equal, _chunk_records, _mismatch, _mx_exact_ref, _panel_records,
                               tile_coords)

pytestmark = pytest.mark.gpu

ENGINE_CTAS = 32          # the engine bench.py runs beside the fused GEMM
SMALL_GRID = 13           # odd: the pair kernels round it down to 6 CTAs (3 units)
WS_SLOTS = 80             # stream-K workspace slots (gemm_send.cu kWsSlots)


# ------------------------------------------------------------------ schedule model of both kernels
class Schedule:
    """One launch of K4 (`gemm_send.cu`) or K7 (`gemm_mxfp8.cu`) as the host launches it and the tile loop walks it:
    grid clamp (<= SMs), pair rounding (grid & ~1, <= 2 * tiles), n_units = grid / CTAs, unit u runs tiles u,
    u + n_units, ...; K4's cta_group 3 with stream-K splits the last partial wave along K (`StreamK`).  Every unit's
    producer and consumers advance one ring stage per k-block, so a segment starts at stage (k-blocks before it) % STAGES.
    `units[u]` lists unit u's segments (tile, kb0, kb1) in order."""

    def __init__(self, kernel, M, N, K, cta_group, grid=0, stream_k=False, group_m=1, sms=H100_SMS):
        assert kernel in ("k4", "k7")
        if grid <= 0 or grid > sms:
            grid = sms
        self.kernel, self.M, self.N, self.K, self.group_m = kernel, M, N, K, group_m
        if kernel == "k4":
            bm, bn, bk, self.stages = 128, 256, 64, 3
            two = cta_group in (2, 3) and grid >= 2
        else:
            bm, bn, bk, self.stages = 128, 128, 128, 4
            two = (cta_group == 2 or (cta_group == 0 and M > bm)) and grid >= 2
        self.ctas = 2 if two else 1
        self.m_tiles, self.n_blks, self.k_blks = -(-M // (self.ctas * bm)), -(-N // bn), -(-K // bk)
        self.n_tiles = self.m_tiles * self.n_blks
        if two:
            grid &= ~1
            grid = min(grid, 2 * self.n_tiles)
        else:
            grid = min(grid, self.n_tiles)
        self.grid, self.n_units = grid, grid // self.ctas
        W, R = divmod(self.n_tiles, self.n_units)
        self.stream_k = (kernel == "k4" and cta_group == 3 and two and stream_k and R != 0 and self.n_units <= WS_SLOTS)
        self.units = [[(w * self.n_units + u, 0, self.k_blks) for w in range(W)] for u in range(self.n_units)]
        if self.stream_k:
            self.sk = StreamK(M, N, K, grid, group_m, sms=sms, ws_slots=WS_SLOTS)
            assert self.sk.stream_k and self.sk.n_units == self.n_units
            for u, j, kb0, kb1 in self.sk.segs:
                self.units[u].append((W * self.n_units + j, kb0, kb1))
        else:
            for u in range(R):
                self.units[u].append((W * self.n_units + u, 0, self.k_blks))

    def coords(self, tile):
        """(m tile, n block) of a tile: grouped rasterisation in K4, row-major in K7."""
        if self.kernel == "k4":
            return tile_coords(tile, self.m_tiles, self.n_blks, self.group_m)
        return divmod(tile, self.n_blks)

    def entry_stages(self):
        """Ring stage at which each segment after a unit's first starts."""
        out = []
        for segs in self.units:
            kbs = 0
            for i, (_, kb0, kb1) in enumerate(segs):
                if i:
                    out.append(kbs % self.stages)
                kbs += kb1 - kb0
        return out

    def max_tiles_per_unit(self):
        return max(len(s) for s in self.units)

    def panel_done_slots(self):
        """Panel -> (slot, unit) of the segment that completes it (a tile's owner segment: kb0 == 0), where slot is the
        segment's position in its unit's list: units run their segments side by side, slot by slot."""
        panels = -(-self.M // 128)
        done = {}
        for u, segs in enumerate(self.units):
            for slot, (tile, kb0, _) in enumerate(segs):
                if kb0 != 0:
                    continue
                mt, _ = self.coords(tile)
                for r in range(self.ctas):
                    p = mt * self.ctas + r
                    if p < panels and (p not in done or slot > done[p][0]):
                        done[p] = (slot, u)
        assert sorted(done) == list(range(panels))
        return done

    def panels_race(self):
        """Adjacent panels whose last tiles run in the same slot on different units (or in one pair tile): the schedule
        leaves the order they complete, and are posted, in to run time."""
        d = self.panel_done_slots()
        return any(d[p + 1][0] <= d[p][0] for p in range(len(d) - 1))

    def facts(self):
        return {"max_tiles_per_unit": self.max_tiles_per_unit(), "mid_ring_entry": any(s != 0 for s in self.entry_stages()),
                "stream_k": self.stream_k}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid(token, sms):
    return {"default": 0, "beside_engine": sms - ENGINE_CTAS, "small": SMALL_GRID}[token]


# ------------------------------------------------------------------ exact operands at scale (generated on the GPU)
_CACHE = {}


@pytest.fixture(autouse=True, scope="module")
def _release_operands():
    """Return the cached operands' memory before later modules run (some of them free and reallocate device memory)."""
    yield
    _CACHE.clear()
    torch.cuda.empty_cache()


def _cached(key, make):
    """One shape's operands and reference at a time: the cases of a shape run next to each other."""
    if key not in _CACHE:
        _CACHE.clear()
        torch.cuda.empty_cache()
        _CACHE[key] = make()
    return _CACHE[key]


def _sparse_positions(rows, K, nnz, g):
    """nnz distinct k positions per row, one in each K // nnz wide window."""
    s = K // nnz
    return torch.arange(nnz, device="cuda") * s + torch.randint(0, s, (rows, nnz), device="cuda", generator=g)


def _k4_operands(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    nnz = min(K, 128)
    a = torch.zeros(M, K, device="cuda")
    idx = _sparse_positions(M, K, nnz, g)
    a.scatter_(1, idx, torch.randint(-1, 5, (M, nnz), device="cuda", generator=g).float())
    a[0].scatter_(0, idx[0], torch.full((nnz,), 4.0, device="cuda"))        # row 0 x row 0 reaches 128 * 16 = 2048
    b = torch.randint(-1, 5, (N, K), device="cuda", generator=g).float()
    b[0] = 4.0
    a, b = a.to(torch.bfloat16), b.to(torch.bfloat16)
    # S = |A| @ |B|^T <= (nonzeros of a row of A) * max|a| * max|b|
    bound = (a != 0).sum(1).max().item() * a.abs().max().item() * b.abs().max().item()
    assert bound <= 2 ** 11, "operands too large for order-independent fp32 accumulation"
    exact = a.double() @ b.double().T
    assert exact[0, 0].item() == 2048.0
    return a, b, exact


def _assert_schedule(sch, token):
    f = sch.facts()
    assert f["mid_ring_entry"], f"no tile enters the ring at a nonzero stage: {f}"
    if token == "small":
        assert f["max_tiles_per_unit"] >= 8, f
    else:
        assert f["max_tiles_per_unit"] >= 2, f
    return f


BENCH_SHAPES = [(4096, 4096, 4096), (8192, 8192, 2048), (16384, 4096, 1024), (8192, 8192, 8192)]
# k_blks = 16 (K tail of 40) and 17: a unit's second tile enters the 3-stage ring at stage 1 and at stage 2
RING_SHAPES = [(4096, 4096, 1000), (4096, 4096, 1088)]
K4_SCALE_CASES = ([(s, cg, gt) for s in BENCH_SHAPES for cg in (1, 2, 3) for gt in ("default", "beside_engine", "small")] +
                  [(s, cg, "small") for s in RING_SHAPES for cg in (1, 2, 3)])


@pytest.mark.parametrize("shape,cta_group,grid_token", K4_SCALE_CASES,
                         ids=[f"{m}x{n}x{k}-cg{cg}-{gt}" for (m, n, k), cg, gt in K4_SCALE_CASES])
def test_k4_exact_at_scale(ctx, shape, cta_group, grid_token):
    M, N, K = shape
    sms = _sms()
    grid = _grid(grid_token, sms)
    stream_k = cta_group == 3
    sch = Schedule("k4", M, N, K, cta_group, grid, stream_k=stream_k, group_m=8, sms=sms)
    _assert_schedule(sch, grid_token)
    a, b, exact = _cached(("k4", M, N, K), lambda: _k4_operands(M, N, K))
    ref = exact.to(torch.bfloat16)
    guard = N + 8                                   # guard rows' worth in front of C and behind it, 16-byte aligned
    buf = torch.full((M * N + 2 * guard,), 7.0, device="cuda", dtype=torch.bfloat16)
    c = buf[guard:guard + M * N].view(M, N)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=cta_group, grid=grid, stream_k=stream_k)
    assert r.ok, r.status
    assert r.variant == cta_group and r.stream_k == sch.stream_k, (r.variant, r.stream_k, sch.facts())
    assert _bits_equal(c, ref), _mismatch(c, ref)
    assert torch.all(buf[:guard] == 7.0) and torch.all(buf[guard + M * N:] == 7.0), "stored outside C"


def _send_setup(ctx, M, N, out_fp8):
    if out_fp8:
        nb = -(-M // 128) * ops.panel_record_bytes(N)
        c = torch.full((nb + 4096,), 0xAB, dtype=torch.uint8, device="cuda")
        d = torch.full((nb + 4096,), 0xCD, dtype=torch.uint8, device="cuda")
    else:
        c = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        d = torch.full((M + 16, N), 3.0, device="cuda", dtype=torch.bfloat16)
    return c, d


@pytest.mark.parametrize("out_fp8", [False, True], ids=["bf16", "fp8"])
def test_k4_fused_send_at_bench_shape_exact(ctx, out_fp8):
    """What bench.py's fused extra does at 8192 x 8192 x 2048: a loopback QP, 32 engine CTAs, signal_every=4 and the
    GEMM on the SMs the engine leaves.  Every panel posted once, the destination equal to the source bit for bit."""
    M, N, K = 8192, 8192, 2048
    sms = _sms()
    grid = sms - ENGINE_CTAS
    sch = Schedule("k4", M, N, K, 2, grid, group_m=4, sms=sms)
    _assert_schedule(sch, "beside_engine")
    assert sch.panels_race(), "every panel's completion is ordered by the schedule"
    a, b, exact = _cached(("k4", M, N, K), lambda: _k4_operands(M, N, K))
    c, d = _send_setup(ctx, M, N, out_fp8)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp()
    panels = M // 128
    torch.cuda.synchronize()
    ctx.engine_start(ctas=ENGINE_CTAS, idle_timeout_ms=5000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, signal_every=4, grid=grid, out_fp8=out_fp8)
    finally:
        ctx.engine_stop()
    assert ctx.last_engine_fatal == 0, "the engine did not exit cleanly"
    assert r.ok and r.variant == 2, (r.status, r.variant)
    assert r.panels_posted == panels, r.panels_posted
    cnt = qp.counters()
    assert cnt["n_wqe"] == panels + 1 and cnt["n_err"] == 0 and cnt["n_db_order_violations"] == 0, cnt
    if out_fp8:
        nb = panels * ops.panel_record_bytes(N)
        ref = ops.ref_fp8_panels(exact.float())
        assert torch.equal(c[:nb], ref), f"{int((c[:nb] != ref).sum())} record bytes differ at the sender"
        assert torch.equal(d[:nb], ref), f"{int((d[:nb] != ref).sum())} record bytes differ at the destination"
        assert torch.all(c[nb:] == 0xAB) and torch.all(d[nb:] == 0xCD), "stored beyond the last record"
    else:
        ref = exact.to(torch.bfloat16)
        assert _bits_equal(c, ref), _mismatch(c, ref)
        assert _bits_equal(d[:M], c), _mismatch(d[:M], c)
        assert torch.all(d[M:] == 3.0), "written beyond the destination rows"


# ------------------------------------------------------------------ K7 at scale
def _mx_sparse_operand(rows, K, g, nnz):
    """e4m3 codes of integers in [-4, 4] on `nnz` positions per row (all of them when nnz >= K), scale bytes 127 +- 3."""
    if nnz >= K:
        v = torch.randint(-4, 5, (rows, K), device="cuda", generator=g).float()
    else:
        v = torch.zeros(rows, K, device="cuda")
        v.scatter_(1, _sparse_positions(rows, K, nnz, g), torch.randint(-4, 5, (rows, nnz), device="cuda", generator=g).float())
    q = v.to(torch.float8_e4m3fn).view(torch.uint8)
    s = torch.randint(124, 131, (rows, K // 32), device="cuda", generator=g).to(torch.uint8)
    return q, s


def _k7_operands(M, N, K):
    """A sparse (128 nonzeros per row) against a dense B: S stays below 2^24 of the smallest scale product's quantum, the
    bound _mx_exact_ref asserts, at any K."""
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + K)
    aq, as_ = _mx_sparse_operand(M, K, g, 128)
    bq, bs = _mx_sparse_operand(N, K, g, K)
    return aq, as_, bq, bs, _mx_exact_ref(aq, as_, bq, bs)


def _k7_operand(kind, q, s):
    rows, K = q.shape
    if kind == "plain":
        return MX.MxOperand.from_tensors(q, s), None
    if kind == "panel":
        rec = _panel_records(q, s)
        return MX.MxOperand.from_panel_records(rec, rows, K), rec
    chunk = 128 * K * 2
    rec = _chunk_records(q, s, chunk)
    return MX.MxOperand.from_chunk_records(rec, rows, K, chunk), rec


# k_blks = 9 and 11: a unit's second tile enters the 4-stage ring at stage 1 and at stage 3
K7_SCALE_CASES = [(kind, shape, cg, gt) for cg in (1, 2) for kind, shape, gt in [
    ("plain", (4096, 4096, 4096), "default"), ("panel", (4096, 4096, 4096), "beside_engine"), ("chunk", (4096, 4096, 4096), "small"),
    ("plain", (8192, 8192, 2048), "small"), ("panel", (8192, 8192, 2048), "default"), ("chunk", (8192, 8192, 2048), "beside_engine"),
    ("plain", (4096, 4096, 1152), "small"), ("panel", (4096, 4096, 1408), "beside_engine")]]


@pytest.mark.parametrize("kind,shape,cta_group,grid_token", K7_SCALE_CASES,
                         ids=[f"{kd}-{m}x{n}x{k}-cg{cg}-{gt}" for kd, (m, n, k), cg, gt in K7_SCALE_CASES])
def test_k7_exact_at_scale(ctx, kind, shape, cta_group, grid_token):
    M, N, K = shape
    sms = _sms()
    grid = _grid(grid_token, sms)
    sch = Schedule("k7", M, N, K, cta_group, grid, sms=sms)
    f = sch.facts()
    if K % (128 * 4):
        assert f["mid_ring_entry"], f
    else:
        assert not f["mid_ring_entry"], f                    # k_blks % 4 == 0: every tile enters the ring at stage 0
    assert f["max_tiles_per_unit"] >= (8 if grid_token in ("small", "default") else 2), f
    aq, as_, bq, bs, ref = _cached(("k7", M, N, K), lambda: _k7_operands(M, N, K))
    oa, keep = _k7_operand(kind, aq, as_)
    pad = torch.full((M + 2, N), 7.0, device="cuda", dtype=torch.bfloat16)
    c = pad[:M]
    torch.cuda.synchronize()
    r = ops.gemm_mxfp8(ctx, oa, MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group, grid=grid)
    assert r.ok and r.variant == cta_group, (r.status, r.variant)
    assert _bits_equal(c, ref), _mismatch(c, ref)
    assert torch.all(pad[M:] == 7.0), "the epilogue wrote past the last row"
    del keep


def test_k7_gated_records_already_landed_at_scale(ctx):
    """Receive-side fusion's gate with every arrival word already set: no tile is lost or repeated at 4096^3."""
    M, N, K = 4096, 4096, 4096
    sms = _sms()
    grid = sms - ENGINE_CTAS
    aq, as_, bq, bs, ref = _cached(("k7", M, N, K), lambda: _k7_operands(M, N, K))
    oa, rec = _k7_operand("panel", aq, as_)
    ready = torch.ones(M // 128, dtype=torch.int64, device="cuda")
    c = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_mxfp8(ctx, oa, MX.MxOperand.from_tensors(bq, bs), c, cta_group=2, grid=grid, a_ready=ready)
    assert r.ok, r.status
    assert _bits_equal(c, ref), _mismatch(c, ref)
    del rec


# ------------------------------------------------------------------ K4 epilogues at their edges
BIG, TINY = 2.0 ** 100, 2.0 ** -70
HUGE_BLOCK, TINY_BLOCK = 6, 7          # output column blocks whose B factors are 2^100 and 2^-70; the others have 1
FP32_MAX = torch.finfo(torch.float32).max
BF16_MAX = torch.finfo(torch.bfloat16).max


def _pairs(*vals):
    """A 32-column block of (first product, second product): a bare number is (v, 0); the rest of the block is 0."""
    out = [v if isinstance(v, tuple) else (v, 0.0) for v in vals]
    assert len(out) <= 32
    return out + [(0.0, 0.0)] * (32 - len(out))


def _scale0(*vals):
    """A block whose amax 256 gives the UE8M0 scale 2^0, then `vals`."""
    return _pairs(256.0, *vals)


N18 = 2.0 ** -18
# Finite classes on the columns whose B factors are 1.  Every sum is exact in fp32 (asserted).
FINITE_BLOCKS = [
    _pairs(),                                                                                      # all zero: scale byte 0
    _pairs(1792.0, *[1.0] * 31),                                                                   # amax 448 * 2^2 exactly
    _pairs((1792.0, 2.0 ** -13), *[1.0] * 31),                                                     # the next fp32 above it
    _pairs(448.0 * 2.0 ** -10, -448.0 * 2.0 ** -10, *[2.0 ** -12] * 30),                          # 448 * 2^-10: scale 2^-10
    # e4m3 ties at scale 2^0: 17 (16 | 18), 19 (18 | 20), -17, 1.0625, 1.1875, 2.125, -9.5, 304 (288 | 320), 200, -27
    _scale0(17.0, 19.0, -17.0, 1.0625, 1.1875, 2.125, -9.5, 304.0, 200.0, -27.0),
    # the same ties nudged by 2^-18 (2^-14 at 304 and 200, where fp32 has no bit at 2^-18), far below bf16 precision:
    # each must leave the tie
    _scale0((17.0, N18), (19.0, -N18), (-17.0, -N18), (1.0625, N18), (1.1875, -N18), (2.125, N18), (-9.5, N18),
            (304.0, 2.0 ** -14), (200.0, -(2.0 ** -14)), (-27.0, N18)),
    # e4m3 subnormals at scale 2^0 (k * 2^-9) and ties among them, values that round to +-0, and nudged subnormal ties
    _scale0(2.0 ** -7, 3 * 2.0 ** -10, 2.0 ** -10, 5 * 2.0 ** -10, 7 * 2.0 ** -10, 2.0 ** -11, -(2.0 ** -9), -(2.0 ** -11),
            -(2.0 ** -10), -(3 * 2.0 ** -10), 2.0 ** -20, (2.0 ** -10, N18), (3 * 2.0 ** -10, -N18), (-(2.0 ** -10), -N18)),
    # bf16 ties and the same a few bits past them: 1 + 2^-8 (-> 1), + 2^-15 (-> 1 + 2^-7), - 2^-15 (-> 1),
    # 1 + 2^-7 + 2^-8 (-> 1 + 2^-6), 257 (-> 256), 259 (-> 260), 2^20 + 2^12 (-> 2^20) and + 2^5 (-> 2^20 + 2^13)
    _pairs((1.0, 2.0 ** -8), (1.0, 2.0 ** -8 + 2.0 ** -15), (1.0, 2.0 ** -8 - 2.0 ** -15), (1.0 + 2.0 ** -7, 2.0 ** -8),
           (256.0, 1.0), (258.0, 1.0), (2.0 ** 20, 2.0 ** 12), (2.0 ** 20, 2.0 ** 12 + 2.0 ** 5), (-1.0, -(2.0 ** -8) - 2.0 ** -15),
           (3.0, 2.0 ** -7), (3.0, 2.0 ** -7 + 2.0 ** -14)),
]
# Classes on the 2^100 columns (written as the product's value): finite values near fp32 max.  1.99609375 * 2^127 is a
# bf16 tie that rounds to 2^128 = Inf; 1.99997 * 2^127 is the largest sum of two bf16 products below fp32 max.
NEAR_MAX = _pairs(BF16_MAX, (BF16_MAX, 2.0 ** 119), (-BF16_MAX, -(2.0 ** 119)), (BF16_MAX, BF16_MAX * 2.0 ** -8), 1.5 * 2.0 ** 127,
                  (2.0 ** 127, 2.0 ** 120), 3.0 * 2.0 ** 100, -(2.0 ** 101))
ORDINARY = _pairs(*[float(v) for v in range(-7, 25)])
# Classes whose result depends on the hardware's IEEE behaviour (each in a row of its own)
INF = float("inf")
NONFINITE_HUGE = _pairs((BIG * BIG, 0.0), (0.0, -BIG * BIG), (BIG * BIG, -BIG * BIG), (BF16_MAX, BF16_MAX), 5.0 * 2.0 ** 100)
SUBNORMAL_TINY = _pairs(*[(c * 2.0 ** -140, d * 2.0 ** -140) for c, d in
                          [(1, 0), (64, 0), (128, 0), (192, 0), (64, 128), (255, 1), (3 * 2 ** 12, 0), (2 ** 11, 2 ** 11 + 2 ** 4),
                           (-192, 0), (-64, -1), (96, 32), (200, 55)]])


def _row_kinds():
    """Row kinds: (name, per-column-block classes, IEEE-dependent).  Blocks HUGE_BLOCK and TINY_BLOCK hold values of the
    2^100 / 2^-70 columns."""
    fin = FINITE_BLOCKS
    kinds = []
    for i in range(len(fin)):
        blocks = [fin[(i + j) % len(fin)] for j in range(16)]
        blocks[HUGE_BLOCK] = NEAR_MAX if i % 2 == 0 else ORDINARY
        blocks[TINY_BLOCK] = ORDINARY
        kinds.append(("finite", blocks, False))
    nonfin = [ORDINARY] * 16
    nonfin[HUGE_BLOCK], nonfin[TINY_BLOCK] = NONFINITE_HUGE, SUBNORMAL_TINY
    kinds.append(("inf_nan_subnormal", nonfin, True))
    neg = [_pairs(*[(-0.0, -0.0)] * 31, (-1.5, -0.0))] * 16            # every A entry of the row <= -0: -0 sums
    kinds.append(("negative_zero", neg, True))
    kinds.append(("nan_row", None, True))
    return kinds


ROW_KINDS = _row_kinds()


def _edge_operands(M, N):
    """A [M, 2N], B [N, 2N] bf16 with B[n, n] = B[n, N + n] = the column's power of two and zeros elsewhere: output (m, n)
    is p1 + p2 with p1 = A[m, n] * B[n, n] (k-block n // 64) and p2 = A[m, N + n] * B[n, N + n] (k-block (N + n) // 64,
    always a later one).  Returns a, b, p1, p2 (fp64, NaN in the NaN rows) and a per-row flag for the rows whose values
    depend on the hardware's Inf / NaN / subnormal / -0 behaviour."""
    assert N % 32 == 0 and N >= 256
    K = 2 * N
    col_scale = torch.ones(N, dtype=torch.float64)
    col_scale[HUGE_BLOCK * 32:(HUGE_BLOCK + 1) * 32] = BIG
    col_scale[TINY_BLOCK * 32:(TINY_BLOCK + 1) * 32] = TINY
    p1 = torch.zeros(M, N, dtype=torch.float64)
    p2 = torch.zeros(M, N, dtype=torch.float64)
    ieee = torch.zeros(M, dtype=torch.bool)
    nan_rows = []
    for m in range(M):
        name, blocks, dep = ROW_KINDS[m % len(ROW_KINDS)]
        ieee[m] = dep
        if blocks is None:
            nan_rows.append(m)
            continue
        for blk in range(N // 32):
            cls = blocks[blk % len(blocks)]
            if blk not in (HUGE_BLOCK, TINY_BLOCK) and cls in (NEAR_MAX, NONFINITE_HUGE, SUBNORMAL_TINY):
                cls = ORDINARY
            if blk == TINY_BLOCK and cls is NEAR_MAX:
                cls = ORDINARY
            p1[m, blk * 32:(blk + 1) * 32] = torch.tensor([v[0] for v in cls], dtype=torch.float64)
            p2[m, blk * 32:(blk + 1) * 32] = torch.tensor([v[1] for v in cls], dtype=torch.float64)
    a64 = torch.cat([p1 / col_scale, p2 / col_scale], dim=1)
    a = a64.to(torch.bfloat16)
    assert torch.equal(a.double(), a64), "an operand value is not a bf16"
    a[nan_rows] = float("nan")
    b = torch.zeros(N, K, dtype=torch.float64)
    idx = torch.arange(N)
    b[idx, idx] = col_scale
    b[idx, N + idx] = col_scale
    b = b.to(torch.bfloat16)
    assert torch.equal(b.double().diagonal(), col_scale)
    exact = p1 + p2
    fin = torch.isfinite(exact.float())
    assert torch.equal(exact.float()[fin].double(), exact[fin]), "an output is not exact in fp32"
    assert torch.isfinite(exact.float()[~ieee]).all() and (exact[~ieee].float().abs() >= 2.0 ** -126).logical_or(exact[~ieee] == 0).all()
    # the same through an fp64 GEMM of the finite rows: no other product contributes
    rows = ~ieee
    assert torch.equal(a[rows].double() @ b.double().T, exact[rows])
    p1[nan_rows] = float("nan")
    p2[nan_rows] = float("nan")
    return a, b, p1, p2, ieee


def _wgmma_accumulator(p1, p2, split):
    """fp32 value K4's accumulator holds for p1 + p2, as wgmma on an H100 gives it (DESIGN.md, fp8 numerics): each k-block's
    products join the fp32 accumulator before they are rounded (so +Inf stays +Inf when a later product of -2^200 comes),
    a stream-K partial is rounded to fp32 before the epilogue adds it (Inf + -Inf = NaN there), subnormals are kept and a
    zero sum is +0.  Where every value is finite and nonzero this is the exact sum."""
    first = p1.float()
    whole = (first.double() + p2).float()
    folded = first + p2.float()
    w = torch.where(split, folded, whole)
    w[w == 0] = 0.0
    return w


def _check_bf16(c, want, rows, label):
    got, ref = c[rows], want[rows].to(torch.bfloat16)
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), f"{label}: NaN at different positions"
    g, r = got.view(torch.int16)[~nan], ref.view(torch.int16)[~nan]
    bad = (g != r).nonzero()
    assert bad.numel() == 0, (f"{label}: {bad.numel()} bf16 outputs differ, first got {got[~nan][bad[0, 0]].item()} "
                              f"want {ref[~nan][bad[0, 0]].item()}")


def _check_records(rec, want, rows, N, label):
    """Rows `rows` of the records equal ref_fp8_panels(want) byte for byte; NaN codes compared without their sign."""
    M = want.shape[0]
    P_ = -(-M // 128)
    ref = ops.ref_fp8_panels(want).reshape(P_, -1)
    got = rec[:P_ * ops.panel_record_bytes(N)].reshape(P_, -1)
    pad = P_ * 128 - M
    rmask = torch.cat([rows, torch.ones(pad, dtype=torch.bool, device=rows.device)])      # zero rows past M: always checked
    gq, rq = got[:, :128 * N].reshape(-1, N)[rmask], ref[:, :128 * N].reshape(-1, N)[rmask]
    gs, rs = got[:, 128 * N:].reshape(-1, N // 32)[rmask], ref[:, 128 * N:].reshape(-1, N // 32)[rmask]
    nan = (rq & 0x7F) == 0x7F
    assert torch.equal((gq & 0x7F) == 0x7F, nan), f"{label}: NaN codes at different positions"
    bad = (gq != rq) & ~nan
    assert not bad.any(), f"{label}: {int(bad.sum())} fp8 codes differ, first at {bad.nonzero()[0].tolist()}"
    bad = gs != rs
    assert not bad.any(), f"{label}: {int(bad.sum())} scale bytes differ, first at {bad.nonzero()[0].tolist()}"


# (M, N, cta_group, grid, stream_k): tile-aligned, ragged (edge tiles zero-filled), and a stream-K split of a tile
# holding edge blocks (700 rows: three pair tiles on two units, the third split along K between them)
EDGE_CASES = [(256, 256, 1, 0, False), (256, 256, 2, 0, False), (256, 256, 3, 0, False),
              (200, 288, 1, 0, False), (300, 288, 2, 0, False), (330, 320, 3, 0, False),
              (700, 256, 3, 4, True)]
EDGE_IDS = [f"{m}x{n}-cg{cg}" + (f"-g{g}-streamk" if sk else "") for m, n, cg, g, sk in EDGE_CASES]


def _edge_run(ctx, M, N, cta_group, grid, stream_k):
    a, b, p1, p2, ieee = _edge_operands(M, N)
    K = 2 * N
    split = torch.zeros(M, N, dtype=torch.bool)
    if stream_k:
        m = StreamK(M, N, K, grid, 1)
        assert m.stream_k and m.split_tiles(), "no tile is split"
        for j, segs in m.split_tiles().items():       # p1 and p2 of every output of the tile on different CTA pairs
            assert [(kb0, kb1) for _, _, kb0, kb1 in segs] == [(0, N // 64), (N // 64, K // 64)], segs
            mt, n = m.coords(j)
            split[mt * 256:(mt + 1) * 256, n * 256:(n + 1) * 256] = True
    want = _wgmma_accumulator(p1, p2, split)
    exact = (p1 + p2)[~ieee].float()
    assert torch.equal(want[~ieee], exact) and not torch.signbit(exact[exact == 0]).any()   # finite rows: the exact sum
    a, b, want, ieee = a.cuda(), b.cuda(), want.cuda(), ieee.cuda()
    kw = dict(cta_group=cta_group, grid=grid, stream_k=stream_k, group_m=1)
    out = {}
    c = torch.full((M + 2, N), 7.0, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c[:M], **kw)
    assert r.ok and r.stream_k == stream_k, (r.status, r.stream_k)
    assert torch.all(c[M:] == 7.0), "stored past the last row"
    out["bf16"] = c[:M]
    if M % 128 == 0 and N % 256 == 0:
        cp = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        assert ops.gemm_send(ctx, a, b, cp, plain_stores=True, **kw).ok
        out["plain_stores"] = cp
    nb = -(-M // 128) * ops.panel_record_bytes(N)
    rec = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert ops.gemm_send(ctx, a, b, rec, out_fp8=True, **kw).ok
    assert torch.all(rec[nb:] == 0xAB), "stored beyond the last record"
    out["fp8"] = rec
    return want, ieee, out


def _check_edge(want, ieee, out, N, rows, label):
    for k, v in out.items():
        if k == "fp8":
            _check_records(v, want, rows, N, f"{label} fp8")
        else:
            _check_bf16(v, want, rows, f"{label} {k}")


@pytest.mark.parametrize("M,N,cta_group,grid,stream_k", EDGE_CASES, ids=EDGE_IDS)
def test_k4_epilogues_finite_edges(ctx, M, N, cta_group, grid, stream_k):
    """bf16 (staged TMA and plain stores) and fp8 records of the finite classes, bit for bit."""
    want, ieee, out = _edge_run(ctx, M, N, cta_group, grid, stream_k)
    _check_edge(want, ieee, out, N, ~ieee, "finite rows")


@pytest.mark.parametrize("M,N,cta_group,grid,stream_k", EDGE_CASES, ids=EDGE_IDS)
def test_k4_epilogues_wgmma_nonfinite_subnormal_zero(ctx, M, N, cta_group, grid, stream_k):
    """The rows whose values rest on what wgmma does outside finite normal fp32 (`_wgmma_accumulator`, observed on an
    H100): products overflowing to +-Inf, +Inf followed by a -2^200 product (Inf; NaN across a stream-K fold), sums that
    overflow, a NaN row of A (every output of the row NaN), fp32 subnormal products and sums, and sums of -0 products.
    Both epilogues must then round, and quantise, whatever the accumulator holds exactly as the references do."""
    want, ieee, out = _edge_run(ctx, M, N, cta_group, grid, stream_k)
    _check_edge(want, ieee, out, N, ieee, "non-finite / subnormal / zero rows")
