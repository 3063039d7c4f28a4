"""Numerics of the compute kernels against fp64 references.

* Exact arithmetic: integer operands small enough that every partial sum the tensor core and the fp32 accumulator form
  is an exact integer (or an exact multiple of the smallest block scale), so the result is independent of summation
  order and the kernel's bf16 output must equal the round-to-nearest-even of the fp64 product bit for bit.  The
  precondition is asserted in each test: S = |A| @ |B|^T (fp64) stays <= 2^11 for K4, so exactness does not depend on
  how wide the tensor core's internal alignment is.  This covers K4 (1-CTA, CTA pair, pair + stream-K, bf16 and fp8
  epilogues) and K7 (block-scaled fp8, plain operands and records).
* Floating-point data: a per-element bound |c - r| <= 2^-8 |r| + gamma * S against fp64, with the operands scaled per
  row, per column and per k-block by powers of two over 2^+-20 and rows that cancel, so an error that is wrong
  relative to its own row or block fails.
* The fp8 pack / unpack kernels at their edges (subnormals, ties, bf16 max, NaN, +-Inf, scale bytes 0x00 / 0xFF) and on
  the chunk sizes and grids that run every path of their tile loops.

The stream-K schedule model at the top mirrors gemm_send.cu; test_numerics_references.py checks it on the CPU."""
import ctypes as C

import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import gemm_mx as MX
from rocnrdma_b200.ops import pack as P

pytestmark = pytest.mark.gpu

H100_SMS = 132


# ------------------------------------------------------------------ stream-K schedule model (gemm_send.cu, gemm_tile_body)
def tile_coords(t, m_blks, n_blks, group_m):
    per_group = group_m * n_blks
    grp, r = divmod(t, per_group)
    m0 = grp * group_m
    gm = min(group_m, m_blks - m0)
    return m0 + r % gm, r // gm


class StreamK:
    """The schedule of the CTA-pair kernel with the stream-K tail (cta_group=3, stream_k=True) for one launch:
    W whole waves round robin, then the R = n_tiles % n_units tail tiles split into R * k_blks (tile, k-block) units
    dealt out evenly to the first n_tail clusters.  `segs` lists (unit, tail tile j, kb0, kb1) in schedule order."""

    def __init__(self, M, N, K, grid, group_m, sms=H100_SMS, ws_slots=80):
        if grid <= 0 or grid > sms:
            grid = sms
        self.requested_grid = grid
        self.m_tiles, self.n_blks, self.k_blks = -(-M // 256), -(-N // 256), -(-K // 64)
        self.M, self.N, self.K, self.group_m = M, N, K, group_m
        self.n_tiles = self.m_tiles * self.n_blks
        grid &= ~1
        grid = min(grid, 2 * self.n_tiles)
        self.grid, self.n_units = grid, grid // 2
        self.W, self.R = divmod(self.n_tiles, self.n_units)
        self.stream_k = self.R != 0 and self.n_units <= ws_slots
        self.tail_units = self.R * self.k_blks
        n_tail = self.n_units
        if self.tail_units // 4 < n_tail:
            n_tail = self.tail_units // 4
        if n_tail < self.R:
            n_tail = self.R
        self.n_tail = n_tail
        self.segs = []
        if self.stream_k:
            for u in range(n_tail):
                x, end = self.share(u)
                while x < end:
                    j, kb0 = divmod(x, self.k_blks)
                    kb1 = min(kb0 + end - x, self.k_blks)
                    self.segs.append((u, j, kb0, kb1))
                    x += kb1 - kb0

    def share(self, u):
        return self.tail_units * u // self.n_tail, self.tail_units * (u + 1) // self.n_tail

    def unit_of(self, x):
        """Unit that holds tail unit x (largest c with tail_units * c / n_tail <= x), as the kernel computes it."""
        c = x * self.n_tail // self.tail_units + 1
        c = min(c, self.n_tail - 1)
        while self.tail_units * c // self.n_tail > x:
            c -= 1
        return c

    def n_contrib(self, u, j, kb0, kb1):
        """Partials the owner segment (kb0 == 0) folds, as the kernel computes it."""
        if kb1 == self.k_blks:
            return 0
        return self.unit_of((j + 1) * self.k_blks - 1) - u

    def tiles(self):
        """tail tile j -> its segments."""
        out = {}
        for s in self.segs:
            out.setdefault(s[1], []).append(s)
        return out

    def split_tiles(self):
        return {j: v for j, v in self.tiles().items() if len(v) > 1}

    def coords(self, j):
        return tile_coords(self.W * self.n_units + j, self.m_tiles, self.n_blks, self.group_m)

    def hangs(self, j):
        mt, n = self.coords(j)
        return (mt + 1) * 256 > self.M, (n + 1) * 256 > self.N

    def facts(self):
        f = set()
        k_tail = self.K % 64 != 0
        for j, segs in self.split_tiles().items():
            f.add("split")
            om, on = self.hangs(j)
            f.add({(True, True): "over_mn", (True, False): "over_m", (False, True): "over_n", (False, False): "inside"}[(om, on)])
            owner = [s for s in segs if s[2] == 0][0]
            if self.n_contrib(*owner) >= 2:
                f.add("folds_2_or_more")
            if k_tail and any(s[2] == self.k_blks - 1 and s[3] == self.k_blks for s in segs if s[2] != 0):
                f.add("contrib_only_k_tail")
        if self.requested_grid % 2:
            f.add("odd_grid")
        return f


# (M, N, K, grid, group_m) and what the model says each case exercises
STREAM_K_CASES = [
    ((520, 776, 328, 15, 1), {"split", "over_m", "over_n", "over_mn", "contrib_only_k_tail", "odd_grid"}),
    ((520, 776, 1000, 15, 3), {"split", "over_m", "over_n", "over_mn", "folds_2_or_more", "odd_grid"}),
    ((520, 520, 1000, 15, 16), {"split", "over_mn", "folds_2_or_more", "odd_grid"}),
    ((300, 1056, 1000, 15, 3), {"split", "over_m", "over_n", "over_mn", "folds_2_or_more", "odd_grid"}),   # N % 32 == 0: fp8 output
]


# ------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _sparse_int(rows, K, nnz, lo, hi, g):
    """rows x K integers in [lo, hi] on `nnz` random positions per row, zeros elsewhere."""
    x = torch.zeros(rows, K)
    idx = torch.argsort(torch.rand(rows, K, generator=g), dim=1)[:, :nnz]
    x.scatter_(1, idx, torch.randint(lo, hi + 1, (rows, nnz), generator=g).float())
    return x


def _exact_operands(M, N, K, seed):
    """A sparse, B dense, entries in [-1, 4]: |products| <= 16 and at most 128 nonzero products per output, so
    S <= 2^11, while many results lie in [256, 2048] where bf16 rounds (odd integers in [256, 512) are ties).
    Row 0 x row 0 reaches exactly 128 * 16 = 2048."""
    g = _gen(seed)
    nnz = min(K, 128)
    a = _sparse_int(M, K, nnz, -1, 4, g)
    a[0][a[0] != 0] = 4.0
    b = torch.randint(-1, 5, (N, K), generator=g).float()
    b[0] = 4.0
    a, b = a.to(torch.bfloat16).cuda(), b.to(torch.bfloat16).cuda()
    S = a.double().abs() @ b.double().abs().T
    assert S.max().item() <= 2 ** 11, "operands too large for order-independent fp32 accumulation"
    exact = a.double() @ b.double().T
    return a, b, exact


def _bits_equal(x, y):
    return torch.equal(x.view(torch.int16), y.view(torch.int16))


def _mismatch(c, ref):
    d = (c.view(torch.int16) != ref.view(torch.int16)).nonzero()
    if d.numel() == 0:
        return ""
    i, j = d[0].tolist()
    return f"{d.shape[0]} elements differ, first at ({i}, {j}): got {c[i, j].item()}, want {ref[i, j].item()}"


# ------------------------------------------------------------------ K4: exact bf16 output
K4_SHAPES = [(100, 256, 64), (1000, 520, 328), (130, 8, 8), (384, 264, 72), (515, 1000, 4104), (257, 1032, 200),
             (300, 520, 136), (300, 520, 232), (300, 520, 120), (260, 264, 8)]    # K tails 8, 40, 56 past a 64 multiple; K = 8


@pytest.mark.parametrize("cta_group", [1, 2, 3])
@pytest.mark.parametrize("M,N,K", K4_SHAPES)
def test_k4_exact_integer_gemm_rounds_to_nearest_even(ctx, M, N, K, cta_group):
    a, b, exact = _exact_operands(M, N, K, seed=M * 7 + N * 3 + K)
    ref = exact.to(torch.bfloat16)
    buf = torch.full(((M + 2) * N + 64,), 7.0, device="cuda", dtype=torch.bfloat16)
    off = N + 8                                     # guard band in front of C, keeping the 16-byte alignment TMA needs
    c = buf[off:off + M * N].view(M, N)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=cta_group)
    assert r.ok, r.status
    assert _bits_equal(c, ref), _mismatch(c, ref)
    assert torch.all(buf[:off] == 7.0) and torch.all(buf[off + M * N:] == 7.0), "stored outside C"


@pytest.mark.parametrize("cta_group", [1, 2])
def test_k4_exact_plain_stores_epilogue(ctx, cta_group):
    """The per-thread row-store epilogue rounds the same way as the staged TMA one."""
    M, N, K = 512, 768, 4096
    a, b, exact = _exact_operands(M, N, K, seed=17 + cta_group)
    c = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_send(ctx, a, b, c, cta_group=cta_group, plain_stores=True).ok
    ref = exact.to(torch.bfloat16)
    assert _bits_equal(c, ref), _mismatch(c, ref)


# ------------------------------------------------------------------ K4: stream-K on ragged shapes, exact
@pytest.mark.parametrize("case,expect", STREAM_K_CASES, ids=[f"{m}x{n}x{k}-g{gr}-gm{gm}" for (m, n, k, gr, gm), _ in STREAM_K_CASES])
def test_k4_stream_k_ragged_exact(ctx, case, expect):
    M, N, K, grid, group_m = case
    assert grid <= torch.cuda.get_device_properties(0).multi_processor_count
    model = StreamK(M, N, K, grid, group_m)
    assert model.stream_k and expect <= model.facts(), (expect, model.facts())
    a, b, exact = _exact_operands(M, N, K, seed=M + N + K + grid)
    ref = exact.to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    for _ in range(2):                              # twice: the epoch-stamped flags need no reset between launches
        c.fill_(7.0)
        r = ops.gemm_send(ctx, a, b, c, cta_group=3, grid=grid, group_m=group_m, stream_k=True)
        assert r.ok and r.variant == 3 and r.stream_k, (r.status, r.variant, r.stream_k)
        assert _bits_equal(c, ref), _mismatch(c, ref)
    c2 = torch.zeros_like(c)
    r2 = ops.gemm_send(ctx, a, b, c2, cta_group=3, grid=grid, group_m=group_m, stream_k=False)
    assert r2.ok and not r2.stream_k
    assert _bits_equal(c2, c)


def test_k4_stream_k_ragged_fp8_records_exact(ctx):
    M, N, K, grid, group_m = STREAM_K_CASES[3][0]
    model = StreamK(M, N, K, grid, group_m)
    assert {"folds_2_or_more", "over_m", "over_n", "over_mn"} <= model.facts()
    a, b, exact = _exact_operands(M, N, K, seed=3)
    nb = -(-M // 128) * ops.panel_record_bytes(N)
    c = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda")
    r = ops.gemm_send(ctx, a, b, c, cta_group=3, grid=grid, group_m=group_m, stream_k=True, out_fp8=True)
    assert r.ok and r.stream_k
    assert torch.equal(c[:nb], ops.ref_fp8_panels(exact.float()))
    assert torch.all(c[nb:] == 0xAB), "stored beyond the last record"


def test_k4_stream_k_ragged_send_exact(ctx):
    """Split tiles through the panel accounting: every (short) panel is posted once, after all its tiles."""
    M, N, K, grid, group_m = STREAM_K_CASES[0][0]
    model = StreamK(M, N, K, grid, group_m)
    assert {"split", "over_mn", "contrib_only_k_tail"} <= model.facts()
    a, b, exact = _exact_operands(M, N, K, seed=4)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    d = torch.full((M + 16, N), 3.0, device="cuda", dtype=torch.bfloat16)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, cta_group=3, grid=grid, group_m=group_m, stream_k=True)
    finally:
        ctx.engine_stop()
    assert r.ok and r.stream_k and r.panels_posted == -(-M // 128), (r.status, r.panels_posted)
    ref = exact.to(torch.bfloat16)
    assert _bits_equal(c, ref), _mismatch(c, ref)
    assert _bits_equal(d[:M], c) and torch.all(d[M:] == 3.0)


# ------------------------------------------------------------------ K4: fp8 epilogue, exact accumulators
@pytest.mark.parametrize("cta_group", [1, 2, 3])
@pytest.mark.parametrize("M,N,K", [(300, 32, 200), (300, 288, 1000), (130, 288, 72), (512, 544, 328)])
def test_k4_fp8_records_byte_exact(ctx, M, N, K, cta_group):
    """With exact accumulators there is no rounding-boundary excuse: the records equal the reference byte for byte,
    including the zero rows of the padded last panel."""
    a, b, exact = _exact_operands(M, N, K, seed=M + 5 * N + K + cta_group)
    nb = -(-M // 128) * ops.panel_record_bytes(N)
    c = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, out_fp8=True, cta_group=cta_group)
    assert r.ok, r.status
    ref = ops.ref_fp8_panels(exact.float())
    diff = (c[:nb] != ref).nonzero()
    assert diff.numel() == 0, f"{diff.numel()} record bytes differ, first at {diff[0].item()}"
    assert torch.all(c[nb:] == 0xAB), "stored beyond the last record"


# ------------------------------------------------------------------ K7: exact
def _mx_exact_operand(rows, K, g, scale_lo=124, scale_hi=130):
    """e4m3 codes of integers in [-4, 4] and scale bytes 127 +- 3."""
    v = torch.randint(-4, 5, (rows, K), generator=g).float()
    q = v.to(torch.float8_e4m3fn).view(torch.uint8)
    s = torch.randint(scale_lo, scale_hi + 1, (rows, K // 32), generator=g).to(torch.uint8)
    return q.cuda(), s.cuda()


def _deq64(q, s):
    """fp64 value of an MX operand: e4m3 * 2^(byte - 127), which is 2^-127 for byte 0 (no fp32 range limits)."""
    rows, K = q.shape
    v = q.view(torch.float8_e4m3fn).double().reshape(rows, K // 32, 32)
    return (v * torch.exp2(s.double() - 127)[..., None]).reshape(rows, K)


def _mx_exact_ref(aq, as_, bq, bs):
    A, B = _deq64(aq, as_), _deq64(bq, bs)
    # every product is a multiple of 2^(min scale exponents) and the block sums are integers <= 512: the fp32 accumulator
    # (24 bits) is exact while S stays below 2^24 of that quantum
    quantum = 2.0 ** (int(as_.min()) - 127 + int(bs.min()) - 127)
    S = A.abs() @ B.abs().T
    assert S.max().item() <= 2 ** 24 * quantum, "operands too large for an exact fp32 accumulation"
    return (A @ B.T).to(torch.bfloat16)


def _panel_records(q, s):
    rows, K = q.shape
    P_ = -(-rows // 128)
    rec = torch.zeros(P_, 128 * K + 128 * (K // 32), dtype=torch.uint8, device=q.device)
    qp = torch.zeros(P_ * 128, K, dtype=torch.uint8, device=q.device)
    sp = torch.full((P_ * 128, K // 32), 127, dtype=torch.uint8, device=q.device)
    qp[:rows], sp[:rows] = q, s
    rec[:, :128 * K] = qp.reshape(P_, -1)
    rec[:, 128 * K:] = sp.reshape(P_, -1)
    return rec.reshape(-1)


def _chunk_records(q, s, chunk):
    rows, K = q.shape
    n = rows * K
    rec = torch.zeros(n // chunk, P.record_bytes(chunk), dtype=torch.uint8, device=q.device)
    rec[:, :chunk] = q.reshape(n // chunk, chunk)
    rec[:, chunk:chunk + chunk // 32] = s.reshape(n // chunk, chunk // 32)
    return rec.reshape(-1)


def _mx_operand(kind, q, s):
    rows, K = q.shape
    if kind == "plain":
        return MX.MxOperand.from_tensors(q, s)
    if kind == "panel":
        return MX.MxOperand.from_panel_records(_panel_records(q, s), rows, K)
    chunk = 128 * K * (2 if rows % 256 == 0 else 1)
    return MX.MxOperand.from_chunk_records(_chunk_records(q, s, chunk), rows, K, chunk)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("kind,M,N,K", [("plain", 200, 136, 160), ("plain", 130, 72, 96), ("plain", 64, 300, 32), ("plain", 700, 520, 256),
                                        ("panel", 300, 136, 160), ("panel", 130, 264, 224), ("chunk", 256, 200, 160), ("chunk", 384, 72, 96),
                                        ("b_panel", 200, 300, 160), ("b_panel", 130, 264, 224), ("b_chunk", 96, 256, 160), ("b_chunk", 300, 384, 96)])
def test_k7_exact_integer_gemm_rounds_to_nearest_even(ctx, kind, M, N, K, cta_group):
    """kind: where A lives (plain, K4 panel records, K3 chunk records), or b_*: B in records (a ragged N: a short last
    panel record) with A plain."""
    g = _gen(M + N + K + cta_group)
    aq, as_ = _mx_exact_operand(M, K, g)
    bq, bs = _mx_exact_operand(N, K, g)
    ref = _mx_exact_ref(aq, as_, bq, bs)
    pad = torch.full((M + 1, N), 7.0, device="cuda", dtype=torch.bfloat16)
    c = pad[:M]
    a_kind, b_kind = (kind, "plain") if not kind.startswith("b_") else ("plain", kind[2:])
    r = ops.gemm_mxfp8(ctx, _mx_operand(a_kind, aq, as_), _mx_operand(b_kind, bq, bs), c, cta_group=cta_group)
    assert r.ok, r.status
    assert _bits_equal(c, ref), _mismatch(c, ref)
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


@pytest.mark.parametrize("cta_group", [1, 2])
def test_k7_scale_bytes_at_both_ends(ctx, cta_group):
    """Scale bytes 0x00 (2^-127), 0x01 and 0xFE paired across the operands so every block's scale product is a normal
    number: a decode of byte 0 as 0.0 (or as 2^-126) changes the result."""
    M, N = 256, 136
    pairs = [(0x00, 0xFE), (0x01, 0xFE), (0xFE, 0x00), (0xFE, 0x01), (0x7F, 0x7F)]      # exponent sums 0, 1, 0, 1, 0
    K = 32 * len(pairs)
    g = _gen(99)
    aq, _ = _mx_exact_operand(M, K, g)
    bq, _ = _mx_exact_operand(N, K, g)
    as_ = torch.tensor([p[0] for p in pairs], dtype=torch.uint8, device="cuda").repeat(M, 1)
    bs = torch.tensor([p[1] for p in pairs], dtype=torch.uint8, device="cuda").repeat(N, 1)
    A, B = _deq64(aq, as_), _deq64(bq, bs)
    exact = A @ B.T
    assert exact.abs().max().item() < 2 ** 11                                           # exact, and a normal bf16 where nonzero
    ref = exact.to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group).ok
    assert _bits_equal(c, ref), _mismatch(c, ref)


# ------------------------------------------------------------------ floating-point data: per-element fp64 error bound
def _spread(rows, K, g, kblk, cancel_rows=0, mirror_rows=0):
    """randn scaled by 2^[-20, 20] per row and per `kblk`-deep k-block.  The first `cancel_rows` rows have their second
    half equal to minus the first half, the first `mirror_rows` rows their second half equal to the first half: a
    cancelling row times a mirrored row is exactly 0 with a large S."""
    x = torch.randn(rows, K, generator=g)
    x = x * torch.exp2(torch.randint(-20, 21, (rows, 1), generator=g).float())
    kb = -(-K // kblk)
    x = x * torch.exp2(torch.randint(-20, 21, (kb,), generator=g).float()).repeat_interleave(kblk)[:K]
    h = K // 2
    x[:cancel_rows, h:2 * h] = -x[:cancel_rows, :h]
    x[:mirror_rows, h:2 * h] = x[:mirror_rows, :h]
    return x


def _bound_check(c, r, S, gamma, label):
    err = (c.double() - r).abs()
    bound = 2.0 ** -8 * r.abs() + gamma * S
    S = S.clamp_min(1e-300)
    ratio = (err / S).max().item()
    beyond = ((err - 2.0 ** -8 * r.abs()).clamp_min(0) / S).max().item()     # what the bf16 output rounding does not explain
    print(f"\n{label}: largest |c - r| / S = {ratio:.3e}, beyond bf16 output rounding {beyond:.3e} (gamma = {gamma:.3e})")
    bad = (err > bound).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} elements over the bound, first at {bad[0].tolist()}: "
                              f"got {c[tuple(bad[0])].item()}, fp64 {r[tuple(bad[0])].item()}")
    return ratio


@pytest.mark.parametrize("cta_group,stream_k", [(1, False), (2, False), (3, True)])
@pytest.mark.parametrize("M,N,K", [(515, 1000, 4104), (1000, 520, 1000)])
def test_k4_fp64_error_bound_with_spread_scales(ctx, M, N, K, cta_group, stream_k):
    g = _gen(M + N + K)
    a = _spread(M, K, g, 64, cancel_rows=8).to(torch.bfloat16).cuda()
    b = _spread(N, K, g, 64, mirror_rows=8).to(torch.bfloat16).cuda()
    r64 = a.double() @ b.double().T
    S = a.double().abs() @ b.double().abs().T
    assert torch.all(r64[:8, :8].abs() <= 1e-9 * S[:8, :8])          # cancelling rows: ~0 against a large S
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    r = ops.gemm_send(ctx, a, b, c, cta_group=cta_group, grid=15 if stream_k else 0, stream_k=stream_k)
    assert r.ok and r.stream_k == stream_k, (r.status, r.stream_k)
    _bound_check(c, r64, S, K * 2.0 ** -23, f"K4 {M}x{N}x{K} cta_group={cta_group}")


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("M,N,K", [(700, 520, 1024), (256, 264, 4096)])
def test_k7_fp64_error_bound_with_spread_scales(ctx, M, N, K, cta_group):
    g = _gen(M * 3 + N + K)
    aq, as_ = MX.quantize_mx(_spread(M, K, g, 32, cancel_rows=8).cuda())
    bq, bs = MX.quantize_mx(_spread(N, K, g, 32, mirror_rows=8).cuda())
    A, B = _deq64(aq, as_), _deq64(bq, bs)
    r64 = A @ B.T
    S = A.abs() @ B.abs().T
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group).ok
    _bound_check(c, r64, S, (K / 32) * 2.0 ** -23 + 32 * 2.0 ** -11, f"K7 {M}x{N}x{K} cta_group={cta_group}")


# ------------------------------------------------------------------ fp8 pack / unpack edges
def _bf16(vals):
    return torch.tensor(vals, dtype=torch.float32).to(torch.bfloat16)


def _edge_payload(n):
    """One payload holding every edge the quantiser has, one 32-element block each, then random blocks."""
    inf, nan = float("inf"), float("nan")
    bmax = torch.finfo(torch.bfloat16).max
    tiny = 2.0 ** -133                                                   # smallest bf16 subnormal
    blocks = [
        [tiny, -tiny, 3 * tiny, 2.0 ** -127, -(2.0 ** -126) * 0.5, 2.0 ** -130] + [0.0] * 26,   # bf16 subnormals
        [bmax, -bmax, 1.0, -3.0] + [0.0] * 28,                                                   # +-bf16 max
        [-0.0] * 31 + [1.5],                                                                     # -0 next to a value
        [-0.0] * 32,                                                                             # an all -0 block
        # amax 256 -> scale 2^0: e4m3 ties (17 between 16 and 18, 1.0625, 2.125, -9.5 ...) and the e4m3 subnormal range
        [256.0, 17.0, 19.0, -17.0, 1.0625, 1.1875, 2.125, -9.5, 2.0 ** -7, 3 * 2.0 ** -10, 2.0 ** -10, 5 * 2.0 ** -10,
         2.0 ** -11, -(2.0 ** -9), 7 * 2.0 ** -10, 0.0] + [1.0] * 16,
        [448.0 * 4] + [1.0] * 31,                                                                # exactly 448 * 2^k
        [1806.0] + [1.0] * 31,                                                                   # the bf16 just above 448 * 4
        [448.0 * 2.0 ** -10, -448.0 * 2.0 ** -10] + [2.0 ** -12] * 30,
        [nan, 3.0, 0.0, -1.25] + [0.5] * 28,                                                     # NaN inside a block
        [1.0, 2.0, inf, -0.5] + [0.25] * 28,                                                     # +Inf inside a block
        [-inf, 2.0, -3.0, 0.0] + [-1.0] * 28,                                                    # -Inf inside a block
        [nan] * 32,                                                                              # all NaN
        [inf, -inf] + [nan] * 30,
    ]
    head = _bf16([v for blk in blocks for v in blk])
    g = _gen(1)
    tail = (torch.randn(n - head.numel(), generator=g) * torch.exp2(torch.randint(-30, 30, ((n - head.numel()) // 32,), generator=g)
                                                                     .float()).repeat_interleave(32)).to(torch.bfloat16)
    return torch.cat([head, tail])


def _records_equal_up_to_nan_sign(got, ref, chunk):
    """Record bytes equal; an e4m3 NaN (0x7F / 0xFF) is compared without its sign bit, since the hardware conversion
    may produce one canonical NaN where the reference keeps the input's sign."""
    n_rec = got.numel() // P.record_bytes(chunk)
    g2, r2 = got.reshape(n_rec, -1), ref.reshape(n_rec, -1)
    gq, rq = g2[:, :chunk], r2[:, :chunk]
    nan = (rq & 0x7F) == 0x7F
    assert torch.equal((gq & 0x7F) == 0x7F, nan), "NaN codes at different positions"
    assert torch.equal(gq[~nan], rq[~nan]), "fp8 codes differ"
    assert torch.equal(g2[:, chunk:], r2[:, chunk:]), "scale bytes differ"


def test_pack_edge_values_match_reference(ctx):
    chunk = 8192
    x = _edge_payload(2 * chunk).cuda()
    staging = torch.zeros(P.staging_bytes(x.numel(), chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(staging)
    torch.cuda.synchronize()
    P.pack_fp8_write(ctx, x, smr, qp=None, chunk_elems=chunk)
    torch.cuda.synchronize()
    _records_equal_up_to_nan_sign(staging, P.ref_pack_fp8(x.cpu(), chunk).cuda(), chunk)
    sc = staging[chunk:chunk + 13].tolist()
    assert sc[9] == sc[10] == sc[12] == 254, sc                          # a block holding +-Inf: exponent 127
    assert sc[8] == 120 and sc[11] == 0, sc                              # NaN takes no part in its block's amax (3.0 -> 2^-7)


@pytest.mark.parametrize("chunk,grid", [(16384, 0), (49152, 1), (24576, 3), (16384, 3), (49152, 0)])
def test_pack_only_chunk_sizes_and_grid_stride(ctx, chunk, grid):
    """16384 / 49152: two tiles per step (pack_group<2>); 24576: one tile per step, three per chunk; grid 1 and 3 make
    the grid-stride loop take many steps."""
    n = chunk * 6
    x = torch.nan_to_num(_edge_payload(n).float(), nan=1.0, posinf=2.0, neginf=-2.0).to(torch.bfloat16).cuda()
    staging = torch.zeros(P.staging_bytes(n, chunk), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(staging)
    torch.cuda.synchronize()
    P.pack_fp8_write(ctx, x, smr, qp=None, chunk_elems=chunk, grid=grid)
    torch.cuda.synchronize()
    assert torch.equal(staging, P.ref_pack_fp8(x, chunk))


@pytest.mark.parametrize("chunk,pack_grid", [(16384, 3), (49152, 1), (24576, 0)])
def test_fused_pack_write_and_unpack_odd_grids(ctx, chunk, pack_grid):
    """Pack fused with the RDMA write over a loopback QP, then unpack at grid 3 both waiting on the receive CQ and
    from records already in place."""
    n_chunks = 6
    n = chunk * n_chunks
    x = torch.nan_to_num(_edge_payload(n).float(), nan=1.0, posinf=2.0, neginf=-2.0).to(torch.bfloat16).cuda()
    nb = P.staging_bytes(n, chunk)
    staging = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    remote = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    out = torch.zeros_like(x)
    out2 = torch.zeros_like(x)
    smr, rmr = ctx.reg_mr(staging), ctx.reg_mr(remote)
    cq_a, cq_b = ctx.create_cq(256), ctx.create_cq(256)
    qa = ctx.create_qp(cq_a, cq_a, 64, 64)
    qb = ctx.create_qp(cq_b, cq_b, 64, 64)
    qa.connect(qb)
    for _ in range(n_chunks):
        qb.post_recv(rmr, 0)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        uview, ustream = P.unpack_fp8(ctx, remote, out, chunk, qp=qb, grid=3, sync=False, stream=ctx.aux_stream)
        r = P.pack_fp8_write(ctx, x, smr, qp=qa, dst_mr=rmr, chunk_elems=chunk, with_imm=True, grid=pack_grid)
        ustream.synchronize()
    finally:
        ctx.engine_stop()
    assert r.ok and r.wqes == n_chunks, r
    ref = P.ref_pack_fp8(x, chunk)
    assert torch.equal(staging, ref) and torch.equal(remote, ref)
    w = (C.c_int64 * 8).from_buffer(uview)
    assert w[0] == 0 and w[3] == n_chunks, list(w)
    want = P.ref_unpack_fp8(ref, n, chunk)
    assert _bits_equal(out, want)
    res = P.unpack_fp8(ctx, remote, out2, chunk, grid=3)
    assert res["status"] == "OK" and _bits_equal(out2, want)


def test_unpack_scale_bytes_at_both_ends(ctx):
    """Hand-made records: every e4m3 code (NaN included) under scale bytes 0x00, 0x01, 0xFE, 0xFF and a few in between.
    0x00 decodes as 2^-127; 0xFF as 2^128 = Inf (q * Inf: +-Inf, or NaN for a zero code); never produced, but pinned."""
    chunk = 8192 * 2
    n = chunk * 3
    g = _gen(5)
    q = torch.randint(0, 256, (n,), generator=g, dtype=torch.int32).to(torch.uint8)
    q[:256] = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    q[0], q[1] = 0x38, 0xB8                                                  # +-1.0 under scale byte 0x00: +-2^-127
    s =torch.tensor([0x00, 0x01, 0xFE, 0xFF, 0x7F, 0x02, 0x80, 0xFD], dtype=torch.uint8).repeat(n // 32 // 8)
    s = s[torch.randperm(s.numel(), generator=g)]
    s[:8] = torch.tensor([0x00, 0x01, 0xFE, 0xFF, 0x00, 0x01, 0xFE, 0xFF], dtype=torch.uint8)
    rec = torch.zeros(n // chunk, P.record_bytes(chunk), dtype=torch.uint8)
    rec[:, :chunk] = q.reshape(-1, chunk)
    rec[:, chunk:chunk + chunk // 32] = s.reshape(-1, chunk // 32)
    rec = rec.reshape(-1)
    want = P.ref_unpack_fp8(rec, n, chunk)
    out =torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    res = P.unpack_fp8(ctx, rec.cuda(), out, chunk, grid=3)
    assert res["status"] == "OK"
    got = out.cpu()
    assert got[:2].view(torch.int16).tolist() == [0x0040, -0x8000 | 0x0040], "scale byte 0x00 is not 2^-127"
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), "NaN at different positions"
    assert _bits_equal(got[~nan], want[~nan]), f"{int((got[~nan].view(torch.int16) != want[~nan].view(torch.int16)).sum())} values differ"
