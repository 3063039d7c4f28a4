"""K7 (`gemm_mxfp8.cu`) over the whole range of its scale bytes, against ``ops.ref_gemm_mxfp8``, the reference of its
arithmetic, bit for bit (fp64 on the GPU).

* Every pair of scale bytes 0 .. 254, one output each, under five classes of block partial (zero from disjoint supports,
  zero from cancelling products, the smallest, the largest, a negative one).  A scale product 2^ea * 2^eb formed in
  fp32 is Inf from ea + eb = 128 up and 0 below -149, while the block's contribution can still be an ordinary number:
  the kernel must not form it.  A plain, in panel and in chunk records, B plain and in records, both kernels.
* Operands made by the producers (K3 chunk records, K4 fp8 panel records) from bf16 data at both ends of the range,
  against `quantize_mx` weights: finite where the reference is, within the fp64 error bound, and the reference's Inf and
  NaN elsewhere; at a small shape and at 4096^3 beside a 32-CTA engine grid.  The three operands where the fp32 scale
  product is Inf or 0 are pinned.
* B held in records: K4 panel records (a ragged N) and K3 chunk records, both kernels.
* Edge classes, every output the sum of at most two chosen block contributions: bf16 ties and the same ties nudged,
  bf16-subnormal outputs, an fp32 sum that rounds to bf16 Inf, two finite blocks whose sum overflows, +Inf then -Inf
  across blocks, exact cancellation.  The classes whose value rests on the e4m3 MMA (subnormal codes, NaN codes against
  zero codes, a sum of -0 products) are checked against what an H100 gives, which DESIGN.md records.
* Accumulation order: exact block partials under scales spread over 2^+-30 across k, with half the blocks cancelling
  the other half, so the outputs are what the fp32 running sum rounded, on schedules where tiles enter the operand ring
  mid-way and units run many tiles: one rounding per block, in k order.  A kernel that rounds the scaled partial before
  adding it, or folds blocks out of order, fails; the exact-integer tests cannot see either.

Outside the producer test every block partial has at most 11 significant bits, so no bit-for-bit comparison depends on
the MMA's internal width."""
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import gemm_mx as MX
from test_gpu_gemm_scale import ENGINE_CTAS, SMALL_GRID, Schedule, _sms
from test_gpu_numerics import _bits_equal, _deq64, _mismatch, _mx_operand

pytestmark = pytest.mark.gpu


def _same(c, ref):
    """Bit equality, any NaN against any NaN."""
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(c), nan), f"{int((torch.isnan(c) != nan).sum())} outputs differ in NaN-ness"
    c2, r2 = torch.where(nan, 0.0, c.float()).to(torch.bfloat16), torch.where(nan, 0.0, ref.float()).to(torch.bfloat16)
    assert _bits_equal(c2, r2), _mismatch(c2, r2)


def _run(ctx, oa, ob, M, N, cta_group, grid=0):
    c = torch.full((M + 1, N), 7.0, device="cuda", dtype=torch.bfloat16)
    r = ops.gemm_mxfp8(ctx, oa, ob, c[:M], cta_group=cta_group, grid=grid)
    assert r.ok and r.variant == cta_group, (r.status, r.variant)
    assert torch.all(c[M] == 7.0), "the epilogue wrote past the last row"
    return c[:M]


# ------------------------------------------------------------------ every pair of scale bytes
# (A's codes, B's codes) at the first positions of one block: the block partial class each column group gets
PAIR_CLASSES = [
    ("disjoint_zero", [1.0] * 16 + [0.0] * 16, [0.0] * 16 + [1.0] * 16),
    ("cancel_zero", [1.0, 1.0], [1.0, -1.0]),
    ("smallest", [2.0 ** -9], [2.0 ** -9]),
    ("largest", [448.0] * 32, [448.0] * 32),
    ("negative", [1.5, 2.0, 3.0], [-1.0, 448.0, -3.0]),
]


def _every_pair_operands():
    """A [256, 32 * classes]: row i carries scale byte i on every block (row 255: 127) and every class's A codes in
    that class's block.  B [256 * classes, ...]: column group c has B's codes only in block c, column j of a group byte
    j (j = 255: 127).  Output (i, 256 c + j) is block c's partial times 2^(i + j - 254); the other blocks add p = 0."""
    n = len(PAIR_CLASSES)
    K = 32 * n
    aq = torch.zeros(256, K, dtype=torch.uint8)
    bq = torch.zeros(256 * n, K, dtype=torch.uint8)
    for c, (_, av, bv) in enumerate(PAIR_CLASSES):
        aq[:, 32 * c:32 * c + len(av)] = _e4m3_codes(av)
        bq[256 * c:256 * c + 256, 32 * c:32 * c + len(bv)] = _e4m3_codes(bv)
    byte = torch.arange(256, dtype=torch.int32)
    byte[255] = 127
    as_ = byte[:, None].expand(256, n).to(torch.uint8).contiguous()
    bs = byte.repeat(n)[:, None].expand(256 * n, n).to(torch.uint8).contiguous()
    return aq.cuda(), as_.cuda(), bq.cuda(), bs.cuda()


EVERY_PAIR_KINDS = [("plain", "plain"), ("panel", "plain"), ("chunk", "plain"), ("plain", "panel"), ("plain", "chunk"), ("chunk", "panel")]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("a_kind,b_kind", EVERY_PAIR_KINDS, ids=[f"A{a}-B{b}" for a, b in EVERY_PAIR_KINDS])
def test_k7_every_scale_byte_pair(ctx, a_kind, b_kind, cta_group):
    aq, as_, bq, bs = _every_pair_operands()
    ref = MX.ref_gemm_mxfp8(aq, as_, bq, bs)
    e = as_[:, :1].int() - 127 + (bs[:, 0].int() - 127)[None, :]
    assert e.max().item() == 254 and e.min().item() == -254
    assert torch.isinf(ref).any() and (ref[e > 127] != 0).any() and (ref[e < -149] != 0).any(), "the range ends are not exercised"
    assert not torch.isnan(ref).any()
    c = _run(ctx, _mx_operand(a_kind, aq, as_), _mx_operand(b_kind, bq, bs), aq.shape[0], bq.shape[0], cta_group)
    wrong = (torch.isnan(c) | (c.view(torch.int16) != ref.view(torch.int16))).sum().item()
    assert wrong == 0, f"{wrong} of {c.numel()} outputs differ from the reference; " + _mismatch(torch.nan_to_num(c), ref)


# ------------------------------------------------------------------ operands from the producers, at both ends of the range
def _edge_matrix(rows, K, g, finite_only):
    """bf16 [rows, K]: random blocks spread over 2^+-40, and in each row a few blocks at the top of the range (exponent
    119, and 120 with values that saturate to code 240), at 2^-67, bf16 subnormals, zero blocks, and (unless
    finite_only) blocks holding NaN or +-Inf."""
    x = torch.randn(rows, K, generator=g) * torch.exp2(torch.randint(-40, 41, (rows, K // 32, 1), generator=g).float()).expand(
        rows, K // 32, 32).reshape(rows, K)
    kinds = [lambda: torch.randn(32, generator=g) * 2.0 ** 126,
             lambda: torch.full((32,), 3.3e38) * torch.sign(torch.randn(32, generator=g)),
             lambda: torch.randn(32, generator=g) * 2.0 ** -67,
             lambda: torch.randint(-3, 4, (32,), generator=g).float() * 2.0 ** -133,
             lambda: torch.zeros(32)]
    if not finite_only:
        kinds += [lambda: torch.tensor([float("nan")] + [1.0] * 31), lambda: torch.tensor([float("inf"), -2.0] + [0.5] * 30),
                  lambda: torch.tensor([float("-inf")] + [3.0] * 31)]
    for r in range(rows):
        for kb in torch.randperm(K // 32, generator=g)[:len(kinds)].tolist():
            x[r, 32 * kb:32 * kb + 32] = kinds[(r + kb) % len(kinds)]()
    return x.to(torch.bfloat16)


def _k3_records(ctx, x, chunk):
    M, K = x.shape
    stg = torch.zeros(ops.staging_bytes(x.numel(), chunk), dtype=torch.uint8, device="cuda")
    ops.pack_fp8_write(ctx, x.reshape(-1), ctx.reg_mr(stg), qp=None, chunk_elems=chunk)
    torch.cuda.synchronize()
    r = stg.reshape(M * K // chunk, -1)
    return stg, r[:, :chunk].reshape(M, K), r[:, chunk:chunk + chunk // 32].reshape(M, K // 32)


def _k4_records(ctx, x):
    """K4's fp8 panel records of x itself: x @ I^T accumulates x exactly (finite data only: an Inf times the identity's
    zeros would be NaN), and the epilogue quantises it."""
    M, K = x.shape
    rec = torch.zeros(-(-M // 128) * ops.panel_record_bytes(K), dtype=torch.uint8, device="cuda")
    assert ops.gemm_send(ctx, x, torch.eye(K, device="cuda", dtype=torch.bfloat16), rec, out_fp8=True).ok
    r = rec.reshape(-(-M // 128), -1)
    return rec, r[:, :128 * K].reshape(-1, K)[:M], r[:, 128 * K:].reshape(-1, K // 32)[:M]


BF16_OVERFLOW = (2.0 - 2.0 ** -8) * 2.0 ** 127        # the least magnitude that rounds to bf16 Inf


def _check_against_reference(c, aq, as_, bq, bs):
    """Block partials of random codes need more than 11 bits, so K7 is held to the fp64 bound, not to bits: finite where
    the reference is, the reference's Inf and NaN elsewhere -- except where the result, or a running sum on the way to
    it (at most S), comes within the bound of overflow: there an inexact partial may land on either side."""
    ref = MX.ref_gemm_mxfp8(aq, as_, bq, bs)
    A, B = _deq64(aq, as_), _deq64(bq, bs)
    A, B = torch.nan_to_num(A, nan=0.0, posinf=0.0, neginf=0.0), torch.nan_to_num(B, nan=0.0, posinf=0.0, neginf=0.0)
    r64, S = A @ B.T, A.abs() @ B.abs().T
    slack = 2.0 ** -8 * r64.abs() + ((aq.shape[1] / 32) * 2.0 ** -23 + 32 * 2.0 ** -11) * S
    edge = (r64.abs() + slack >= BF16_OVERFLOW) | (S >= 2.0 ** 127)
    fin = torch.isfinite(ref) & ~edge
    assert torch.isfinite(c[fin]).all(), f"{int((~torch.isfinite(c[fin])).sum())} outputs not finite where the reference is"
    bad = fin & ((c.double() - r64).abs() > slack)
    assert not bad.any(), f"{int(bad.sum())} outputs over the fp64 bound, first at {bad.nonzero()[0].tolist()}"
    inf = torch.isinf(ref) & ~edge
    assert torch.equal(c[inf], ref[inf]), f"{int((c[inf] != ref[inf]).sum())} Infs of the reference come out otherwise"
    nan = torch.isnan(ref) & ~edge
    assert torch.isnan(c[nan]).all() and not torch.isnan(c[torch.isfinite(ref) & ~edge]).any(), "NaN where the reference has none, or the other way"
    return int(torch.isinf(ref).sum()), int(torch.isnan(ref).sum())


PRODUCER_CASES = [("k3", 256, 256, 512, 0), ("k4", 256, 256, 512, 0), ("k3", 4096, 4096, 4096, "beside_engine"),
                  ("k4", 4096, 4096, 4096, "beside_engine")]


@pytest.mark.parametrize("producer,M,N,K,grid", PRODUCER_CASES, ids=[f"{p}-{m}x{n}x{k}" for p, m, n, k, _ in PRODUCER_CASES])
def test_k7_producer_records_at_both_ends_of_the_range(ctx, producer, M, N, K, grid):
    g = torch.Generator().manual_seed(M + K + len(producer))
    x = _edge_matrix(M, K, g, finite_only=producer == "k4").cuda()
    if producer == "k3":
        chunk = 128 * K * 2
        rec, aq, as_ = _k3_records(ctx, x, chunk)
        oa = MX.MxOperand.from_chunk_records(rec, M, K, chunk)
    else:
        rec, aq, as_ = _k4_records(ctx, x)
        oa = MX.MxOperand.from_panel_records(rec, M, K)
    aq, as_ = aq.contiguous(), as_.contiguous()
    assert {0, 246, 247}.issubset(set(as_.unique().tolist())) and (as_ <= 60).any()
    grid = _sms() - ENGINE_CTAS if grid == "beside_engine" else 0
    for scale in (1.0, 2.0 ** 60):                    # ordinary weights, and weights that push sums past fp32 max
        bq, bs = MX.quantize_mx((torch.randn(N, K, generator=g) * scale).to(torch.bfloat16).cuda())
        for cg in (1, 2):
            c = _run(ctx, oa, MX.MxOperand.from_tensors(bq, bs), M, N, cg, grid=grid)
            n_inf, n_nan = _check_against_reference(c, aq, as_, bq, bs)
            if scale > 1:
                assert n_inf > 0, "no output overflows"
            if producer == "k3":
                assert n_nan > 0, "no NaN block reached the product"
    del rec


TABLE = [
    # (A blocks, B blocks as bf16 values; the exact product): scale-byte sums 128, 128 and -150
    ("sum_128_finite", [[2.0 ** 127], [1.0]], [[1.0, 2.0 ** 17], [1.0]], 2.0 ** 127 + 1),
    ("sum_128_zero_partial", [[2.0 ** 127], [1.0]], [[0.0, 2.0 ** 17], [1.0]], 1.0),
    ("sum_minus_150", [[2.0 ** -67] * 32] * 128, [[2.0 ** -67] * 32] * 128, 4096 * 2.0 ** -134),
]


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("name,a,b,exact", TABLE, ids=[t[0] for t in TABLE])
def test_k7_scale_range_regressions(ctx, name, a, b, exact, cta_group):
    """Finite bf16 operands, quantised by the producers' rule, whose fp32 scale product is Inf (+Inf, or NaN against a
    zero partial, in place of a finite result) or 0 (0 in place of a normal bf16)."""
    def mat(blocks):
        row = [v for blk in blocks for v in list(blk) + [0.0] * (32 - len(blk))]
        return torch.tensor([row] * 3, dtype=torch.float32).to(torch.bfloat16).cuda()
    (aq, as_), (bq, bs) = MX.quantize_mx(mat(a)), MX.quantize_mx(mat(b))
    want = torch.full((3, 3), exact, dtype=torch.float64).to(torch.bfloat16)
    assert torch.equal(MX.ref_gemm_mxfp8(aq, as_, bq, bs).cpu(), want)
    c = _run(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), 3, 3, cta_group)
    assert _bits_equal(c.cpu(), want), (c[0, 0].item(), want[0, 0].item())


# ------------------------------------------------------------------ edge classes: at most two chosen block contributions
# each case: two blocks of (products (a value, b value), exponent sum ea + eb), and whether its value rests on the MMA
NAN = float("nan")
EDGE_CASES = [
    ("tie_to_even_down", [([(1.0, 1.0)], 0), ([(1.0, 1.0)], -8)], False),                      # 1 + 2^-8 -> 1
    ("tie_to_even_up", [([(1.0, 1.0), (0.125, 0.0625)], 0), ([(1.0, 1.0)], -8)], False),      # 1 + 2^-7 + 2^-8 -> 1 + 2^-6
    ("tie_nudged_below", [([(1.0, 1.0)], 0), ([(1.5, 1.0)], -9)], False),
    ("tie_nudged_above", [([(1.0, 1.0)], 0), ([(1.125, 1.0)], -8)], False),
    ("bf16_subnormal_tie", [([(3.0, 1.0)], -134), ([], 0)], False),                            # 1.5 * 2^-133
    ("bf16_subnormal_to_zero", [([(1.0, 1.0)], -140), ([], 0)], False),
    ("fp32_rounds_to_bf16_inf", [([(448.0, 1.0), (7.0, 9.0)], 119), ([], 0)], False),          # 511 * 2^119
    ("finite_blocks_overflow", [([(1.5, 1.0)], 127), ([(1.5, 1.0)], 127)], False),
    ("inf_then_minus_inf", [([(448.0, 448.0)], 127), ([(-448.0, 448.0)], 127)], False),        # each block overflows alone
    ("cancel_across_blocks", [([(3.0, 1.0)], 50), ([(-3.0, 1.0)], 50)], False),
    ("cancel_at_the_top", [([(448.0, 448.0)], 110), ([(-448.0, 448.0)], 110)], False),
    ("e4m3_subnormal_codes", [([(2.0 ** -9, 3.0 * 2.0 ** -9)], 0), ([(2.0 ** -8, 1.0)], -3)], True),
    ("minus_zero_partial", [([(-0.125, 0.125)], -149), ([(-0.0, 1.0)], 0)], True),             # -0 accumulator, then a -0 partial
    ("nan_code_in_a", [([(NAN, 1.0)], 0), ([(1.0, 1.0)], 0)], True),
    ("nan_code_in_b", [([(1.0, NAN)], 0), ([(1.0, 1.0)], 0)], True),
]
# What an H100 SXM gives for the classes that rest on the e4m3 MMA (DESIGN.md, fp8 numerics): subnormal codes are
# multiplied exactly and a NaN code makes its block's partial NaN even against zero codes, as IEEE has it; a sum of -0
# products comes out +0 (as in K4's bf16 MMA), where IEEE gives -0, so the -0 accumulator before it becomes +0.
H100_MMA = {"e4m3_subnormal_codes": "reference", "minus_zero_partial": "[0.0] vs [-0.0]",
            "nan_code_in_a": "reference", "nan_code_in_b": "reference"}


def _e4m3_codes(vals):
    t = torch.tensor(vals, dtype=torch.float32)
    q = t.to(torch.float8_e4m3fn)
    ok = torch.isnan(t) | (q.float() == t)
    assert ok.all(), f"not e4m3 values: {t[~ok].tolist()}"
    return q.view(torch.uint8)


def _edge_operands():
    """Case i is row i of A and column i of B, its products at positions 2i and 2i + 1 of each block (zeros elsewhere),
    its exponent sum split between the two scale bytes; every other output is a sum of zero products."""
    n = len(EDGE_CASES)
    aq, bq = torch.zeros(n, 64, dtype=torch.uint8), torch.zeros(n, 64, dtype=torch.uint8)
    as_, bs = torch.full((n, 2), 127, dtype=torch.uint8), torch.full((n, 2), 127, dtype=torch.uint8)
    for i, (_, blocks, _) in enumerate(EDGE_CASES):
        for k, (prods, e) in enumerate(blocks):
            for t, (va, vb) in enumerate(prods):
                aq[i, 32 * k + 2 * i + t], bq[i, 32 * k + 2 * i + t] = _e4m3_codes([va])[0], _e4m3_codes([vb])[0]
            as_[i, k], bs[i, k] = 127 + e // 2, 127 + e - e // 2
        if EDGE_CASES[i][0] == "minus_zero_partial":
            aq[i, 32:] |= 0x80                        # every product of block 1 is -0: an IEEE sum of -0
    return aq.cuda(), as_.cuda(), bq.cuda(), bs.cuda()


@pytest.mark.parametrize("cta_group", [1, 2])
def test_k7_edge_classes(ctx, cta_group):
    aq, as_, bq, bs = _edge_operands()
    n = len(EDGE_CASES)
    ref = MX.ref_gemm_mxfp8(aq, as_, bq, bs).cpu()
    want = {"tie_to_even_down": 1.0, "tie_to_even_up": 1.0 + 2.0 ** -6, "tie_nudged_below": 1.0, "tie_nudged_above": 1.0 + 2.0 ** -7,
            "bf16_subnormal_tie": 2.0 ** -132, "bf16_subnormal_to_zero": 0.0, "fp32_rounds_to_bf16_inf": float("inf"),
            "finite_blocks_overflow": float("inf"), "inf_then_minus_inf": float("inf"), "cancel_across_blocks": 0.0,
            "cancel_at_the_top": 0.0, "e4m3_subnormal_codes": 3.0 * 2.0 ** -18 + 2.0 ** -11, "minus_zero_partial": -0.0}
    for i, (name, _, _) in enumerate(EDGE_CASES):
        if name in want:
            assert ref[i, i].view(torch.int16) == torch.tensor(want[name], dtype=torch.bfloat16).view(torch.int16), (name, ref[i, i].item())
        else:
            assert torch.isnan(ref[i, i]), name
    c = _run(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), n, n, cta_group).cpu()
    mma = torch.zeros(n, n, dtype=torch.bool)
    for i, (name, _, on_mma) in enumerate(EDGE_CASES):
        if on_mma:
            mma[i, i] = True
            if name.startswith("nan_code"):
                mma[i, :] = mma[:, i] = True
            if name == "minus_zero_partial":
                mma[i, :] = True
    _same(torch.where(mma, 0.0, c.float()).to(torch.bfloat16), torch.where(mma, 0.0, ref.float()).to(torch.bfloat16))
    seen = {}
    for i, (name, _, on_mma) in enumerate(EDGE_CASES):
        if not on_mma:
            continue
        rows = torch.arange(n) if name == "nan_code_in_b" else torch.tensor([i])
        cols = torch.arange(n) if name == "nan_code_in_a" else torch.tensor([i])
        got, exp = c[rows][:, cols], ref[rows][:, cols]
        same = torch.equal(torch.isnan(got), torch.isnan(exp)) and torch.equal(torch.nan_to_num(got).view(torch.int16),
                                                                               torch.nan_to_num(exp).view(torch.int16))
        seen[name] = "reference" if same else f"{got.flatten()[:4].tolist()} vs {exp.flatten()[:4].tolist()}"
    print("\nK7 MMA classes:", seen)
    assert seen == H100_MMA, seen


# ------------------------------------------------------------------ accumulation order
def _spread_operand(rows, K, g, negate):
    """Integer codes in [-4, 4] (block partials are integers below 2^10: exact in any MMA) under scale bytes 127 +- 30.
    In the first half of the rows the second half of the blocks repeats the first (negated when `negate`), so those rows
    of A against those of B cancel exactly and leave what the fp32 running sum rounded, in the order it rounded it."""
    q = torch.randint(-4, 5, (rows, K), generator=g).float().to(torch.float8_e4m3fn).view(torch.uint8)
    s = torch.randint(97, 158, (rows, K // 32), generator=g).to(torch.uint8)
    h, r = K // 2, rows // 2
    q[:r, h:] = q[:r, :h] ^ (0x80 if negate else 0)
    s[:r, h // 32:] = s[:r, :h // 32]
    return q.cuda(), s.cuda()


ORDER_CASES = [((1536, 1536, 1152), 1, SMALL_GRID), ((1536, 1536, 1152), 2, SMALL_GRID), ((1000, 776, 1408), 1, 40),
               ((1000, 776, 1408), 2, 40), ((1536, 1536, 2048), 2, SMALL_GRID)]


@pytest.mark.parametrize("shape,cta_group,grid", ORDER_CASES, ids=[f"{m}x{n}x{k}-cg{cg}-g{gr}" for (m, n, k), cg, gr in ORDER_CASES])
def test_k7_one_rounding_per_block_in_k_order(ctx, shape, cta_group, grid):
    M, N, K = shape
    sch = Schedule("k7", M, N, K, cta_group, grid, sms=_sms())
    f = sch.facts()
    assert f["mid_ring_entry"] == (K % 512 != 0), f
    if grid == SMALL_GRID:
        assert f["max_tiles_per_unit"] >= 8, f
    g = torch.Generator().manual_seed(M + N + K + cta_group)
    (aq, as_), (bq, bs) = _spread_operand(M, K, g, False), _spread_operand(N, K, g, True)
    ref = MX.ref_gemm_mxfp8(aq, as_, bq, bs)
    # the fp32 running sum does round: where the blocks cancel exactly, most outputs are what it rounded
    assert (ref[:M // 2, :N // 2] != 0).float().mean().item() > 0.5
    c = _run(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), M, N, cta_group, grid=grid)
    _same(c, ref)
