"""``ops.ref_gemm_mxfp8``, the bit-exact reference of K7's arithmetic, against an independent model in exact rationals
(``fractions.Fraction``: e4m3 codes decoded from their bits, each block's contribution exact, one round to fp32 per
block, one round to bf16), against the fp64 product of ``dequantize_mx`` where every partial sum is exact in fp32, and
on the three operands at the top and bottom of the scale range where a scale product formed in fp32 is Inf or 0."""
import math
from fractions import Fraction

import pytest
import torch

from rocnrdma_b200.ops import gemm_mx as MX

INF, NAN = float("inf"), float("nan")


# ------------------------------------------------------------------ exact-rational model
def _e4m3(code):
    """e4m3 (fn) code -> Fraction, or None for NaN; the sign of a zero is returned separately."""
    s, e, m = code >> 7, (code >> 3) & 0xF, code & 7
    if e == 0xF and m == 7:
        return None, s
    v = Fraction(m, 8) * Fraction(2) ** -6 if e == 0 else (1 + Fraction(m, 8)) * Fraction(2) ** (e - 7)
    return (-v if s else v), s


def _round(x, mant_bits, emin):
    """Fraction -> the nearest float with `mant_bits` fraction bits, exponents from emin (subnormals below) up to 127,
    ties to even, +-Inf past the largest; returned as a Python float (exact: both formats fit in fp64)."""
    if x == 0:
        return 0.0
    neg, m = x < 0, abs(x)
    e = m.numerator.bit_length() - m.denominator.bit_length()
    if Fraction(2) ** e > m:
        e -= 1
    ulp = Fraction(2) ** (max(e, emin) - mant_bits)
    q, r = divmod(m, ulp)
    if r * 2 > ulp or (r * 2 == ulp and q % 2 == 1):
        q += 1
    v = q * ulp
    out = INF if v >= Fraction(2) ** 128 else float(v)
    return -out if neg else out


def _fp32_add(acc, x):
    """IEEE fp32 acc + x, x exact (Fraction with a zero sign, or a float +-Inf / NaN), rounded once."""
    if not math.isfinite(acc):
        return acc + x if isinstance(x, float) else acc            # Inf + a finite value stays Inf
    if isinstance(x, float):
        return acc + x
    v, zsign = x
    total = Fraction(acc) + v
    if total == 0:
        if acc == 0 and v == 0:                       # -0 only when both are -0
            return -0.0 if (math.copysign(1, acc) < 0 and zsign) else 0.0
        return 0.0
    r = _round(total, 23, -126)
    return math.copysign(0.0, -1 if total < 0 else 1) if r == 0 else r


def _model(aq, as_, bq, bs):
    M, K = aq.shape
    Nn = bq.shape[0]
    out = torch.empty(M, Nn, dtype=torch.float32)
    for i in range(M):
        for j in range(Nn):
            acc = 0.0
            for k in range(K // 32):
                p, nan, all_negzero = Fraction(0), False, True
                for t in range(32 * k, 32 * k + 32):
                    (va, sa), (vb, sb) = _e4m3(int(aq[i, t])), _e4m3(int(bq[j, t]))
                    if va is None or vb is None:
                        nan = True
                        continue
                    p += va * vb
                    all_negzero &= (va * vb == 0) and (sa != sb)
                ba, bb = int(as_[i, k]), int(bs[j, k])
                if nan:
                    x = NAN
                elif ba == 255 or bb == 255:
                    x = NAN if p == 0 else math.copysign(INF, p)
                else:
                    x = (p * Fraction(2) ** (ba + bb - 254), all_negzero)
                acc = _fp32_add(acc, x)
            out[i, j] = _round(Fraction(acc), 7, -126) if math.isfinite(acc) and acc != 0 else acc
    return out.to(torch.bfloat16)                      # exact: every value is already a bf16


def _same(got, want):
    """bf16 bit equality, NaN against NaN regardless of its payload and sign."""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), "NaN at different positions"
    g, w = got.view(torch.int16)[~nan], want.view(torch.int16)[~nan]
    bad = (g != w).nonzero()
    assert bad.numel() == 0, f"{bad.numel()} outputs differ: {got[~nan][bad[:4, 0]].tolist()} vs {want[~nan][bad[:4, 0]].tolist()}"


# ------------------------------------------------------------------ the reference against the model
@pytest.mark.parametrize("seed", range(4))
def test_reference_matches_rational_model_on_random_codes_and_bytes(seed):
    """Every code (NaN and -0 included) and every scale byte 0 .. 255, so blocks overflow, underflow, cancel and carry
    Inf and NaN across k."""
    g = torch.Generator().manual_seed(seed)
    M, Nn, K = 5, 6, 128
    aq = torch.randint(0, 256, (M, K), generator=g, dtype=torch.int32).to(torch.uint8)
    bq = torch.randint(0, 256, (Nn, K), generator=g, dtype=torch.int32).to(torch.uint8)
    if seed % 2:                                                      # half the seeds without NaN codes
        aq[(aq & 0x7F) == 0x7F] = 0x38
        bq[(bq & 0x7F) == 0x7F] = 0x38
    as_ = torch.randint(0, 256 if seed < 2 else 255, (M, K // 32), generator=g, dtype=torch.int32).to(torch.uint8)
    bs = torch.randint(0, 256 if seed < 2 else 255, (Nn, K // 32), generator=g, dtype=torch.int32).to(torch.uint8)
    _same(MX.ref_gemm_mxfp8(aq, as_, bq, bs), _model(aq, as_, bq, bs))


def _sparse_codes(rows, K, g, codes):
    """Each block holds 1 or 2 codes from `codes` at random positions, zeros (+0 or -0) elsewhere."""
    q = torch.where(torch.rand(rows, K, generator=g) < 0.5, 0x00, 0x80).to(torch.uint8)
    for r in range(rows):
        for k in range(K // 32):
            n = int(torch.randint(1, 3, (1,), generator=g))
            pos = torch.randperm(32, generator=g)[:n] + 32 * k
            q[r, pos] = torch.tensor(codes, dtype=torch.uint8)[torch.randint(0, len(codes), (n,), generator=g)]
    return q


@pytest.mark.parametrize("seed", range(3))
def test_reference_matches_rational_model_on_edge_operands(seed):
    """Sparse blocks of edge codes (448, 240, subnormals, +-0) under bytes near both ends of the range and at the
    seams of fp32 (sums of exponents -150 .. -148, 126 .. 129): ties, subnormal accumulators, overflow of one block
    and of a sum of blocks, +-Inf from 0xFF, and -0 sums."""
    g = torch.Generator().manual_seed(100 + seed)
    M, Nn, K = 6, 5, 96
    codes = [0x7E, 0xFE, 0x77, 0xF7, 0x01, 0x81, 0x07, 0x38, 0xB8, 0x00, 0x80, 0x3C, 0x40]
    aq, bq = _sparse_codes(M, K, g, codes), _sparse_codes(Nn, K, g, codes)
    pick = torch.tensor([0, 1, 2, 52, 100, 104, 105, 106, 127, 200, 253, 254, 255], dtype=torch.int32)
    as_ = pick[torch.randint(0, len(pick), (M, K // 32), generator=g)].to(torch.uint8)
    bs = (254 - pick)[torch.randint(0, len(pick), (Nn, K // 32), generator=g)].clamp(0, 255).to(torch.uint8)
    _same(MX.ref_gemm_mxfp8(aq, as_, bq, bs), _model(aq, as_, bq, bs))


def test_reference_matches_dequantised_fp64_product_where_fp32_sums_are_exact():
    """Integer codes in [-4, 4] under bytes 124 .. 130: every running sum is an exact fp32 number, so the rule reduces
    to the fp64 product of the dequantised operands, rounded once to bf16."""
    g = torch.Generator().manual_seed(7)
    M, Nn, K = 37, 29, 320
    aq = torch.randint(-4, 5, (M, K), generator=g).float().to(torch.float8_e4m3fn).view(torch.uint8)
    bq = torch.randint(-4, 5, (Nn, K), generator=g).float().to(torch.float8_e4m3fn).view(torch.uint8)
    as_ = torch.randint(124, 131, (M, K // 32), generator=g).to(torch.uint8)
    bs = torch.randint(124, 131, (Nn, K // 32), generator=g).to(torch.uint8)
    A, B = MX.dequantize_mx(aq, as_).double(), MX.dequantize_mx(bq, bs).double()
    S = A.abs() @ B.abs().T
    assert S.max().item() <= 2.0 ** 24 * 2.0 ** -6, "an fp32 running sum could round"
    _same(MX.ref_gemm_mxfp8(aq, as_, bq, bs), (A @ B.T).to(torch.bfloat16))


def test_round_once_per_block_not_twice():
    """acc = 1 + 2^-24 + 2^-60 in one block: the fp64 sum 1 + 2^-24 is an fp32 tie and would round to 1.0; the exact sum
    is above it and must round up to 1 + 2^-23."""
    acc = torch.tensor([1.0], dtype=torch.float32)
    x = torch.tensor([2.0 ** -24 + 2.0 ** -60], dtype=torch.float64)
    assert (acc.double() + x).float().item() == 1.0                   # what a plain fp64 add then .float() gives
    assert MX._add_rn32(acc, x).item() == 1.0 + 2.0 ** -23


# ------------------------------------------------------------------ operands at both ends of the range, made by the quantiser
def _bf16_blocks(*blocks):
    row = []
    for b in blocks:
        row += list(b) + [0.0] * (32 - len(b))
    return torch.tensor([row], dtype=torch.float32).to(torch.bfloat16)


TOP_A = ((2.0 ** 127,), (1.0,))


def range_cases():
    """(A bf16, B bf16, the exact product's value): scale-byte sums 128, 128 and -150, where 2^ea * 2^eb in fp32 is Inf,
    Inf (against a zero partial) and 0."""
    return [
        ("sum_128_finite", _bf16_blocks(*TOP_A), _bf16_blocks((1.0, 2.0 ** 17), (1.0,)), 2.0 ** 127 + 1),
        ("sum_128_zero_partial", _bf16_blocks(*TOP_A), _bf16_blocks((0.0, 2.0 ** 17), (1.0,)), 1.0),
        ("sum_minus_150", torch.full((1, 4096), 2.0 ** -67).to(torch.bfloat16), torch.full((1, 4096), 2.0 ** -67).to(torch.bfloat16),
         4096 * 2.0 ** -134),
    ]


@pytest.mark.parametrize("name,a,b,exact", range_cases(), ids=[c[0] for c in range_cases()])
def test_reference_at_the_ends_of_the_scale_range(name, a, b, exact):
    (aq, as_), (bq, bs) = MX.quantize_mx(a), MX.quantize_mx(b)
    sums = (as_.int() + bs.int() - 254).tolist()[0]
    assert max(sums) == 128 if name.startswith("sum_128") else min(sums) == -150, sums
    fp32_scales = MX.ue8m0(as_) * MX.ue8m0(bs)                        # a scale product formed in fp32
    assert torch.isinf(fp32_scales).any() if name.startswith("sum_128") else torch.all(fp32_scales == 0)
    want = torch.tensor([[exact]], dtype=torch.float64).to(torch.bfloat16)
    got = MX.ref_gemm_mxfp8(aq, as_, bq, bs)
    assert torch.isfinite(want).all() and got.view(torch.int16).item() == want.view(torch.int16).item(), (got.item(), want.item())
    _same(got, _model(aq, as_, bq, bs))
    assert {"sum_128_finite": 1.70e38, "sum_128_zero_partial": 1.0, "sum_minus_150": 1.88e-37}[name] == pytest.approx(got.item(), rel=1e-2)
