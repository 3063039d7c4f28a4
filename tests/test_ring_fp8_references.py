"""An independent model of the fp8 ring all-reduce on the CPU, held against ``ops.ref_allreduce_fp8``.

The model shares nothing with ``ops.pack``'s quantiser: no ``torch.float8_e4m3fn``, ``_scale_exponent``, ``ue8m0``,
``quantize_blocks`` or ``_quantized_records``.  Its encoder takes the block exponent from ``np.frexp`` of amax / 448
(the smallest e with amax / 2^e <= 448, clamped to [-127, 127]), rounds to nearest even on the e4m3 grid in fp64
(subnormals included, step 2^-9), ignores NaN in amax, gives a block holding Inf e = 127 and multiplier 0, and at e = 120
saturates scaled values above 240 to 240.  It decodes with ``test_gpu_reduce_schedule``'s bit-field decoder, adds in
numpy fp32 and rounds to bf16 with its bit-level RNE.  The ring works element-wise on independent 32-element blocks, so
the model is per block: shard s packs ``x_s``; hop h = 1..N-1 adds ``x_{(s+h) mod N}`` (the addend first, one fp32 add)
and re-quantises; the final records decode to bf16.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.parallel import ring_fp8 as RF
from test_gpu_reduce_schedule import bf16_rne_bits, e4m3_fp64, ue8m0_fp64

CHUNK = 16384                                   # two tiles per record: blocks 0, 255, 256 and 511 start / end one
BF16_MAX = float(torch.finfo(torch.bfloat16).max)
FLT_MAX = float(np.finfo(np.float32).max)
_GRID = e4m3_fp64(np.arange(0x7F))              # the 127 non-negative finite codes 0..0x7E, ascending: 0 .. 448


# ------------------------------------------------------------------ the model
def encode(x):
    """fp32 blocks ``x[..., 32]`` -> (e4m3 codes uint8, scale bytes uint8)."""
    x = np.asarray(x, dtype=np.float64)
    a = np.where(np.isnan(x), 0.0, np.abs(x))
    amax = a.max(axis=-1)
    inf = np.isinf(amax)
    with np.errstate(invalid="ignore"):
        f, k = np.frexp(np.where(inf, 0.0, amax) / 448.0)
    e = np.where(f == 0.5, k - 1, k)                        # amax / 448 = f * 2^k: the smallest e with it <= 2^e
    e = np.where(amax == 0, -127, e)
    e = np.where(inf, 127, np.clip(e, -127, 127))
    mult = np.where(inf, 0.0, np.exp2(-e.astype(np.float64)))
    with np.errstate(invalid="ignore"):
        y = x * mult[..., None]                              # exact in fp64; Inf * 0 is NaN, a finite neighbour +-0
        mag = np.abs(y)
        mag = np.where((e[..., None] == 120) & (mag > 240.0), 240.0, mag)
    fin = np.where(np.isnan(mag), 0.0, np.minimum(mag, 448.0))
    hi = np.clip(np.searchsorted(_GRID, fin), 0, 126)        # _GRID[hi - 1] < fin <= _GRID[hi]
    lo = np.maximum(hi - 1, 0)
    dlo, dhi = fin - _GRID[lo], _GRID[hi] - fin
    code = np.where(dlo < dhi, lo, np.where(dhi < dlo, hi, np.where(lo % 2 == 0, lo, hi)))   # ties to the even code
    code = np.where(np.isnan(mag), 0x7F, code) | np.where(np.signbit(y), 0x80, 0)
    return code.astype(np.uint8), (e + 127).astype(np.uint8)


def decode(codes, scales):
    """fp32 values of (codes, scale bytes): the fp64 product of the bit fields, rounded once to fp32."""
    with np.errstate(over="ignore", invalid="ignore"):
        return (e4m3_fp64(codes) * ue8m0_fp64(scales)[..., None]).astype(np.float32)


def ring_blocks(xs, trace=None):
    """bf16 bits of the all-reduce of one shard's blocks.  ``xs``: [N, B, 32] fp32 with ``xs[h]`` the tensor that
    enters at hop h (rank (s + h) mod N for shard s).  ``trace``, a list, receives (quantised value, codes, scales)
    per hop."""
    xs = np.asarray(xs, dtype=np.float32)
    v = xs[0]
    codes, sc = encode(v)
    if trace is not None:
        trace.append((v, codes, sc))
    for h in range(1, len(xs)):
        with np.errstate(over="ignore", invalid="ignore"):
            v = xs[h] + decode(codes, sc)
        codes, sc = encode(v)
        if trace is not None:
            trace.append((v, codes, sc))
    return bf16_rne_bits(decode(codes, sc))


def ring_model(xs):
    """bf16 bits [n] of the all-reduce of the N ranks' bf16 tensors, shard by shard."""
    N = len(xs)
    x = np.stack([t.float().numpy() for t in xs])
    m = x.shape[1] // N
    out = np.empty(x.shape[1], dtype=np.uint16)
    for s in range(N):
        blocks = x[[(s + h) % N for h in range(N)], s * m:(s + 1) * m].reshape(N, -1, 32)
        out[s * m:(s + 1) * m] = ring_blocks(blocks).reshape(-1)
    return out


def assert_bits_equal(got, want_bits, label=""):
    """bf16 tensor against bf16 bits: NaN at the same positions (sign free), every other value identical."""
    g = got.view(torch.int16).numpy().astype(np.uint16)
    gn, wn = (g & 0x7FFF) > 0x7F80, (want_bits & 0x7FFF) > 0x7F80
    assert np.array_equal(gn, wn), f"{label}: NaN at {int((gn != wn).sum())} different positions"
    bad = np.flatnonzero(g[~wn] != want_bits[~wn])
    assert bad.size == 0, f"{label}: {bad.size} values differ, first at {np.flatnonzero(~wn)[bad[0]]}: " \
                          f"0x{g[~wn][bad[0]]:04x}, want 0x{want_bits[~wn][bad[0]]:04x}"


# ------------------------------------------------------------------ payloads
def spread(N, n, seed, lo=-20, hi=20):
    """N bf16 tensors of n: randn times 2^k per 32-element block, k uniform in [lo, hi]."""
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) *
             torch.exp2(torch.randint(lo, hi + 1, (n // 32,), generator=g).float()).repeat_interleave(32)).to(torch.bfloat16)
            for _ in range(N)]


def _kind_blocks(kind, g):
    """(what the entering rank holds, what the next rank holds, what every other rank holds) in one block, fp32."""
    z = np.zeros(32, np.float32)
    r = (torch.randn(32, generator=g) * 4).numpy()
    if kind == "nan":
        a = r.copy(); a[5] = np.nan
        return a, z, z
    if kind == "inf":
        a, b = z.copy(), z.copy(); a[7], b[7] = np.inf, -np.inf; a[8] = 3.0
        return a, b, z
    if kind == "overflow":                    # a finite partial sum that overflows fp32 where the second one joins
        a = z.copy(); a[9] = 1.5 * 2.0 ** 127; a[10] = -2.0
        return a, a.copy(), z
    if kind == "top":                         # top-of-range values with a finite exact sum
        a, b = z.copy(), z.copy()
        a[3], b[3] = 3.3e38, -1e38
        a[4], b[4] = -BF16_MAX, 2e38
        a[11] = BF16_MAX
        return a, b, z
    if kind == "zero":                        # an all-zero block among ranks that hold values
        return z, r, r
    if kind == "subnormal":                   # bf16 subnormals: amax / 448 far under 2^-127
        a = (np.arange(32) % 7 - 3).astype(np.float32) * np.float32(2.0 ** -133)
        a[0] = 127 * 2.0 ** -133
        return a, z, z
    if kind == "cancel":                      # x and -x
        return r, -r, z
    if kind == "huge":                        # one huge value, tiny neighbours
        a = (r * 2.0 ** -100).astype(np.float32); a[17] = 2.0 ** 100
        return a, z, z
    raise ValueError(kind)


KINDS = ("nan", "inf", "overflow", "top", "zero", "subnormal", "cancel", "huge")
POSITIONS = (0, 255, 256, 511)                # first / last block of a record and of each of its two tiles


def edge_payload(N, seed, chunk=CHUNK, base=None):
    """N bf16 tensors in which every kind enters every shard's ring at every hop: for shard s and hop h the kind's
    block sits on rank (s + h) mod N (its partner on the next rank), at the first or last block of a record or of a
    tile.  Returns (xs, R); R = 2N records per shard of ``chunk``.  Every other block holds ``base`` (default: spread
    values)."""
    assert chunk // 32 > max(POSITIONS)
    R = 2 * N
    n = N * R * chunk
    xs = [t.float().numpy().copy() for t in (base or spread(N, n, seed))]
    g = torch.Generator().manual_seed(seed + 1)
    m = n // N
    bpr = chunk // 32
    for s in range(N):
        for k, kind in enumerate(KINDS):
            for h in range(N):
                c = k * N + h                              # combination (kind, hop) -> one block position of one record
                blk = s * (m // 32) + (c // 4) * bpr + POSITIONS[c % 4]
                a, b, rest = _kind_blocks(kind, g)
                for q in range(N):
                    d = (q - s - h) % N
                    xs[q][blk * 32:(blk + 1) * 32] = a if d == 0 else b if d == 1 else rest
    return [torch.from_numpy(x).to(torch.bfloat16) for x in xs], R


# ------------------------------------------------------------------ the encoder on its own
def test_encoder_on_hand_picked_blocks():
    x = np.zeros((6, 32), np.float32)
    x[0, 0] = 448.0                                          # e = 0, code 0x7E
    x[1, :3] = [449.0, 1.0, -0.0]                            # e = 1: 224.5 -> 224, 0.5, -0
    x[2, :2] = [3.3e38, np.nan]                              # e = 120: 248.2 saturates to 240; NaN kept
    x[3, :2] = [2.0 ** -133, -3 * 2.0 ** -133]               # e = -127: 2^-6 and -3 * 2^-6
    x[4, :2] = [np.inf, 1.0]                                 # Inf: e = 127, multiplier 0
    x[5, :4] = [17.0, 18.0, 19.0, 2.0 ** -9 * 2.0 ** -1]     # amax 19 -> e = -4: 272, 288, 304 on the grid; 2^-6 under it
    codes, sc = encode(x)
    assert sc.tolist() == [127, 128, 247, 0, 254, 123]
    assert codes[0, 0] == 0x7E and codes[1, :3].tolist() == [0x76, 0x30, 0x80]
    assert codes[2, 0] == 0x77 and codes[2, 1] & 0x7F == 0x7F
    assert codes[3, :2].tolist() == [0x08, 0x94]
    assert codes[4, 0] & 0x7F == 0x7F and codes[4, 1] == 0x00
    # 272 is a tie between 256 and 288 -> 256 (even mantissa); 304 a tie between 288 and 320 -> 320; 2^-6 * 2^4 = 2^-2
    assert e4m3_fp64(codes[5, :3]).tolist() == [256.0, 288.0, 320.0]
    d = decode(codes, sc)
    assert d[2, 0] == 240 * 2.0 ** 120 and np.isfinite(d[2, 0])


@pytest.mark.parametrize("v", [FLT_MAX, BF16_MAX, 3.3e38], ids=["fp32_max", "bf16_max", "3.3e38"])
def test_saturation_stays_inside_the_bound(v):
    """At e = 120 the worst case is the largest fp32, 255.99.. * 2^120 -> 240 * 2^120: a relative error just under
    2^-4, so the bound of DESIGN.md 3.4 (2^-4 |v| per quantisation) still holds, and the decoded value is finite.  The
    package's quantiser agrees."""
    x = np.zeros((1, 32), np.float32)
    x[0, 0], x[0, 1] = v, -v
    codes, sc = encode(x)
    d = decode(codes, sc)[0, :2].astype(np.float64)
    assert sc[0] == 247 and np.isfinite(d).all() and d[0] == 240 * 2.0 ** 120 and d[1] == -d[0]
    err = abs(float(np.float32(v)) - d[0])
    assert err <= 2.0 ** -4 * float(np.float32(v)), (v, err / float(np.float32(v)))
    q, s = ops.pack.quantize_blocks(torch.from_numpy(x))
    assert torch.equal(q, torch.from_numpy(codes)) and torch.equal(s, torch.from_numpy(sc))


def test_encoder_equals_the_package_quantiser_on_spread_and_edge_blocks():
    """Every code and scale byte, NaN codes compared without their sign: values from bf16 subnormals to bf16 max and
    fp32 sums past it, and every edge kind."""
    x = np.concatenate([t.float().numpy() for t in spread(1, 1 << 16, 3, -133, 127)])
    x = np.concatenate([x, np.array([_kind_blocks(k, torch.Generator().manual_seed(4))[0] for k in KINDS]).reshape(-1),
                        np.float32([FLT_MAX, -FLT_MAX, 2.0 ** -149, 1.5 * 2.0 ** -127] + [0.0] * 28)]).reshape(-1, 32)
    codes, sc = encode(x)
    q, s = ops.pack.quantize_blocks(torch.from_numpy(x))
    q = q.numpy()
    nan = (codes & 0x7F) == 0x7F
    assert np.array_equal((q & 0x7F) == 0x7F, nan) and np.array_equal(q[~nan], codes[~nan])
    assert np.array_equal(s.numpy(), sc)


# ------------------------------------------------------------------ the model against the reference
@pytest.mark.parametrize("N", range(2, 9))
def test_model_equals_the_reference_on_spread_payloads(N):
    chunk = 8192
    xs = spread(N, N * 2 * chunk, seed=40 + N)
    assert_bits_equal(ops.ref_allreduce_fp8(xs, chunk), ring_model(xs), f"N={N}")


@pytest.mark.parametrize("N", range(2, 9))
def test_model_equals_the_reference_on_the_edge_payload(N):
    """Every kind enters at every hop; the top-of-range blocks come out finite."""
    xs, R = edge_payload(N, seed=60 + N)
    got = ops.ref_allreduce_fp8(xs, CHUNK)
    want = ring_model(xs)
    assert_bits_equal(got, want, f"N={N}")
    m = len(want) // N
    x = np.stack([t.float().numpy() for t in xs])
    top = np.zeros(len(want), bool)
    for s in range(N):
        for h in range(N):
            c = KINDS.index("top") * N + h
            blk = s * (m // 32) + (c // 4) * (CHUNK // 32) + POSITIONS[c % 4]
            top[blk * 32 + np.array([3, 4, 11])] = True
    assert np.isfinite(got.float().numpy()[top]).all(), "finite top-of-range inputs came out non-finite"
    with np.errstate(invalid="ignore"):
        exact = x.astype(np.float64).sum(axis=0)
    assert np.all(np.abs(got.double().numpy()[top] - exact[top]) <= 2.0 ** -4 * N * np.abs(x[:, top]).max(axis=0))


def test_top_of_range_sum_is_finite_on_every_shard():
    """The case that gave NaN: rank 0 holds 3.3e38, rank 1 -1e38 at element 3 of both shards.  The exact sum is 2.3e38;
    both shards must come out finite and within the bound, whichever rank owns them."""
    chunk = 8192
    xs = [torch.zeros(2 * chunk, dtype=torch.bfloat16) for _ in range(2)]
    for s in range(2):
        xs[0][s * chunk + 3], xs[1][s * chunk + 3] = 3.3e38, -1e38
    out = ops.ref_allreduce_fp8(xs, chunk).double()
    exact = float(xs[0][3].double() + xs[1][3].double())
    for s in range(2):
        v = out[s * chunk + 3].item()
        assert np.isfinite(v) and abs(v - exact) <= 2.0 ** -4 * (3.3e38 + abs(exact)), (s, v, exact)
    assert_bits_equal(out.to(torch.bfloat16), ring_model(xs))


# ------------------------------------------------------------------ the error bound and its domain
def _bound_and_domain(xs):
    """Per element: the bound of DESIGN.md 3.4 and whether the element's block is inside its domain (every partial sum
    of every element of the block finite in fp32 at every hop)."""
    N = len(xs)
    x = np.stack([t.float().numpy() for t in xs])
    n = x.shape[1]
    m = n // N
    bound, inside = np.zeros(n), np.zeros(n, bool)
    for s in range(N):
        blocks = x[[(s + h) % N for h in range(N)], s * m:(s + 1) * m].reshape(N, -1, 32)
        trace = []
        ring_blocks(blocks, trace)
        b = np.zeros(blocks.shape[1:])
        ok = np.ones(blocks.shape[1], bool)
        for h, (v, _, sc) in enumerate(trace):
            v = v.astype(np.float64)
            ok &= np.isfinite(v).all(axis=-1)
            e = sc.astype(np.float64)[..., None] - 127
            b += np.maximum(2.0 ** -4 * np.abs(v), 2.0 ** (e - 10))
            if h:
                b += np.abs(v) * 2.0 ** -24                  # the fp32 add that made v
        b += 2.0 ** -134                                      # the bf16 output, exact above its subnormals
        bound[s * m:(s + 1) * m] = b.reshape(-1)
        inside[s * m:(s + 1) * m] = np.repeat(ok, 32)
    return bound, inside


@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_error_bound_holds_inside_its_domain_up_to_bf16_max(N):
    """Inputs spread from bf16 subnormals to bf16 max.  Inside the domain every output is finite and within the bound;
    outside it the output is NaN exactly where the model says, and the bound is approached."""
    chunk = 8192
    xs = spread(N, N * 4 * chunk, seed=80 + N, lo=-133, hi=120)
    g = torch.Generator().manual_seed(90 + N)
    for x in xs:                                              # blocks near the top of the range on every rank
        top = torch.randint(0, x.numel() // 32, (x.numel() // 256,), generator=g)
        x.view(-1, 32)[top] = (torch.rand(top.numel(), 32, generator=g) * 2 - 1).mul(BF16_MAX).to(torch.bfloat16)
    got = ops.ref_allreduce_fp8(xs, chunk)
    want = ring_model(xs)
    assert_bits_equal(got, want, f"N={N}")
    bound, inside = _bound_and_domain(xs)
    assert inside.any() and (~inside).any(), "the payload must reach both sides of the domain"
    out = got.double().numpy()
    exact = np.sum([x.double().numpy() for x in xs], axis=0)
    assert np.isfinite(out[inside]).all(), "a finite output was expected inside the domain"
    err = np.abs(out - exact)[inside]
    assert np.all(err <= bound[inside]), f"max excess {np.max(err - bound[inside])}"
    assert np.max(err / np.maximum(bound[inside], 1e-300)) > 0.01, "the bound is never approached: the check is vacuous"
    assert np.array_equal(np.isnan(out[~inside]), ((want[~inside] & 0x7FFF) > 0x7F80))


# ------------------------------------------------------------------ plans the receive queue cannot hold
@pytest.mark.parametrize("N", range(2, 9))
def test_plan_refuses_records_the_receive_queue_cannot_hold(N):
    """A plan needs 2 x 2(N-1)R receive entries, rounded up to a power of two, and a queue holds at most 16384: the
    constructor refuses a larger R before it touches the context (``ctx=None`` reaches the check) and names the
    largest R for that N."""
    chunk = 8192
    R = RF.max_records(N)
    assert RF._pow2(4 * (N - 1) * R) <= RF.MAX_QUEUE_DEPTH < RF._pow2(4 * (N - 1) * (R + 1))
    with pytest.raises(AttributeError):                      # accepted: it goes on to allocate on the context
        RF.RingAllreduceFp8(None, N * R * chunk, chunk, 0, N)
    with pytest.raises(ValueError, match=f"at most {R}$"):
        RF.RingAllreduceFp8(None, N * (R + 1) * chunk, chunk, 0, N)


def test_largest_plans_at_the_boundary():
    assert RF.max_records(2) == 4096 and RF.max_records(8) == 585
    with pytest.raises(ValueError, match="R=4097 .* at most 4096"):
        RF.RingAllreduceFp8(None, 2 * 4097 * 8192, 8192, 0, 2)
