"""The fp8 ring reduce-scatter's reference against the independent e4m3 block model, and the layout identity between
K4's fp8 panel records and K3's chunk records that the GEMM-reduce-scatter rests on, on the CPU."""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from test_gpu_reduce_schedule import bf16_rne_bits
from test_ring_fp8_references import CHUNK, KINDS, _kind_blocks, assert_bits_equal, decode, edge_payload, encode, spread


def model_reduce_scatter(xs):
    """bf16 bits of every rank's shard, by the block model of test_ring_fp8_references (its own encoder and decoder):
    shard s's blocks enter at ranks s+1, s+2, ..., s (mod N); each later rank adds its part to the decode (one fp32
    add) and re-quantises, and the last sum is rounded to bf16 with nothing quantised after it."""
    N = len(xs)
    x = np.stack([t.float().numpy() for t in xs])
    m = x.shape[1] // N
    out = []
    for s in range(N):
        blocks = x[[(s + 1 + h) % N for h in range(N)], s * m:(s + 1) * m].reshape(N, -1, 32)
        v = blocks[0]
        for h in range(1, N):
            codes, sc = encode(v)
            with np.errstate(over="ignore", invalid="ignore"):
                v = blocks[h] + decode(codes, sc)
        out.append(bf16_rne_bits(v).reshape(-1))
    return out


@pytest.mark.parametrize("N", range(2, 9))
def test_reference_matches_block_model_on_spread_payloads(N):
    xs = spread(N, N * 2 * CHUNK, seed=300 + N)
    got, want = ops.ref_reduce_scatter_fp8(xs, CHUNK), model_reduce_scatter(xs)
    assert len(got) == N
    for s in range(N):
        assert_bits_equal(got[s], want[s], f"N={N} shard {s}")


@pytest.mark.parametrize("N", range(2, 9))
def test_reference_matches_block_model_on_the_edge_payload(N):
    """NaN, Inf, fp32 overflow, top-of-range, zero, subnormal, cancelling and huge blocks enter every shard at every hop,
    at the first and last blocks of records and tiles."""
    xs, _ = edge_payload(N, seed=400 + N)
    got, want = ops.ref_reduce_scatter_fp8(xs, CHUNK), model_reduce_scatter(xs)
    for s in range(N):
        assert_bits_equal(got[s], want[s], f"N={N} shard {s}")


@pytest.mark.parametrize("N", [2, 3, 5])
def test_fp32_partials_exact_in_bf16_give_the_bf16_result(N):
    chunk = 8192
    g = torch.Generator().manual_seed(100 + N)
    xs = [(torch.randint(-128, 129, (N * chunk,), generator=g) * 0.25).to(torch.bfloat16) for _ in range(N)]
    a = ops.ref_reduce_scatter_fp8(xs, chunk)
    b = ops.ref_reduce_scatter_fp8([x.float() for x in xs], chunk)
    for s in range(N):
        assert torch.equal(a[s].view(torch.int16), b[s].view(torch.int16)), s


@pytest.mark.parametrize("Nb", [64, 128, 320, 512])
@pytest.mark.parametrize("p", [1, 3])
def test_fp8_panels_are_chunk_records(Nb, p):
    """A K4 panel record of an [M, Nb] result is, byte for byte, a K3 chunk record of 128 * Nb elements."""
    g = torch.Generator().manual_seed(Nb + p)
    c = torch.randn(128 * p, Nb, generator=g) * 2.0 ** torch.randint(-30, 30, (128 * p, Nb), generator=g)
    assert ops.panel_record_bytes(Nb) == ops.record_bytes(128 * Nb)
    assert torch.equal(ops.ref_fp8_panels(c), ops.ref_pack_fp8(c.reshape(-1), 128 * Nb))


# ------------------------------------------------------------------ fp32 partials that are not exact in bf16
NB_EDGE = 64                                  # panel records of [128, 64]: two blocks a row, 256 a record
CHUNK_P = 128 * NB_EDGE
POSITIONS_P = (0, 3, 128, 255)                # first block of a record (and of row 0), last of row 1, first of row 64,
                                              # last of the record (and of row 127)
FP32_KINDS = KINDS + ("scale0", "e120")


def spread_fp32(N, n, seed):
    """N fp32 tensors of n: (1 + u) * 2^k with a random sign, u uniform in [0, 1) at full fp32 precision and k uniform
    in [-126, 126] per 32-element block, so every value is normal, from 2^-126 up to near FLT_MAX."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(N):
        k = torch.randint(-126, 127, (n // 32,), generator=g).double().repeat_interleave(32)
        v = (1 + torch.rand(n, generator=g, dtype=torch.float64)) * torch.exp2(k)
        sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0).double()
        out.append((v * sign).float())
    assert all(bool((x.abs() >= 2.0 ** -126).all()) and bool(torch.isfinite(x).all()) for x in out)
    return out


def _fp32_kind_blocks(kind, g):
    """``_kind_blocks`` for fp32 partials, and two kinds of the fused add's range: ``scale0``, blocks whose amax / 448
    is at most 2^-127 on both ranks (scale byte 0, decoded values fp32 subnormals), and ``e120``, a finite sum whose
    block exponent is 120, where the quantiser saturates scaled values above 240."""
    z = np.zeros(32, np.float32)
    if kind == "scale0":
        u = (1 + torch.rand(32, generator=g).numpy()) * np.where(np.arange(32) % 3 == 0, -1, 1)
        a = (u * 2.0 ** -123).astype(np.float32)
        b = (u[::-1] * 2.0 ** -122).astype(np.float32)
        return a, b, z
    if kind == "e120":
        a, b = z.copy(), z.copy()
        a[2], a[6], a[20] = 3.2e38, -2.9e38, 1e30
        b[2], b[21] = 1e37, -7.5
        return a, b, z
    return _kind_blocks(kind, g)


def edge_payload_fp32(N, seed):
    """N fp32 tensors of spread partials in which every kind of ``FP32_KINDS`` enters every shard at every hop, at the
    first and last blocks of a panel row and of a record (``POSITIONS_P``), as ``edge_payload`` places them."""
    R = -(-len(FP32_KINDS) * N // len(POSITIONS_P))
    n = N * R * CHUNK_P
    xs = [x.numpy().copy() for x in spread_fp32(N, n, seed)]
    g = torch.Generator().manual_seed(seed + 1)
    m, bpr = n // N, CHUNK_P // 32
    for s in range(N):
        for k, kind in enumerate(FP32_KINDS):
            for h in range(N):
                c = k * N + h
                blk = s * (m // 32) + (c // len(POSITIONS_P)) * bpr + POSITIONS_P[c % len(POSITIONS_P)]
                a, b, rest = _fp32_kind_blocks(kind, g)
                for q in range(N):
                    d = (q - s - h) % N
                    xs[q][blk * 32:(blk + 1) * 32] = a if d == 0 else b if d == 1 else rest
    return [torch.from_numpy(x) for x in xs]


def _records_of(codes, sc, chunk):
    n_rec = codes.size // chunk
    out = np.zeros((n_rec, ops.record_bytes(chunk)), np.uint8)
    out[:, :chunk] = codes.reshape(n_rec, chunk)
    out[:, chunk:chunk + chunk // 32] = sc.reshape(n_rec, chunk // 32)
    return torch.from_numpy(out.reshape(-1))


def records_equal_up_to_nan_sign(got, want, chunk, label):
    """K3 records byte for byte, except that a NaN code (0x7F / 0xFF) matches a NaN code of either sign."""
    g, w = got.reshape(-1, ops.record_bytes(chunk)), want.reshape(-1, ops.record_bytes(chunk))
    assert torch.equal(g[:, chunk:], w[:, chunk:]), f"{label}: scale bytes differ"
    gq, wq = g[:, :chunk], w[:, :chunk]
    nan = (wq & 0x7F) == 0x7F
    assert torch.equal((gq & 0x7F) == 0x7F, nan), f"{label}: NaN codes at other positions"
    assert torch.equal(gq[~nan], wq[~nan]), f"{label}: {int((gq[~nan] != wq[~nan]).sum())} codes differ"


def check_hop_by_hop(xs, chunk, label):
    """Every hop of every shard of the reference (``ref_pack_fp8``, then ``ref_reduce_fp8`` with the next rank's part)
    against the block model: the records of every hop up to the sign of NaN, and the last hop's bf16 sum bit for bit
    (NaN sign free).  The final outputs are ``ref_reduce_scatter_fp8``'s."""
    N = len(xs)
    m = xs[0].numel() // N
    got = ops.ref_reduce_scatter_fp8(xs, chunk)
    want = model_reduce_scatter(xs)
    x = np.stack([t.float().numpy() for t in xs])
    for s in range(N):
        assert_bits_equal(got[s], want[s], f"{label} shard {s}")
        part = slice(s * m, (s + 1) * m)
        recs = ops.ref_pack_fp8(xs[(s + 1) % N][part], chunk)
        codes, sc = encode(x[(s + 1) % N, part].reshape(-1, 32))
        records_equal_up_to_nan_sign(recs, _records_of(codes, sc, chunk), chunk, f"{label} shard {s} pack")
        for h in range(2, N + 1):
            y, recs = ops.ref_reduce_fp8(recs, 1, m, chunk, local=xs[(s + h) % N][part])
            with np.errstate(over="ignore", invalid="ignore"):
                v = x[(s + h) % N, part].reshape(-1, 32) + decode(codes, sc)
            codes, sc = encode(v)
            if h < N:
                records_equal_up_to_nan_sign(recs, _records_of(codes, sc, chunk), chunk, f"{label} shard {s} hop {h - 1}")
        assert_bits_equal(y, bf16_rne_bits(v).reshape(-1), f"{label} shard {s} last hop")
    return got


@pytest.mark.parametrize("N", range(2, 9))
def test_reference_matches_block_model_on_spread_fp32_partials(N):
    """Partials from 2^-126 to near FLT_MAX at full fp32 precision (``run_gemm``'s input, not exact in bf16)."""
    xs = spread_fp32(N, N * 3 * CHUNK_P, seed=700 + N)
    assert not all(torch.equal(x, x.to(torch.bfloat16).float()) for x in xs)
    check_hop_by_hop(xs, CHUNK_P, f"N={N}")


@pytest.mark.parametrize("N", range(2, 9))
def test_reference_matches_block_model_on_the_fp32_edge_payload(N):
    """NaN, +-Inf, finite top-of-range partials whose sum overflows in the add, scale byte 0, the e = 120 band,
    cancellation and one huge value among tiny ones enter every shard at every hop, at the first and last blocks of a
    panel row and of a record.  Each kind's effect is checked to be there: NaN and Inf reach the outputs, a scale byte 0
    and a block exponent of 120 appear in the records, and some output is exactly zero after a cancellation."""
    xs = edge_payload_fp32(N, seed=800 + N)
    got = check_hop_by_hop(xs, CHUNK_P, f"N={N}")
    out = torch.cat(got).float()
    assert bool(torch.isnan(out).any()) and bool(torch.isinf(out).any())
    m = xs[0].numel() // N
    scales = torch.cat([ops.ref_pack_fp8(xs[(s + 1) % N][s * m:(s + 1) * m], CHUNK_P)
                        .reshape(-1, ops.record_bytes(CHUNK_P))[:, CHUNK_P:] for s in range(N)])
    assert bool((scales == 0).any()) and bool((scales == 120 + 127).any())
