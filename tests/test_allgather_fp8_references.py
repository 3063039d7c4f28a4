"""Operands whose all-gather GEMM has a known exact answer, and the gather's reference held to an independent model, on
the CPU.

* ``exact_shard`` makes bf16 shards that K3 quantises without error and that give K7 block partials of at most 11
  significant bits against ``_mx_exact_operand`` weights (integer codes in [-4, 4] under scale bytes 127 +- 3).  Each
  32-element block holds integers in [-4, 4] with at least one +-4, times 2^e with e drawn per block: its amax is
  4 * 2^e, so its scale byte is 127 + e - 6 and its codes are the integers times 64, {0, 64, 128, 192, 256} in
  magnitude.  A block partial is then at most 32 * 256 * 4 = 512 units of 64, which any MMA forms exactly, and K7's C
  must equal ``ops.ref_gemm_mxfp8`` bit for bit (test_gpu_allgather_fp8_shapes.py).
* ``ops.ref_allgather_fp8`` is built from ``ref_pack_fp8`` and ``ref_unpack_fp8``, which every pack test also uses.  Here
  it is held to test_ring_fp8_references.py's ``encode`` / ``decode``, which share nothing with the package's quantiser,
  on spread payloads and on the edge payload (NaN, +-Inf, blocks that overflow, bf16 max, bf16 subnormals, zeros), as
  gathered records and as bf16 bits.  NaN codes are compared without their sign: the hardware conversion may
  canonicalise it.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from test_gpu_reduce_schedule import bf16_rne_bits, e4m3_fp64
from test_ring_fp8_references import CHUNK, assert_bits_equal, decode, edge_payload, encode, spread

EXACT_CODES = {0.0, 64.0, 128.0, 192.0, 256.0}


# ------------------------------------------------------------------ the exact construction
def exact_shard(rows, K, g, lo=-20, hi=20):
    """bf16 [rows, K]: per 32-element block, integers in [-4, 4] with one +-4 at a random position, times 2^e with e
    uniform in [lo, hi].  K3 packs it without error (codes {0, 64, 128, 192, 256} in magnitude, scale byte 121 + e)."""
    nb = rows * K // 32
    v = torch.randint(-4, 5, (nb, 32), generator=g).float()
    pos = torch.randint(0, 32, (nb,), generator=g)
    v[torch.arange(nb), pos] = 4.0 * (torch.randint(0, 2, (nb,), generator=g) * 2 - 1).float()
    e = torch.randint(lo, hi + 1, (nb, 1), generator=g).float()
    return (v * torch.exp2(e)).reshape(rows, K).to(torch.bfloat16)


def record_fields(recs, chunk, K):
    """(codes [rows, K], scale bytes [rows, K / 32]) of K3 chunk records of a row-major [rows, K] matrix."""
    r = recs.reshape(-1, P.record_bytes(chunk))
    return r[:, :chunk].reshape(-1, K), r[:, chunk:chunk + chunk // 32].reshape(-1, K // 32)


@pytest.mark.parametrize("seed", range(3))
def test_exact_shards_decode_back_to_themselves(seed):
    """At K = 160 (five blocks a row, chunk = 256 rows): the records decode to the shard bit for bit, every code is one
    of the five multiples of 64 and the scale bytes run over 101 .. 141."""
    K, rows, chunk = 160, 512, 256 * 160
    g = torch.Generator().manual_seed(700 + seed)
    x = exact_shard(rows, K, g)
    recs = ops.ref_pack_fp8(x.reshape(-1), chunk)
    assert torch.equal(ops.ref_unpack_fp8(recs, x.numel(), chunk).view(torch.int16), x.reshape(-1).view(torch.int16))
    q, s = record_fields(recs, chunk, K)
    mags = set(np.abs(e4m3_fp64(q.numpy())).reshape(-1).tolist())
    assert mags == EXACT_CODES, mags
    assert s.min().item() == 101 and s.max().item() == 141
    # the scale byte is 121 + e: the block's amax, 4 * 2^e, is 256 under it
    amax = x.float().reshape(-1, 32).abs().amax(1)
    assert torch.equal(amax, 256.0 * torch.exp2(s.reshape(-1).double() - 127).float())


def test_exact_block_partials_fit_in_11_bits():
    """Every block partial of an exact shard's codes against ``_mx_exact_operand``'s codes (integers in [-4, 4]) is 64
    times an integer of at most 512 in magnitude: checked in integer arithmetic on a seeded sample of blocks."""
    K, rows, chunk = 256, 256, 256 * 256
    g = torch.Generator().manual_seed(710)
    q, _ = record_fields(ops.ref_pack_fp8(exact_shard(rows, K, g).reshape(-1), chunk), chunk, K)
    a = e4m3_fp64(q.numpy()).reshape(-1, 32)
    assert np.all(a == np.round(a / 64) * 64)
    a_int = (a / 64).astype(np.int64)                         # [-4, 4]
    b_int = torch.randint(-4, 5, (512, 32), generator=g).numpy().astype(np.int64)
    idx = torch.randint(0, a_int.shape[0], (2048,), generator=g).numpy()
    p = a_int[idx] @ b_int.T                                  # partials in units of 64
    assert np.abs(p).max() <= 512
    p = np.abs(p[p != 0])
    odd = p // (p & -p)                                       # the significand without its trailing zeros
    bits = np.floor(np.log2(odd)).astype(int) + 1
    assert 6 <= bits.max() <= 11, bits.max()


# ------------------------------------------------------------------ the reference against the independent model
def model_allgather(shards, chunk):
    """(bf16 bits of the gathered tensor, codes, scale bytes) of the independent model: every block encoded on its own,
    shard after shard, and decoded."""
    x = np.concatenate([t.float().numpy().reshape(-1) for t in shards]).reshape(-1, 32)
    codes, sc = encode(x)
    return bf16_rne_bits(decode(codes, sc)).reshape(-1), codes, sc


def _check_against_model(shards, chunk, label):
    out, recs = P.ref_allgather_fp8(shards, chunk)
    bits, codes, sc = model_allgather(shards, chunk)
    assert_bits_equal(out, bits, label)
    q, s = record_fields(recs, chunk, 32)
    q = q.numpy().reshape(codes.shape)
    nan = (codes & 0x7F) == 0x7F
    assert np.array_equal((q & 0x7F) == 0x7F, nan), f"{label}: NaN codes at other positions"
    assert np.array_equal(q[~nan], codes[~nan]), f"{label}: {int((q[~nan] != codes[~nan]).sum())} codes differ"
    assert np.array_equal(s.numpy().reshape(-1), sc), f"{label}: scale bytes differ"
    return out


@pytest.mark.parametrize("N", range(2, 9))
def test_ref_allgather_equals_the_model_on_spread_payloads(N):
    chunk = 8192
    _check_against_model(spread(N, 2 * chunk, seed=720 + N, lo=-133, hi=120), chunk, f"N={N}")


@pytest.mark.parametrize("N", range(2, 9))
def test_ref_allgather_equals_the_model_on_the_edge_payload(N):
    """Every edge kind at the first and last block of a record and of each of its two tiles, on every shard."""
    xs, _ = edge_payload(N, seed=740 + N)
    out = _check_against_model(xs, CHUNK, f"N={N}")
    x = torch.cat(xs)
    assert bool(torch.isnan(x).any()) and bool(torch.isinf(x).any())
    assert bool(torch.isnan(out).any()), "the NaN blocks did not reach the output"
