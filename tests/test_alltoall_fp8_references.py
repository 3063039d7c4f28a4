"""The fp8 all-to-all's reference held to an independent model, and its exact operands, on the CPU.

``ops.ref_alltoall_fp8`` is built from ``ref_pack_fp8`` and ``ref_unpack_fp8``.  Here it is held to
test_ring_fp8_references.py's ``encode`` / ``decode``, which share nothing with the package's quantiser, for N = 2..8 on
spread payloads and on the edge payload (NaN, +-Inf, blocks that overflow, bf16 max, bf16 subnormals, zeros): rank q's
output and landed records must be every source's shard q, encoded block by block and decoded, in source order.  NaN
codes are compared without their sign.  The exact shards of test_allgather_fp8_references.py (integers in [-4, 4] times
2^e per block) pass through the all-to-all unchanged, which is what lets the GPU test compare K7's C bit for bit.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from test_allgather_fp8_references import exact_shard, record_fields
from test_gpu_reduce_schedule import bf16_rne_bits
from test_ring_fp8_references import CHUNK, assert_bits_equal, decode, edge_payload, encode, spread


def model_alltoall(xs, q):
    """(bf16 bits, codes, scale bytes) of what rank q holds in the independent model: shard q of every source, in
    source order, every block encoded on its own and decoded."""
    N = len(xs)
    m = xs[0].numel() // N
    x = np.concatenate([t.float().numpy().reshape(-1)[q * m:(q + 1) * m] for t in xs]).reshape(-1, 32)
    codes, sc = encode(x)
    return bf16_rne_bits(decode(codes, sc)).reshape(-1), codes, sc


def _check_against_model(xs, chunk, label):
    outs, recs = ops.ref_alltoall_fp8(xs, chunk)
    assert len(outs) == len(recs) == len(xs)
    for q in range(len(xs)):
        bits, codes, sc = model_alltoall(xs, q)
        assert_bits_equal(outs[q], bits, f"{label} rank {q}")
        c, s = record_fields(recs[q], chunk, 32)
        c = c.numpy().reshape(codes.shape)
        nan = (codes & 0x7F) == 0x7F
        assert np.array_equal((c & 0x7F) == 0x7F, nan), f"{label} rank {q}: NaN codes at other positions"
        assert np.array_equal(c[~nan], codes[~nan]), f"{label} rank {q}: codes differ"
        assert np.array_equal(s.numpy().reshape(-1), sc), f"{label} rank {q}: scale bytes differ"
    return outs


@pytest.mark.parametrize("N", range(2, 9))
def test_ref_alltoall_equals_the_model_on_spread_payloads(N):
    chunk = 8192
    _check_against_model(spread(N, N * 2 * chunk, seed=900 + N, lo=-133, hi=120), chunk, f"N={N}")


@pytest.mark.parametrize("N", range(2, 9))
def test_ref_alltoall_equals_the_model_on_the_edge_payload(N):
    xs, _ = edge_payload(N, seed=920 + N)
    outs = _check_against_model(xs, CHUNK, f"N={N}")
    assert bool(torch.isnan(torch.cat(xs)).any()) and bool(torch.isinf(torch.cat(xs)).any())
    assert any(bool(torch.isnan(o).any()) for o in outs), "the NaN blocks did not reach any output"


def test_ref_alltoall_moves_shard_q_of_rank_s_to_slot_s_of_rank_q():
    """Shards of distinct constant values that e4m3 holds exactly, (2d + 1) * 16^s: rank q's slot s holds exactly rank
    s's shard q."""
    N, chunk = 4, 8192
    val = lambda s, d: float((2 * d + 1) * 16 ** s)  # noqa: E731
    xs = [torch.cat([torch.full((chunk,), val(s, d), dtype=torch.bfloat16) for d in range(N)]) for s in range(N)]
    outs, _ = ops.ref_alltoall_fp8(xs, chunk)
    for q in range(N):
        for s in range(N):
            assert torch.all(outs[q][s * chunk:(s + 1) * chunk] == val(s, q))


@pytest.mark.parametrize("N", [2, 3, 8])
def test_exact_shards_pass_through_unchanged(N):
    """Integers in [-4, 4] times 2^e per block: every rank's output is exactly the sources' shards, so K7 on the landed
    records sees the operands it would see without the fp8 wire."""
    rows, K, chunk = 128, 256, 128 * 256
    g = torch.Generator().manual_seed(940 + N)
    xs = [exact_shard(N * rows, K, g).reshape(-1) for _ in range(N)]
    outs, _ = ops.ref_alltoall_fp8(xs, chunk)
    m = rows * K
    for q in range(N):
        want = torch.cat([x[q * m:(q + 1) * m] for x in xs])
        assert torch.equal(outs[q].view(torch.int16), want.view(torch.int16))
