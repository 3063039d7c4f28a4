"""The fp8 ring reduce-scatter's reference against the independent e4m3 block model, and the layout identity between
K4's fp8 panel records and K3's chunk records that the GEMM-reduce-scatter rests on, on the CPU."""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from test_gpu_reduce_schedule import bf16_rne_bits
from test_ring_fp8_references import CHUNK, assert_bits_equal, decode, edge_payload, encode, spread


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
