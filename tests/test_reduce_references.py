"""The reference of the fp8 reduce (``ops.ref_reduce_fp8``) on the CPU: its summation order, and the quantiser rule of
DESIGN.md "fp8 numerics" applied to sums, overflow and non-finite inputs included.  tests/test_gpu_reduce.py holds the
kernel to this reference bit for bit."""
import torch

from rocnrdma_b200.ops import pack as P

CHUNK = 8192
NAN_CODE = 0x7F


def _records(codes, scales):
    """Source-major K3 records from e4m3 codes [P, n] and scale bytes [P, n / 32] (uint8)."""
    n_src, n = codes.shape
    n_rec = n // CHUNK
    rec = torch.zeros(n_src, n_rec, P.record_bytes(CHUNK), dtype=torch.uint8)
    rec[:, :, :CHUNK] = codes.reshape(n_src, n_rec, CHUNK)
    rec[:, :, CHUNK:CHUNK + CHUNK // 32] = scales.reshape(n_src, n_rec, CHUNK // 32)
    return rec.reshape(-1)


def _blank(n_src, n=CHUNK):
    """All-zero codes under scale byte 127 (so 1.0 is code 0x38)."""
    return torch.zeros(n_src, n, dtype=torch.uint8), torch.full((n_src, n // 32), 127, dtype=torch.uint8)


def _decoded(records, n_elems):
    """fp32 values of one source's records, as every decoder reads them."""
    return P._decode_records(records, 1, n_elems, CHUNK)[0]


def _seeded_bf16(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g) * torch.exp2(torch.randint(-20, 20, (n // 32,), generator=g).float()).repeat_interleave(32)
    return x.to(torch.bfloat16)


def test_one_source_without_addend_is_the_unpack():
    n = 3 * CHUNK
    recs = P.ref_pack_fp8(_seeded_bf16(n, 1), CHUNK)
    y, _ = P.ref_reduce_fp8(recs, 1, n, CHUNK)
    assert torch.equal(y.view(torch.int16), P.ref_unpack_fp8(recs, n, CHUNK).view(torch.int16))


def test_requantising_one_source_gives_back_its_values():
    """K3's records decode to values that the quantiser maps back to themselves: re-quantising a decoded block is exact."""
    n = 4 * CHUNK
    x = _seeded_bf16(n, 2)
    x[:64] = 0.0                                                          # all-zero blocks (scale byte 0x00)
    x[64:96] = 2.0 ** -133                                                # bf16 subnormals
    recs = P.ref_pack_fp8(x, CHUNK)
    _, again = P.ref_reduce_fp8(recs, 1, n, CHUNK)
    assert torch.equal(_decoded(again, n), _decoded(recs, n))


def test_sum_order_is_local_then_sources_in_order():
    """2^24, 1 and -2^24: (2^24 + 1) rounds to 2^24 in fp32 (a tie, to even), so adding in source order gives 0, where
    2^24 + (1 - 2^24) would give 1.  The same with 2^24 as the bf16 addend and the other two as sources."""
    codes, scales = _blank(3)
    codes[:, 0] = torch.tensor([0x38, 0x38, 0xB8], dtype=torch.uint8)       # +1, +1, -1
    scales[:, 0] = torch.tensor([127 + 24, 127, 127 + 24], dtype=torch.uint8)
    a, b, c = torch.tensor(2.0 ** 24), torch.tensor(1.0), torch.tensor(-(2.0 ** 24))
    assert (a + b) + c == 0 and a + (b + c) == 1, "the case does not separate the two orders"
    y, recs = P.ref_reduce_fp8(_records(codes, scales), 3, CHUNK, CHUNK)
    assert y[0].item() == 0.0 and _decoded(recs, CHUNK)[0].item() == 0.0
    local = torch.zeros(CHUNK, dtype=torch.bfloat16)
    local[0] = 2.0 ** 24
    y, _ = P.ref_reduce_fp8(_records(codes[1:], scales[1:]), 2, CHUNK, CHUNK, local=local)
    assert y[0].item() == 0.0
    assert not bool(y[1:].ne(0).any())


def test_finite_sum_that_overflows():
    """1.5 * 2^127 twice: each decodes exactly, their fp32 sum overflows to +Inf.  The block of the sum gets scale byte
    254; the Inf becomes NaN and its finite neighbours +-0.  The bf16 sum keeps the Inf."""
    codes, scales = _blank(2)
    codes[:, 0] = 0x3C                                                    # 1.5
    codes[0, 1], codes[0, 2] = 0x38, 0xB8                                 # 2^127 and -2^127 in source 0 only
    scales[:, 0] = 254
    y, recs = P.ref_reduce_fp8(_records(codes, scales), 2, CHUNK, CHUNK)
    assert y[0].item() == float("inf") and y[1].item() == 2.0 ** 127 and y[2].item() == -(2.0 ** 127)
    r = recs.reshape(-1)
    assert r[CHUNK].item() == 254, "scale byte of the overflowing block"
    assert r[0].item() & 0x7F == NAN_CODE, "the Inf is NaN in the records"
    assert r[1].item() == 0x00 and r[2].item() == 0x80, "its neighbours are +0 and -0"
    assert r[CHUNK + 1].item() == 0, "the next block is all zero"


def test_nan_and_inf_inputs():
    """A NaN code stays NaN in the sum and takes no part in its block's scale; scale byte 0xFF decodes as Inf (a zero code
    as NaN); Inf + -Inf is NaN; a block holding Inf is re-quantised with scale byte 254."""
    codes, scales = _blank(2)
    # block 0: a NaN in source 0, 1.0 elsewhere in both sources -> sum 2.0, scale 2^-7 (byte 120), code 256 = 0x78
    codes[:, :32] = 0x38
    codes[0, 2] = NAN_CODE
    # block 1: source 0 under scale byte 0xFF: +Inf at 32, NaN (zero code) at 33..63; source 1 adds -Inf at 32
    codes[0, 32] = 0x38
    scales[0, 1] = 0xFF
    codes[1, 32] = 0xB8
    scales[1, 1] = 0xFF
    codes[1, 33:64] = 0x38
    # block 2: +Inf from scale 0xFF in source 1 next to finite values of source 0
    codes[0, 64:96] = 0x40                                                # 2.0
    codes[1, 64] = 0x38
    scales[1, 2] = 0xFF
    y, recs = P.ref_reduce_fp8(_records(codes, scales), 2, CHUNK, CHUNK)
    yf = y.float()
    assert torch.isnan(yf[2]) and bool((yf[:2] == 2.0).all()) and bool((yf[3:32] == 2.0).all())
    assert bool(torch.isnan(yf[32:64]).all()), "Inf + -Inf, and NaN from a zero code under 0xFF"
    assert yf[64].item() == float("inf")
    assert bool(torch.isnan(yf[65:96]).all()), "0 * Inf under scale byte 0xFF is NaN"
    r = recs.reshape(-1)
    sc = r[CHUNK:CHUNK + 3].tolist()
    assert sc[0] == 120 and r[0].item() == 0x78 and r[2].item() & 0x7F == NAN_CODE, (sc, r[:4].tolist())
    assert sc[1] == 0, "an all-NaN block gets scale byte 0x00"
    assert sc[2] == 254 and r[64].item() & 0x7F == NAN_CODE, "a block holding Inf: scale byte 254, the Inf is NaN"


def test_reference_follows_the_documented_sum_on_random_sources():
    """Several sources and an addend: the reference equals the sum written out element by element in fp32."""
    n, n_src = 2 * CHUNK, 5
    recs = torch.cat([P.ref_pack_fp8(_seeded_bf16(n, 10 + s), CHUNK) for s in range(n_src)])
    local = _seeded_bf16(n, 9)
    y, out = P.ref_reduce_fp8(recs, n_src, n, CHUNK, local=local)
    d = P._decode_records(recs, n_src, n, CHUNK)
    acc = local.float()
    for s in range(n_src):
        acc = acc + d[s]
    assert torch.equal(y.view(torch.int16), acc.to(torch.bfloat16).view(torch.int16))
    assert torch.equal(out, P._quantized_records(acc, CHUNK))               # the records quantise the fp32 sum, not y
