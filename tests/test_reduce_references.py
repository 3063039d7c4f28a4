"""The reference of the fp8 reduce (``ops.ref_reduce_fp8``) on the CPU: its summation order, and the quantiser rule of
DESIGN.md "fp8 numerics" applied to sums, overflow and non-finite inputs included.  tests/test_gpu_reduce.py holds the
kernel to this reference bit for bit.  Also the two things tests/test_gpu_reduce_schedule.py rests on: its model of the
reduce's step walk, against hand-counted walks, and its independent fp64 decoder, against the package's on every
(e4m3 code, scale byte) pair."""
import numpy as np
import torch

from rocnrdma_b200.ops import pack as P
from test_gpu_reduce import SOURCES
from test_gpu_reduce_schedule import (FACTS, POST_CASES, SWEEP, SWEEP_CASES, VARIANTS, WAIT_CASE,
                                      ReduceSchedule, bf16_rne_bits, decode_fp32, e4m3_fp64, independent_sum_bits,
                                      sweep_addend, sweep_records, ue8m0_fp64, variant_of)

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


# ------------------------------------------------------------------ the schedule model of the reduce
def test_reduce_schedule_variant_rule_and_grid_clamp():
    """P and the addend pick (G, PMAX) as rn_k_reduce_fp8 does; the default grid is SMs x 4, or SMs with arrival words,
    and no grid exceeds the tile count."""
    want = {False: {1: (4, 1), 2: (4, 2), 3: (2, 4), 4: (2, 4), 5: (1, 8), 6: (1, 8), 7: (1, 8), 8: (1, 8)},
            True: {1: (2, 2), 2: (2, 2), 3: (1, 8), 4: (1, 8), 5: (1, 8), 6: (1, 8), 7: (1, 8), 8: (1, 8)}}
    for local, table in want.items():
        for p, gp in table.items():
            assert variant_of(p, local) == (*gp, local), (p, local)
    assert {variant_of(p, l) for p in range(1, 9) for l in (False, True)} == set(VARIANTS)
    assert ReduceSchedule(1 << 20, 8, 2, sms=132).grid == 528
    assert ReduceSchedule(1 << 20, 8, 2, ready=True, sms=132).grid == 132
    assert ReduceSchedule(1 << 20, 1, 2, grid=200, sms=132).grid == 128      # capped at the tile count
    assert ReduceSchedule(8192, 5, 2, sms=132).grid == 5
    assert ReduceSchedule(8192, 5, 2, ready=True, grid=3).grid == 3


def test_reduce_schedule_variants_are_the_kernels():
    """VARIANTS and EF_VARIANTS are pack_fp8.cu's RN_REDUCE_VARIANTS (G, PMAX, LOCAL, EF), split by EF; a residual
    takes P = 1 without the addend and P <= 2 with it, one tile per step."""
    import re
    from pathlib import Path
    from test_gpu_reduce_schedule import EF_VARIANTS
    src = (Path(__file__).resolve().parent.parent / "rocnrdma_b200" / "csrc" / "kernels" / "pack_fp8.cu").read_text()
    body = re.search(r"#define RN_REDUCE_VARIANTS\(X\)(.*?)\n\n", src, re.S).group(1)
    xs = [(int(g), int(p), l == "true", e == "true")
          for g, p, l, e in re.findall(r"X\((\d+), (\d+), (true|false), (true|false)\)", body)]
    assert {x[:3] for x in xs if not x[3]} == set(VARIANTS) and {x[:3] for x in xs if x[3]} == set(EF_VARIANTS)
    assert variant_of(1, False, ef=True) == (1, 1, False)
    assert variant_of(1, True, ef=True) == variant_of(2, True, ef=True) == (1, 2, True)
    assert ReduceSchedule(3 * 8192, 7, 2, local=True, ready=True, ef=True).G == 1


def test_reduce_schedule_hand_counted_walks():
    # tpc 3, grid 1, G 4: one CTA, four consecutive tiles per step
    s = ReduceSchedule(24576, 5, 2, grid=1)
    assert (s.tpc, s.G, s.grid) == (3, 4, 1)
    assert s.steps == [[[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10, 11], [12, 13, 14]]]
    assert [s.runs(t) for t in s.steps[0]] == [[(0, 3), (1, 1)], [(1, 2), (2, 2)], [(2, 1), (3, 3)], [(4, 3)]]
    assert [s.waits(t) for t in s.steps[0]] == [[0, 1], [1, 2], [2, 3], [4]]
    # records 0 and 1 finish in steps 0 and 1; step 2 finishes records 2 and 3 at once
    assert s.completing_steps() == {(0, 0): {0}, (0, 1): {1}, (0, 2): {2, 3}, (0, 3): {4}}
    # tpc 5, grid 2, G 2 (P = 1 with the addend): tiles two apart, so CTAs 0 and 1 share every record
    s = ReduceSchedule(40960, 6, 1, local=True, grid=2)
    assert (s.tpc, s.G) == (5, 2)
    assert s.steps[0][:3] == [[0, 2], [4, 6], [8, 10]] and s.steps[1][:3] == [[1, 3], [5, 7], [9, 11]]
    assert [s.runs(t) for t in s.steps[0][:3]] == [[(0, 2)], [(0, 1), (1, 1)], [(1, 1), (2, 1)]]
    assert s.steps[0][-1] == [28] and s.steps[1][-1] == [29]                 # 30 tiles: both last steps are short
    assert all(c == {0, 1} for c in s.owners().values()) and s.completing_steps() == {}
    # G 1: one tile per step, grid apart
    s = ReduceSchedule(1 << 20, 2, 8, grid=100)
    assert s.G == 1 and s.steps[3][:3] == [[3], [103], [203]] and len(s.steps[55]) == 3 and len(s.steps[56]) == 2


def test_reduce_schedule_cases_exercise_what_they_claim():
    """The posting cases of test_gpu_reduce_schedule.py, each with the facts it is there for; together they cover every
    fact, every G and both widths."""
    claims = [
        {"multi_tile_run", "boundary_in_step", "step_completes_two", "record_owned_by_one_cta", "partial_last_step",
         "waits_on_a_later_record"},
        {"multi_tile_run", "record_shared", "partial_last_step", "waits_on_a_later_record"},
        {"multi_tile_run", "record_shared"},
        {"record_shared"},
        {"multi_tile_run", "boundary_in_step", "record_shared", "partial_last_step", "waits_on_a_later_record"},
    ]
    assert len(claims) == len(POST_CASES)
    seen, gs, widths = set(), set(), set()
    for (chunk, n_rec, n_src, local, grid, _), want in zip(POST_CASES, claims):
        for ready in (False, True):
            s = ReduceSchedule(chunk, n_rec, n_src, local, grid, ready=ready)
            f = s.facts()
            assert s.grid == grid and {k for k in FACTS if f[k]} == want, (chunk, n_rec, n_src, local, grid, f)
        seen |= want
        gs.add(s.G)
        widths.add(f["full_width"])
        assert 5 <= n_rec <= 7 and s.tpc in (3, 5, 6, 128) and n_rec % 4, "signal_every 4 must not divide the records"
    assert seen == set(FACTS) and gs == {1, 2, 4} and widths == {False, True}
    assert any(o for *_, o in POST_CASES), "one case lands its records at a nonzero offset"
    chunk, n_rec, n_src, grid = WAIT_CASE
    s = ReduceSchedule(chunk, n_rec, n_src, False, grid, ready=True)
    assert s.G == 4 and s.waits(s.steps[0][0]) == [0, 1]


def test_every_variant_runs_at_full_and_partial_width():
    """test_reduce_matches_reference's P, with and without the addend, reach every variant at P = PMAX, and at P < PMAX wherever
    the variant rule sends a smaller P to it (not (4, 1) or (4, 2) without the addend: P = 1 and P = 2 have their own)."""
    runs = {(p, l) for p in SOURCES for l in (False, True)}
    for v in VARIANTS:
        g, pmax, local = v
        ps = {p for p, l in runs if variant_of(p, l) == v}
        assert pmax in ps, f"{v} never runs at full width"
        if any(variant_of(p, local) == v for p in range(1, pmax)):
            assert min(ps) < pmax, f"{v} never runs at partial width"
    assert {variant_of(p, l) for p, l in SWEEP_CASES} == {variant_of(p, l) for p in (1, 2, 3) for l in (False, True)}


# ------------------------------------------------------------------ the independent decoder
def test_independent_decoder_fields():
    assert e4m3_fp64([0x38, 0xB8, 0x7E, 0x08, 0x07, 0x01, 0x00, 0x80, 0x3C]).tolist() == \
        [1.0, -1.0, 448.0, 2.0 ** -6, 7 * 2.0 ** -9, 2.0 ** -9, 0.0, -0.0, 1.5]
    assert np.signbit(e4m3_fp64([0x80]))[0] and np.isnan(e4m3_fp64([0x7F, 0xFF])).all()
    assert ue8m0_fp64([0, 1, 127, 254, 255]).tolist() == [2.0 ** -127, 2.0 ** -126, 1.0, 2.0 ** 127, float("inf")]
    # ties to even both ways, above a tie, -Inf, fp32 max to Inf, fp32 subnormals: one bf16 ulp, a tie, below half an ulp
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -8 + 2 ** -20, -np.inf, np.finfo(np.float32).max,
                  2.0 ** -133, 3 * 2.0 ** -134, 2.0 ** -140], dtype=np.float32)
    assert bf16_rne_bits(x).tolist() == [0x3F80, 0x3F80, 0x3F82, 0x3F81, 0xFF80, 0x7F80, 0x0001, 0x0002, 0x0000]
    assert bf16_rne_bits(x).tolist() == torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().astype(np.uint16).tolist()
    assert (bf16_rne_bits(np.array([np.nan], dtype=np.float32))[0] & 0x7FFF) > 0x7F80


def test_independent_decoder_agrees_on_every_code_and_scale():
    """Every (e4m3 code, scale byte) pair, decoded from its bit fields in fp64, equals ``ops.pack``'s decode bit for bit,
    NaN at the same positions."""
    recs = sweep_records(1, seed=1)
    mine = decode_fp32(recs, 1, SWEEP, SWEEP)[0]
    ref = P._decode_records(recs, 1, SWEEP, SWEEP)[0].numpy()
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(mine), nan) and nan.sum() == 2 * 256 + 2        # NaN codes, and +-0 x Inf under 0xFF
    assert np.array_equal(mine[~nan].view(np.uint32), ref[~nan].view(np.uint32))
    r = recs.view(-1)
    pairs = set(zip(r[:SWEEP].tolist(), r[SWEEP:SWEEP + SWEEP // 32].repeat_interleave(32).tolist()))
    assert len(pairs) == 65536


def test_independent_sum_agrees_with_the_reference_on_the_sweep():
    """Three permuted sweeps, with and without an addend: the numpy fp32 sum rounded by bf16_rne_bits equals
    ``ref_reduce_fp8``'s bf16 sum, NaN at the same positions; and the sources are permuted differently."""
    recs = sweep_records(3, seed=2)
    assert not torch.equal(recs.view(3, -1)[0], recs.view(3, -1)[1])
    for loc in (None, sweep_addend(3)):
        want = independent_sum_bits(recs, 3, SWEEP, SWEEP, local=loc)
        y, _ = P.ref_reduce_fp8(recs, 3, SWEEP, SWEEP, local=loc)
        got = y.view(torch.int16).numpy().astype(np.uint16)
        nan = (want & 0x7FFF) > 0x7F80
        assert np.array_equal((got & 0x7FFF) > 0x7F80, nan)
        assert np.array_equal(got[~nan], want[~nan])
