"""CPU checks of the fp8 references' edge rules (NaN, +-Inf, scale bytes 0x00 / 0xFF), of their finite behaviour against
the formulas they had before the rules were added, and of the schedule models (stream-K, and both GEMMs' tile loops) the
GPU numerics tests choose their cases with."""
import itertools

import pytest
import torch

from rocnrdma_b200.ops import gemm as G
from rocnrdma_b200.ops import gemm_mx as MX
from rocnrdma_b200.ops import pack as P
from test_gpu_gemm_scale import K4_SCALE_CASES, K7_SCALE_CASES, Schedule
from test_gpu_numerics import STREAM_K_CASES, StreamK

NAN, INF = float("nan"), float("inf")


def _block(vals):
    return torch.tensor(vals + [0.0] * (32 - len(vals)), dtype=torch.float32)


def _quantisers():
    """(name, quantise(x [rows, 32] fp32) -> (codes [rows, 32], scale bytes [rows])) for the three producers' references."""
    def pack(x):
        rec = P.ref_pack_fp8(torch.cat([x, torch.zeros(8192 - x.shape[0], 32)]).to(torch.bfloat16).reshape(-1), 8192)
        return rec[:8192].reshape(256, 32)[:x.shape[0]], rec[8192:8192 + 256][:x.shape[0]]

    def mx(x):
        q, s = MX.quantize_mx(x)
        return q, s.reshape(-1)

    def panels(x):
        rec = G.ref_fp8_panels(x)
        return rec[:128 * 32].reshape(128, 32)[:x.shape[0]], rec[128 * 32:].reshape(128)[:x.shape[0]]
    return [("ref_pack_fp8", pack), ("quantize_mx", mx), ("ref_fp8_panels", panels)]


QUANTISERS = _quantisers()


@pytest.mark.parametrize("name,quant", QUANTISERS, ids=[q[0] for q in QUANTISERS])
def test_nan_stays_in_its_element(name, quant):
    x = torch.stack([_block([NAN, 3.0, 0.0, -1.25]), _block([NAN] * 32), _block([3.0, 0.0, -1.25])])
    q, s = quant(x)
    assert int(s[0]) == int(s[2]) == 120, s                      # 3.0 / 448 -> 2^-7: the NaN takes no part in the amax
    assert torch.equal(q[0, 1:4], q[2, :3])                     # the neighbours quantise as if the NaN were absent
    assert int(q[0, 0]) & 0x7F == 0x7F                           # e4m3 NaN
    assert int(s[1]) == 0 and torch.all((q[1] & 0x7F) == 0x7F)   # all NaN: amax 0 -> scale byte 0, every code NaN


@pytest.mark.parametrize("name,quant", QUANTISERS, ids=[q[0] for q in QUANTISERS])
@pytest.mark.parametrize("inf", [INF, -INF])
def test_inf_block_gets_scale_254_and_loses_its_neighbours(name, quant, inf):
    x = torch.stack([_block([1.0, inf, -2.0, 448.0, -0.0])])
    q, s = quant(x)
    assert int(s[0]) == 254
    assert int(q[0, 1]) & 0x7F == 0x7F                           # Inf * 0.0 = NaN
    assert int(q[0, 0]) == 0x00 and int(q[0, 2]) == 0x80 and int(q[0, 3]) == 0x00 and int(q[0, 4]) == 0x80   # +-0


def test_decoders_read_scale_byte_0_as_2_to_minus_127_and_255_as_inf():
    codes = torch.tensor([0x38, 0xB8, 0x08, 0x00], dtype=torch.uint8)          # 1.0, -1.0, 2^-6 * 1.0 ... as e4m3: 0x08 = 2^-6, 0
    vals = codes.view(torch.float8_e4m3fn).double()
    for byte, scale in ((0x00, 2.0 ** -127), (0x01, 2.0 ** -126), (0xFE, 2.0 ** 127), (0x7F, 1.0)):
        want = (vals * scale).float()
        q = torch.zeros(1, 32, dtype=torch.uint8); q[0, :4] = codes
        s = torch.full((1, 1), byte, dtype=torch.uint8)
        assert torch.equal(MX.dequantize_mx(q, s)[0, :4], want), byte
        rec = torch.zeros(G.panel_record_bytes(32), dtype=torch.uint8)
        rec[:32] = q[0]
        rec[128 * 32] = byte
        assert torch.equal(G.dequant_fp8_panels(rec, 1, 32)[0, :4], want), byte
        crec = torch.zeros(P.record_bytes(8192), dtype=torch.uint8)
        crec[:32] = q[0]
        crec[8192] = byte
        assert torch.equal(P.ref_unpack_fp8(crec, 8192, 8192)[:4], want.to(torch.bfloat16)), byte
    assert P.ue8m0(torch.tensor([0], dtype=torch.uint8)).view(torch.int32).item() == 0x00400000
    inf = MX.dequantize_mx(torch.tensor([[0x38, 0xB8, 0x00] + [0] * 29], dtype=torch.uint8), torch.tensor([[0xFF]], dtype=torch.uint8))[0]
    assert inf[0].item() == INF and inf[1].item() == -INF and torch.isnan(inf[2])   # 0xFF = 2^128: q * Inf


# ------------------------------------------------------------------ finite data: unchanged against the earlier formulas
def _old_scale_exponent(amax):
    v = (amax.float() * (1.0 / 448.0)).contiguous()
    bits = v.view(torch.int32)
    e = ((bits >> 23) & 0xFF) - 127 + ((bits & 0x7FFFFF) != 0).to(torch.int32)
    return e.clamp(-127, 127)


def _old_pow2(e):
    return ((e + 127).to(torch.int32) << 23).view(torch.float32)


def _old_quantize(x):
    e = _old_scale_exponent(x.abs().amax(dim=-1))
    return (x * _old_pow2(-e)[..., None]).to(torch.float8_e4m3fn).view(torch.uint8), (e + 127).to(torch.uint8)


def _old_dequantize(q, s):
    return q.view(torch.float8_e4m3fn).float() * _old_pow2(s.to(torch.int32) - 127)[..., None]


def test_finite_data_is_quantised_as_before_except_at_both_ends_of_the_range():
    """Every block quantises as the earlier formulas did, except the two whose rule changed on purpose: a value near
    bf16 max under scale 2^120 (code 256 there decodes to Inf; now 240) and a bf16-subnormal block (scale 2^-126 before,
    now the smallest, 2^-127)."""
    g = torch.Generator().manual_seed(0)
    M, K = 384, 256
    x = torch.randn(M, K, generator=g) * torch.exp2(torch.randint(-40, 40, (M, K // 32, 1), generator=g).float()).expand(M, K // 32, 32).reshape(M, K)
    x[0] = 0.0
    x[1, :32] = 448.0
    x[2, :32] = torch.finfo(torch.bfloat16).max
    x[3, :32] = 2.0 ** -133
    x = x.to(torch.bfloat16)
    blocks = x.float().reshape(M, K // 32, 32)
    q0, s0 = _old_quantize(blocks)
    q, s = MX.quantize_mx(x)
    # the rule changed on purpose in two blocks (DESIGN.md "fp8 numerics"): bf16 max under scale 2^120 no longer rounds
    # to code 256, which decodes to 2^128 = Inf, but saturates to 240; and amax 2^-133, whose amax / 448 is below
    # 2^-127, takes the smallest scale 2^-127 (byte 0) where the old rule took 2^-126
    changed = torch.zeros(M, K // 32, dtype=torch.bool)
    changed[2, 0] = changed[3, 0] = True
    qb = q.reshape(M, K // 32, 32)
    assert torch.equal(qb[~changed], q0[~changed]) and torch.equal(s[~changed], s0[~changed])
    assert (s0[2, 0].item(), s[2, 0].item()) == (247, 247)
    assert bool((q0[2, 0] == 0x78).all()) and bool((qb[2, 0] == 0x77).all())
    assert (s0[3, 0].item(), s[3, 0].item()) == (1, 0)
    assert bool((q0[3, 0] == 0x04).all()) and bool((qb[3, 0] == 0x08).all())
    assert bool(torch.isfinite(MX.dequantize_mx(q, s)).all())
    rec = G.ref_fp8_panels(x.float()).reshape(M // 128, -1)
    assert torch.equal(rec[:, :128 * K].reshape(M, K), q) and torch.equal(rec[:, 128 * K:].reshape(M, K // 32), s)
    chunk = 128 * K
    crec = P.ref_pack_fp8(x.reshape(-1), chunk).reshape(M // 128, -1)
    assert torch.equal(crec[:, :chunk].reshape(M, K), q) and torch.equal(crec[:, chunk:chunk + chunk // 32].reshape(M, K // 32), s)
    # decoders: identical wherever the scale byte is not 0 (the old rule emitted 0 only for all-zero blocks)
    old = _old_dequantize(q0, s0).reshape(M, K)
    q0, s0 = q0.reshape(M, K), s0
    assert torch.equal(MX.dequantize_mx(q0, s0), old)
    rec0 = torch.cat([q0.reshape(M // 128, -1), s0.reshape(M // 128, -1)], dim=1)
    assert torch.equal(G.dequant_fp8_panels(rec0.reshape(-1), M, K), old)
    crec0 = torch.zeros_like(crec)
    crec0[:, :chunk], crec0[:, chunk:chunk + chunk // 32] = q0.reshape(M // 128, -1), s0.reshape(M // 128, -1)
    assert torch.equal(P.ref_unpack_fp8(crec0.reshape(-1), M * K, chunk).reshape(M, K), old.to(torch.bfloat16))


# ------------------------------------------------------------------ the stream-K schedule model
def _check_model(m):
    covered = [[0] * m.k_blks for _ in range(m.R)]
    per_unit = {}
    for u, j, kb0, kb1 in m.segs:
        assert 0 <= kb0 < kb1 <= m.k_blks
        for kb in range(kb0, kb1):
            covered[j][kb] += 1
        per_unit.setdefault(u, []).append((j, kb0, kb1))
    if m.stream_k:
        assert all(c == 1 for row in covered for c in row), "a (tile, k-block) is computed twice or never"
    for u, segs in per_unit.items():
        # a share holds at most the tail end of one tile (parked) and then the head of the next (owned)
        assert len(segs) <= 2 and all(kb0 == 0 for _, kb0, _ in segs[1:]), (u, segs)
    for j, segs in m.tiles().items():
        owners = [s for s in segs if s[2] == 0]
        assert len(owners) == 1
        u = owners[0][0]
        contrib = sorted(s[0] for s in segs if s[2] != 0)
        assert contrib == list(range(u + 1, u + 1 + m.n_contrib(*owners[0]))), (j, u, contrib)
        for cu in contrib:
            b, e = m.share(cu)
            assert m.unit_of(b) == cu and m.unit_of(e - 1) == cu


def test_stream_k_model_covers_every_k_block_once_and_matches_unit_of():
    n = 0
    for M, N, K, grid, gm in itertools.product([100, 520, 1000, 2048], [256, 520, 1032], [8, 200, 328, 1000, 4104], [2, 5, 8, 15, 60, 132], [1, 3, 16]):
        m = StreamK(M, N, K, grid, gm)
        _check_model(m)
        n += m.stream_k
    assert n > 100


def test_stream_k_model_cases_exercise_what_they_claim():
    for case, expect in STREAM_K_CASES:
        f = StreamK(*case).facts()
        assert expect <= f, (case, f)
    seen = set().union(*(StreamK(*c).facts() for c, _ in STREAM_K_CASES))
    assert {"split", "over_m", "over_n", "over_mn", "contrib_only_k_tail", "folds_2_or_more", "odd_grid"} <= seen
    assert {c[4] for c, _ in STREAM_K_CASES} == {1, 3, 16}


def test_stream_k_flag_is_not_the_same_as_a_split():
    """12 tiles over 5 clusters with 2 k-blocks: stream-K is on, but shares would be under 4 k-blocks, so n_tail == R and
    every tail tile runs whole on one cluster."""
    m = StreamK(1024, 768, 128, 10, 1)
    assert m.stream_k and m.n_tail == m.R and not m.split_tiles()


# ------------------------------------------------------------------ both GEMMs' tile schedules (launch rule + tile loop)
def test_schedule_model_hand_counted_k4():
    # one CTA per 128 x 256 tile, 4096^3 on 132 SMs: 32 x 16 = 512 tiles, 512 = 3 * 132 + 116; k_blks = 64 = 3 * 21 + 1, so
    # a unit's tiles enter the 3-stage ring at stages 0, 1, 2, 0
    s = Schedule("k4", 4096, 4096, 4096, 1, 0)
    assert (s.grid, s.n_units, s.n_tiles, s.k_blks) == (132, 132, 512, 64)
    assert [len(u) for u in s.units].count(4) == 116 and [len(u) for u in s.units].count(3) == 16
    assert s.units[0] == [(0, 0, 64), (132, 0, 64), (264, 0, 64), (396, 0, 64)]
    assert s.entry_stages()[:3] == [1, 2, 0]
    # pair kernel at grid 13: 12 CTAs, 6 units; 8192 x 8192 pair tiles: 32 x 32 = 1024 = 170 * 6 + 4; k_blks 32 = 3 * 10 + 2
    s = Schedule("k4", 8192, 8192, 2048, 2, 13)
    assert (s.grid, s.n_units, s.ctas) == (12, 6, 2)
    assert [len(u) for u in s.units] == [171] * 4 + [170] * 2
    assert s.entry_stages()[:3] == [2, 1, 0] and not s.stream_k
    # grid clamps: past the SM count -> SMs; never more CTAs than tiles (pairs: 2 per tile); a grid of 1 is the 1-CTA kernel
    assert Schedule("k4", 300, 512, 64, 1, 200).grid == 6
    assert (Schedule("k4", 256, 256, 64, 2, 0).grid, Schedule("k4", 256, 256, 64, 2, 0).n_units) == (2, 1)
    assert Schedule("k4", 512, 256, 64, 2, 1).ctas == 1
    # stream-K, 4096^3 at grid 13: 256 pair tiles = 42 * 6 + 4, the 4 * 64 tail k-blocks dealt in shares of 42 or 43: unit 0
    # owns tile 252's first 42 k-blocks; unit 1 finishes tile 252 (22) and starts 253 (21)
    s = Schedule("k4", 4096, 4096, 4096, 3, 13, stream_k=True)
    assert s.stream_k and s.n_units == 6
    assert s.units[0][42:] == [(252, 0, 42)] and s.units[1][42:] == [(252, 42, 64), (253, 0, 21)]
    assert s.max_tiles_per_unit() == 44
    # without stream-K the same launch leaves the 4 tail tiles whole on units 0..3
    s = Schedule("k4", 4096, 4096, 4096, 3, 13)
    assert not s.stream_k and s.units[3][-1] == (255, 0, 64) and len(s.units[4]) == 42


def test_schedule_model_hand_counted_k7():
    # 128 x 128 tiles, 4096 x 4096 x 1152 at grid 13: 1024 tiles = 78 * 13 + 10; k_blks = 9 = 4 * 2 + 1: stages 1, 2, 3, 0
    s = Schedule("k7", 4096, 4096, 1152, 1, 13)
    assert (s.grid, s.n_units, s.k_blks, s.stages) == (13, 13, 9, 4)
    assert [len(u) for u in s.units] == [79] * 10 + [78] * 3
    assert s.entry_stages()[:4] == [1, 2, 3, 0]
    assert s.coords(130) == (4, 2)                                  # row-major: tile // n_blks, tile % n_blks
    # pair kernel: 256 x 128 per cluster; cta_group 0 picks it for M > 128
    s = Schedule("k7", 300, 200, 4096, 0, 0)
    assert (s.ctas, s.n_tiles, s.grid, s.n_units) == (2, 4, 8, 4)
    assert not any(Schedule("k7", 4096, 4096, 4096, cg, 13).facts()["mid_ring_entry"] for cg in (1, 2))   # k_blks % 4 == 0


def test_schedule_model_panel_races():
    # 512 x 512, one CTA per tile, group_m 1: tiles (m, n) = (t // 2, t % 2).  Grid 2: panel p completes in slot p, one
    # after another; grid 4: panels 0 and 1 complete in slot 0 on different units, in an order the schedule leaves open
    s = Schedule("k4", 512, 512, 64, 1, 2)
    assert {p: v[0] for p, v in s.panel_done_slots().items()} == {p: p for p in range(4)} and not s.panels_race()
    assert Schedule("k4", 512, 512, 64, 1, 4).panels_race()
    assert not Schedule("k4", 512, 512, 64, 1, 1).panels_race()
    assert Schedule("k4", 512, 512, 64, 2, 2).panels_race()          # a pair tile completes two panels at once


def test_scale_cases_exercise_what_they_claim():
    for (M, N, K), cg, gt in K4_SCALE_CASES:
        grid = {"default": 0, "beside_engine": 132 - 32, "small": 13}[gt]
        f = Schedule("k4", M, N, K, cg, grid, stream_k=cg == 3, group_m=8).facts()
        assert f["mid_ring_entry"] and f["max_tiles_per_unit"] >= (8 if gt == "small" else 2), (M, N, K, cg, gt, f)
        assert f["stream_k"] == (cg == 3), (M, N, K, cg, gt)
    assert {(-(-K // 64)) % 3 for (_, _, K), _, _ in K4_SCALE_CASES} == {1, 2}
    k7 = [Schedule("k7", M, N, K, cg, {"default": 0, "beside_engine": 100, "small": 13}[gt]).facts() for _, (M, N, K), cg, gt in K7_SCALE_CASES]
    assert any(f["mid_ring_entry"] for f in k7) and max(f["max_tiles_per_unit"] for f in k7) >= 8
    assert Schedule("k4", 8192, 8192, 2048, 2, 100, group_m=4).panels_race()
