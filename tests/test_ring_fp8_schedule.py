"""The fp8 ring all-reduce on the CPU: its schedule, and its reference against an independent fp64 decode chain and
against the exact sum."""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from rocnrdma_b200.ops import pack as P
from rocnrdma_b200.parallel.ring_fp8 import schedule


def _simulate(N):
    """Play every rank's schedule symbolically: a landing slot holds (shard, ranks summed in, final).  Returns what
    each rank wrote to each shard of ``out`` and which ids each rank received."""
    land = {}                                      # (rank, slot) -> (shard, tuple of ranks)
    staging = {}
    received = {q: [] for q in range(N)}
    written = {q: {} for q in range(N)}
    # the ring runs rank by rank per step index, which respects every dependency (a step reads only what an earlier
    # step index of the previous rank sent)
    steps = [schedule(q, N) for q in range(N)]
    for i in range(2 * N):
        for q in range(N):
            st = steps[q][i]
            nxt = (q + 1) % N
            if st.kind == "pack":
                payload = (st.shard, (q,))
                staging[q] = payload
            elif st.kind == "reduce":
                shard, ranks = land[(q, st.read_slot)]
                assert shard == st.shard, (N, q, st)
                assert q not in ranks
                payload = (shard, ranks + (q,))
                staging[q] = payload
            else:
                payload = land[(q, st.read_slot)] if st.read_slot is not None else staging[q]
                assert payload[0] == st.shard and sorted(payload[1]) == list(range(N)), (N, q, st, payload)
                written[q][st.shard] = payload
            if st.send_slot is not None:
                assert (nxt, st.send_slot) not in land, "a slot is written twice"
                land[(nxt, st.send_slot)] = payload
                received[nxt].append(st.send_slot)
    return written, received, land


@pytest.mark.parametrize("N", range(2, 9))
def test_schedule_sends_each_shard_through_every_rank_once(N):
    written, received, land = _simulate(N)
    R = 3
    for q in range(N):
        # every rank writes every shard of out exactly once, from the full sum
        assert sorted(written[q]) == list(range(N))
        # each rank receives every shard except the one it owns... as a partial sum (reduce-scatter) and the final
        # records of every shard except the one it finished itself (all-gather)
        slots = sorted(received[q])
        assert slots == list(range(2 * (N - 1))), (q, slots)
        got_final = {land[(q, m)][0] for m in range(N - 1, 2 * N - 2)}
        assert got_final == set(range(N)) - {(q + 1) % N}
        ids = sorted(m * R + r for m in slots for r in range(R))
        assert ids == list(range(2 * (N - 1) * R))
    # the final records of a shard are produced by one rank and every other rank receives them once
    for s in range(N):
        holders = [q for q in range(N) if any(land[(q, m)][0] == s for m in range(N - 1, 2 * N - 2))]
        assert len(holders) == N - 1


def _gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _decode64(recs, n, chunk):
    """fp64 values of K3 records from the bit fields: e4m3 (sign, 4-bit exponent, 3-bit mantissa) times 2^(byte-127)."""
    rec = P.record_bytes(chunk)
    r = recs.reshape(-1, rec).numpy()
    q = r[:, :chunk].reshape(-1).astype(np.int64)
    sc = r[:, chunk:chunk + chunk // 32].reshape(-1).astype(np.int64)
    sign = np.where(q & 0x80, -1.0, 1.0)
    e, m = (q >> 3) & 0xF, q & 7
    mag = np.where(e == 0, m / 8.0 * 2.0 ** -6, (1 + m / 8.0) * 2.0 ** (e - 7.0))
    mag = np.where((e == 15) & (m == 7), np.nan, mag)
    return sign * mag * np.repeat(2.0 ** (sc - 127.0), 32), np.repeat(sc - 127, 32)


def _xs(N, n, seed, spread=6):
    g = _gen(seed)
    out = []
    for _ in range(N):
        x = torch.randn(n, generator=g) * torch.exp2(torch.randint(-spread, spread + 1, (n // 32,), generator=g).float()).repeat_interleave(32)
        out.append(x.to(torch.bfloat16))
    return out


@pytest.mark.parametrize("N", [2, 3, 5, 8])
def test_reference_equals_an_fp64_decode_chain(N):
    chunk = 8192
    n = N * 2 * chunk
    xs = _xs(N, n, seed=N)
    got = ops.ref_allreduce_fp8(xs, chunk)
    m = n // N
    for s in range(N):
        part = slice(s * m, (s + 1) * m)
        recs = P.ref_pack_fp8(xs[s][part], chunk)
        for h in range(1, N):
            d, _ = _decode64(recs, m, chunk)
            acc = (xs[(s + h) % N][part].double().numpy().astype(np.float32)
                   + d.astype(np.float32))                       # one fp32 add: the addend first, then the records
            recs = P._quantized_records(torch.from_numpy(acc), chunk)
        d, _ = _decode64(recs, m, chunk)
        want = torch.from_numpy(d.astype(np.float32)).to(torch.bfloat16)
        assert torch.equal(got[part].view(torch.int16), want.view(torch.int16)), f"shard {s}"


@pytest.mark.parametrize("N", [2, 4, 8])
def test_reference_error_against_the_exact_sum(N):
    """Per element, |ref - exact| <= sum over hops of max(2^-4 |v_h|, 2^(e_h - 10)) plus the fp32 adds' rounding, where
    v_h is the value quantised at hop h and e_h its block's exponent (half an e4m3 ulp, normal or subnormal)."""
    chunk = 8192
    n = N * chunk
    xs = _xs(N, n, seed=100 + N)
    got = ops.ref_allreduce_fp8(xs, chunk).double().numpy()
    exact = np.sum([x.double().numpy() for x in xs], axis=0)
    m = n // N
    bound = np.zeros(n)
    for s in range(N):
        part = slice(s * m, (s + 1) * m)
        v = xs[s][part].double().numpy()
        recs = P.ref_pack_fp8(xs[s][part], chunk)
        b = np.zeros(m)
        for h in range(N):
            d, e = _decode64(recs, m, chunk)
            b += np.maximum(2.0 ** -4 * np.abs(v), 2.0 ** (e - 10.0))
            if h == N - 1:
                break
            acc = xs[(s + h + 1) % N][part].double().numpy().astype(np.float32) + d.astype(np.float32)
            b += np.abs(acc.astype(np.float64)) * 2.0 ** -24
            v = acc.astype(np.float64)
            recs = P._quantized_records(torch.from_numpy(acc), chunk)
        bound[part] = b
    err = np.abs(got - exact)
    assert np.all(err <= bound), f"max excess {np.max(err - bound)}"
    assert np.max(err / np.maximum(bound, 1e-300)) > 0.01, "the bound is never approached: the check is vacuous"


# ------------------------------------------------------------------ the forwarding unpack's walk (test_gpu_ring_fp8_shapes.py)
def test_unpack_schedule_hand_counted_walks():
    from test_gpu_ring_fp8_shapes import UnpackSchedule
    # tpc 3, R 5, grid 1: one CTA, four consecutive tiles per step; it visits records (0, 1), (1, 2), (2, 3), (4)
    s = UnpackSchedule(3 * 8192, 5, 1)
    assert s.steps == [[[0, 1, 2, 3], [4, 5, 6, 7], [8, 9, 10, 11], [12, 13, 14]]]
    assert [s.visits(t) for t in s.steps[0]] == [[0, 1], [1, 2], [2, 3], [4]]
    assert s.sure_claims() == {(0, 0): {0, 1}, (0, 1): {2}, (0, 2): {3}, (0, 3): {4}}
    # tpc 5, R 4, grid 2: tiles two apart, so both CTAs hold every record and race to claim it
    s = UnpackSchedule(5 * 8192, 4, 2)
    assert s.steps[0] == [[0, 2, 4, 6], [8, 10, 12, 14], [16, 18]] and s.steps[1][0] == [1, 3, 5, 7]
    assert [s.visits(t) for t in s.steps[0]] == [[0, 1], [1, 2], [3]]
    assert all(c == {0, 1} for c in s.owners().values()) and s.sure_claims() == {}
    # the grid clamps to one slot's tile count; the default is one CTA per SM
    s = UnpackSchedule(8192, 2, 7)
    assert (s.grid, s.steps) == (2, [[[0]], [[1]]]) and s.facts()["clamped_grid"]
    assert UnpackSchedule(1 << 20, 2, sms=132).grid == 132 and not UnpackSchedule(1 << 20, 2, sms=132).facts()["clamped_grid"]
    # tpc 1, R 7, grid 1: one step claims four records, the next three
    s = UnpackSchedule(8192, 7, 1)
    assert s.sure_claims() == {(0, 0): {0, 1, 2, 3}, (0, 1): {4, 5, 6}}


def test_ring_geometry_cases_cover_every_fact_and_parameter():
    """The GPU geometry cases: each asserts its facts at run time; together they exercise every fact of the forwarding
    unpack, every N with a multi-tile R > 1 case, and every listed value of tiles per record, R, grid and signal_every."""
    from test_gpu_ring_fp8_shapes import GEOMETRY_CASES, UNPACK_FACTS, case_facts, ring_grid
    seen = set()
    for (N, tpc, R, grid, sig), u, r in GEOMETRY_CASES:
        assert case_facts(N, tpc, R, grid) == (u, r), (N, tpc, R, grid)
        assert 16 + N * (ring_grid(N, grid) + 1) <= 132, "SM budget"
        seen |= u
    assert seen == set(UNPACK_FACTS)
    cases = [c for c, _, _ in GEOMETRY_CASES]
    assert {N for N, tpc, R, _, _ in cases if tpc > 1 and R > 1} == set(range(2, 9))
    assert {c[1] for c in cases} == {1, 3, 5, 8, 128} and {c[2] for c in cases} == {1, 2, 4, 5, 7}
    assert {1, 2, 3, 7, 0} <= {c[3] for c in cases}
    assert any(grid > R * tpc for _, tpc, R, grid, _ in cases), "a grid larger than the slot's tile count"
    assert {1, 3} <= {c[4] for c in cases} and any(sig > R for _, _, R, _, sig in cases)
