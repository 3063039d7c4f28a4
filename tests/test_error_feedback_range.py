"""Error feedback at the top of the fp32 range, on the CPU: finite inputs stay finite.

At block exponent e = 120 quantisation saturates a scaled value up to 255.99 down to 240, and the residual keeps the
difference, up to FLT_MAX - 240 * 2^120.  With round-to-nearest adds the next call's ``x + r`` (or a later hop's
``addend + decoded``) overflowed to Inf, and the Inf rule turned a finite input into NaN every other call.  Every add
of an error-feedback step now saturates at +-FLT_MAX, so:

* finite inputs give finite records, finite residuals and a finite ring output on every run;
* ``decode(records) + r_out == v`` bit for bit, with v the saturated value, and ``|r_out| <= FLT_MAX - 240 * 2^120``;
* the independent ring model of test_error_feedback_references.py (its own numpy saturating add) equals
  ``ref_allreduce_fp8(residuals=)`` bit for bit on top-of-range payloads over consecutive runs.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from test_error_feedback_references import FLT_MAX, _f32_bits, _records_np, ef_add, ring_model_ef
from test_ring_fp8_references import CHUNK as EDGE_CHUNK
from test_ring_fp8_references import BF16_MAX, KINDS, assert_bits_equal, decode, edge_payload, spread

R_MAX = FLT_MAX - 240 * 2.0 ** 120                     # the largest residual the e = 120 saturation leaves
CHUNK = 8192
RUNS = 12


# ------------------------------------------------------------------ the two cases that used to give NaN
def test_bf16_max_pack_stays_finite_from_call_to_call():
    """bf16 max, packed with its own residual: call 1 leaves r = bf16 max - 240 * 2^120 ~ 2e37, and call 2's x + r used
    to overflow to Inf, so every element of call 2 decoded to NaN.  Now it saturates at FLT_MAX and decodes to
    240 * 2^120 on every call."""
    x = torch.full((CHUNK,), BF16_MAX, dtype=torch.bfloat16)
    r = torch.zeros(CHUNK)
    for call in range(3):
        recs, r = ops.ref_pack_fp8(x, CHUNK, residual=r)
        d = decode(*_records_np(recs, CHUNK, CHUNK)).reshape(-1)
        assert np.all(d == np.float32(240 * 2.0 ** 120)), f"call {call}: decoded {d[~(d == d[0])][:4]} / {d[0]}"
        assert torch.isfinite(r).all() and float(r.abs().max()) <= R_MAX, f"call {call}: residual"
    assert float(r[0]) > 0


def test_two_rank_ring_near_the_top_is_finite_on_every_run():
    """2.5e38 on rank 0 and 0.8e38 on rank 1, the same every run: the plain ring gives 3.19e38; with error feedback the
    output used to alternate between finite and NaN.  Now it is finite on all of 6 runs."""
    n = 2 * CHUNK
    xs = [torch.full((n,), 2.5e38).to(torch.bfloat16), torch.full((n,), 0.8e38).to(torch.bfloat16)]
    assert torch.isfinite(ops.ref_allreduce_fp8(xs, CHUNK).float()).all()
    res = [torch.zeros(n) for _ in xs]
    for run in range(6):
        out, res = ops.ref_allreduce_fp8(xs, CHUNK, residuals=res)
        assert torch.isfinite(out.float()).all(), f"run {run}: non-finite output"
        assert all(torch.isfinite(r).all() for r in res), f"run {run}: non-finite residual"


# ------------------------------------------------------------------ payloads
def _near_top(N, n, seed):
    """Every block near the top of the range on every rank, with a finite plain sum: magnitudes up to bf16 max / N,
    some blocks of one sign on every rank (their sums reach bf16 max), others of random signs."""
    g = torch.Generator().manual_seed(seed)
    mag = BF16_MAX / N * (0.5 + 0.5 * torch.rand(N, n, generator=g))
    same = (torch.rand(n // 32, generator=g) < 0.5).repeat_interleave(32)
    sign = torch.where(same, torch.ones(N, n), torch.randint(0, 2, (N, n), generator=g).float() * 2 - 1)
    return [(mag[q] * sign[q]).to(torch.bfloat16) for q in range(N)]


def _finite_edge(N, seed):
    """The edge payload of test_ring_fp8_references.py (records of EDGE_CHUNK) without its non-finite kinds: NaN and
    +-Inf become 0.  Its "overflow" kind stays: finite inputs whose plain sum overflows fp32, which error feedback
    saturates."""
    xs, R = edge_payload(N, seed)
    out = []
    for x in xs:
        x = x.clone()
        x[~torch.isfinite(x)] = 0
        out.append(x)
    return out, R


def _payload(kind, N):
    """(the N ranks' inputs, chunk)."""
    if kind == "spread":
        return spread(N, N * 2 * CHUNK, seed=900 + N, lo=-133, hi=120), CHUNK
    if kind == "near_top":
        return _near_top(N, N * 2 * CHUNK, seed=910 + N), CHUNK
    return _finite_edge(N, seed=920 + N)[0], EDGE_CHUNK


PAYLOADS = ["spread", "near_top", "edge_finite"]


# ------------------------------------------------------------------ finite in, finite out
def _ring_steps(xs, residuals, chunk):
    """``ref_allreduce_fp8(residuals=)`` taken apart: per (shard, hop) the records, the value v the hop quantised
    (made here with ``ef_add``), the residual it wrote and whether an add saturated.  Returns (output, new residuals,
    steps)."""
    N = len(xs)
    n = xs[0].numel()
    m = n // N
    new = [r.clone() for r in residuals]
    out = torch.empty(n, dtype=torch.bfloat16)
    steps = []
    for s in range(N):
        part = slice(s * m, (s + 1) * m)
        recs = None
        for h in range(N):
            q = (s + h) % N
            x, r_in = xs[q][part].float().numpy(), residuals[q][part].numpy()
            if h == 0:
                a = x
                recs, new[q][part] = ops.ref_pack_fp8(xs[q][part], chunk, residual=residuals[q][part])
                sat = False
            else:
                d = decode(*_records_np(recs, m, chunk)).reshape(-1)
                a = ef_add(x, d)
                with np.errstate(over="ignore"):
                    sat = bool(np.isinf(x + d).any())
                _, recs, new[q][part] = ops.ref_reduce_fp8(recs, 1, m, chunk, local=xs[q][part],
                                                           residual=residuals[q][part])
            v = ef_add(a, r_in)
            with np.errstate(over="ignore"):
                sat = sat or bool(np.isinf(a + r_in).any())
            steps.append((s, h, recs, v, new[q][part], sat))
        out[part] = ops.ref_unpack_fp8(recs, m, chunk)
    return out, new, steps


@pytest.mark.parametrize("kind", PAYLOADS)
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_finite_inputs_stay_finite_over_twelve_runs(N, kind):
    """Each rank's input held fixed for 12 runs.  Every output, every decoded record and every residual is finite,
    ``|r| <= FLT_MAX - 240 * 2^120``, and ``decode + r == v`` with v the saturated value.  The pieces put back together
    are ``ref_allreduce_fp8(residuals=)``."""
    xs, chunk = _payload(kind, N)
    assert all(torch.isfinite(x.float()).all() for x in xs)
    n = xs[0].numel()
    res = [torch.zeros(n) for _ in range(N)]
    saturated = 0
    for run in range(RUNS):
        out, new, steps = _ring_steps(xs, res, chunk)
        want, res = ops.ref_allreduce_fp8(xs, chunk, residuals=res)
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), f"run {run}: the steps are not the reference"
        for q in range(N):
            assert torch.equal(new[q].view(torch.int32), res[q].view(torch.int32)), f"run {run}: residual of rank {q}"
        assert torch.isfinite(out.float()).all(), f"run {run}: non-finite output"
        for s, h, recs, v, r, sat in steps:
            label = f"run {run} shard {s} hop {h}"
            d = decode(*_records_np(recs, v.size, chunk)).reshape(-1)
            r = r.numpy()
            assert np.isfinite(v).all() and np.isfinite(d).all() and np.isfinite(r).all(), f"{label}: non-finite"
            assert np.abs(r).max() <= R_MAX, f"{label}: |r| = {np.abs(r).max()!r} above FLT_MAX - 240 * 2^120"
            back = d + r
            bad = np.flatnonzero(_f32_bits(back) != _f32_bits(v))
            assert bad.size == 0, f"{label}: decode + r != v at {bad.size} elements, first v={v[bad[0]]!r}"
            saturated += sat
    if kind == "spread":
        assert saturated == 0
    elif kind == "edge_finite" or N <= 3:
        assert saturated > 0, "no add saturated: the rule is not exercised"


@pytest.mark.parametrize("kind", PAYLOADS)
@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_ring_model_with_saturating_adds_equals_the_reference(N, kind):
    """The independent model, its numpy saturating add included, against ``ref_allreduce_fp8(residuals=)`` over 4
    consecutive runs on the top-of-range payloads as well as the spread one: outputs and residuals bit for bit."""
    xs, chunk = _payload(kind, N)
    n = xs[0].numel()
    res_ref = [torch.zeros(n) for _ in range(N)]
    res_model = [torch.zeros(n) for _ in range(N)]
    for run in range(4):
        got, res_ref = ops.ref_allreduce_fp8(xs, chunk, residuals=res_ref)
        want, new = ring_model_ef(xs, res_model)
        res_model = [torch.from_numpy(r) for r in new]
        assert_bits_equal(got, want, f"N={N} {kind} run {run}")
        for q in range(N):
            assert np.array_equal(_f32_bits(res_ref[q].numpy()), _f32_bits(new[q])), f"run {run}: residual of rank {q}"


def test_edge_payload_keeps_its_overflow_kind():
    """The finite edge payload still holds the kind whose plain sum overflows: the plain ring makes NaN there, error
    feedback does not (the first run starts from zero residuals)."""
    assert "overflow" in KINDS
    xs, _ = _finite_edge(3, seed=923)
    plain = ops.ref_allreduce_fp8(xs, EDGE_CHUNK)
    out, _ = ops.ref_allreduce_fp8(xs, EDGE_CHUNK, residuals=[torch.zeros(xs[0].numel()) for _ in xs])
    assert bool(torch.isnan(plain.float()).any()) and bool(torch.isfinite(out.float()).all())


@pytest.mark.parametrize("op", ["pack", "reduce"])
def test_saturating_add_keeps_nan_and_inf(op):
    """Only finite operands saturate: a NaN or Inf input still gives NaN codes and a zero residual there, and a decode
    that overflows (code 448 under scale byte 254) is still Inf."""
    x = torch.zeros(CHUNK)
    x[0], x[32], x[64] = float("nan"), float("inf"), BF16_MAX
    r = torch.zeros(CHUNK)
    r[64] = 3.0e38
    if op == "pack":
        recs, r_out = ops.ref_pack_fp8(x.to(torch.bfloat16), CHUNK, residual=r)
    else:
        src = torch.zeros(ops.pack.record_bytes(CHUNK), dtype=torch.uint8)
        src[96] = 0x7E                                       # 448 ...
        src[CHUNK + 3] = 254                                 # ... under scale byte 254: 448 * 2^127 = Inf
        _, recs, r_out = ops.ref_reduce_fp8(src, 1, CHUNK, CHUNK, local=x.to(torch.bfloat16), residual=r)
    codes, sc = _records_np(recs, CHUNK, CHUNK)
    assert (codes[0, 0] & 0x7F) == 0x7F and (codes[1, 0] & 0x7F) == 0x7F
    d = decode(codes, sc)
    assert d[2, 0] == np.float32(240 * 2.0 ** 120) and float(r_out[64]) == FLT_MAX - 240 * 2.0 ** 120
    assert float(r_out[0]) == 0 and float(r_out[32]) == 0
    if op == "reduce":
        assert (codes[3, 0] & 0x7F) == 0x7F and float(r_out[96]) == 0
