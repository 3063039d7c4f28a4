"""Error feedback in the fp8 pack, reduce and ring references, on the CPU.

* Exactness: wherever the quantised value v is finite, ``decode(records) + r_out == v`` bit for bit, and ``r_out == 0``
  wherever it is not.  v is made with ``ef_add``, this file's saturating fp32 add (finite operands whose sum overflows
  give +-FLT_MAX), which shares nothing with ``ops.pack``'s -- on spread payloads and on the edge payload of test_ring_fp8_references.py (NaN, Inf, an
  overflowing sum, the 448 and e = 120 boundaries, bf16 subnormals, bf16 max).  ``decode`` is that file's independent
  decoder, not ``ops.pack``'s.
* A zero residual changes nothing but the sign of zero codes (-0 + 0 = +0).
* The independent ring model of test_ring_fp8_references.py, extended with one residual per (rank, shard), equals
  ``ref_allreduce_fp8(residuals=)`` bit for bit over consecutive runs, outputs and residuals both.
* With each rank's input held fixed, the mean output over T runs converges to the exact sum: its error is a small part
  of the (constant) error of one run without feedback, and within the telescoping bound.
"""
import numpy as np
import pytest
import torch

from rocnrdma_b200 import ops
from test_ring_fp8_references import CHUNK, assert_bits_equal, decode, edge_payload, encode, spread
from test_gpu_reduce_schedule import bf16_rne_bits


def _f32_bits(t):
    return np.asarray(t, dtype=np.float32).view(np.uint32)


FLT_MAX = float(np.finfo(np.float32).max)


def ef_add(a, b):
    """Error feedback's fp32 add: the exact sum (in fp64, which rounds to fp32 correctly for one add of fp32 operands)
    clamped to [-FLT_MAX, FLT_MAX] when both operands are finite, then rounded to fp32.  A NaN or Inf operand
    propagates as in an ordinary add."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        s = a.astype(np.float64) + b.astype(np.float64)
        s = np.where(np.isfinite(a) & np.isfinite(b), np.clip(s, -FLT_MAX, FLT_MAX), s)
        return s.astype(np.float32)


def _records_np(recs, n, chunk):
    """(codes [n / 32, 32], scale bytes [n / 32]) of K3 records."""
    r = recs.numpy().reshape(n // chunk, -1)
    return r[:, :chunk].reshape(-1, 32), r[:, chunk:chunk + chunk // 32].reshape(-1)


def _check_identity(v, recs, r_out, chunk, label):
    """decode(records) + r_out == v bit for bit where v is finite; r_out == 0 (+0) where it is not.  A label that
    starts with "spread" is a finite payload, and v must then be finite everywhere: with error feedback every add
    saturates, so finite operands never make a non-finite v.  Any other payload must hold a non-finite v to check."""
    v = np.asarray(v, dtype=np.float32).reshape(-1)
    codes, sc = _records_np(recs, v.size, chunk)
    d = decode(codes, sc).reshape(-1)
    r = r_out.numpy().reshape(-1)
    fin = np.isfinite(v)
    if label.startswith("spread"):
        assert fin.all(), f"{label}: a finite payload gave a non-finite value"
    else:
        assert (~fin).any(), f"{label}: the payload has no non-finite value to check"
    with np.errstate(over="ignore", invalid="ignore"):
        back = d + r
    bad = np.flatnonzero(fin & (_f32_bits(back) != _f32_bits(v)))
    assert bad.size == 0, f"{label}: {bad.size} elements with decode + r_out != v, first {bad[0]}: v={v[bad[0]]!r} " \
                          f"d={d[bad[0]]!r} r={r[bad[0]]!r}"
    assert np.all(_f32_bits(r[~fin]) == 0), f"{label}: a non-finite value left a nonzero residual"
    assert np.isfinite(r).all()


def _residual(n, seed, scale_lo=-30, scale_hi=-8):
    """Residual-sized values: small against the spread payloads, of either sign."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) *
            torch.exp2(torch.randint(scale_lo, scale_hi + 1, (n // 32,), generator=g).float()).repeat_interleave(32))


def _payloads():
    yield "spread", spread(3, 3 * 2 * CHUNK, seed=5, lo=-133, hi=120)
    xs, _ = edge_payload(3, seed=7)
    yield "edge", xs


# ------------------------------------------------------------------ exactness
@pytest.mark.parametrize("kind", ["spread", "edge"])
def test_pack_residual_identity(kind):
    xs = dict(_payloads())[kind]
    for q, x in enumerate(xs):
        r_in = _residual(x.numel(), 100 + q)
        if kind == "edge":                                   # residuals that push blocks over the top and back
            r_in.view(-1, 32)[::97, 1] = 3.0e38
            r_in.view(-1, 32)[::89, 2] = float("nan")
            xf = x.float()                                   # and ones whose sum with a top-of-range x overflows fp32
            top = torch.isfinite(xf) & (xf.abs() >= 1e38)
            r_in[top] = torch.copysign(torch.tensor(3.0e38), xf[top])
        recs, r_out = ops.ref_pack_fp8(x, CHUNK, residual=r_in)
        # the records quantise x + r_in added with saturation: where both are finite and the sum overflows fp32 (bf16
        # max plus 3e38), v is +-FLT_MAX, not +-Inf
        v = ef_add(x.float().numpy(), r_in.numpy())
        if kind == "edge":
            with np.errstate(over="ignore", invalid="ignore"):
                plain = x.float().numpy() + r_in.numpy()
            assert (np.isinf(plain) & (np.abs(v) == FLT_MAX)).any(), "no add saturated: the rule is not exercised"
        assert torch.equal(recs, ops.ref_pack_fp8(torch.from_numpy(v), CHUNK)), "the records quantise ef_add(x, r_in)"
        _check_identity(v, recs, r_out, CHUNK, f"{kind} pack rank {q}")


# With an addend, the edge payload's "overflow" kind makes the addend's sum overflow fp32, and error feedback saturates
# that add at +-FLT_MAX: those cases are "edge_saturating".  At P = 1 without the addend nothing saturates.
REDUCE_IDENTITY_CASES = [(1, True, "spread"), (1, True, "edge_saturating"), (1, False, "spread"), (1, False, "edge"),
                         (2, True, "spread"), (2, True, "edge_saturating")]


@pytest.mark.parametrize("n_src,with_local,kind", REDUCE_IDENTITY_CASES)
def test_reduce_residual_identity(kind, n_src, with_local):
    """The residual is added last, after the addend and every source; the bf16 output is that value, rounded.  Every
    add saturates (``ef_add``): where finite operands overflow fp32, v is +-FLT_MAX and quantises finite."""
    xs = dict(_payloads())[kind.removesuffix("_saturating")]
    n = xs[0].numel()
    recs = torch.cat([ops.ref_pack_fp8(xs[s], CHUNK) for s in range(n_src)])
    local = xs[2] if with_local else None
    r_in = _residual(n, 200 + n_src)
    y, out, r_out = ops.ref_reduce_fp8(recs, n_src, n, CHUNK, local=local, residual=r_in)
    codes = [_records_np(recs[s * len(recs) // n_src:(s + 1) * len(recs) // n_src], n, CHUNK) for s in range(n_src)]
    with np.errstate(over="ignore", invalid="ignore"):
        dec = [decode(c, sc).reshape(-1) for c, sc in codes]
        v = local.float().numpy() if with_local else dec[0]
        for d in (dec if with_local else dec[1:]):
            v = ef_add(v, d)
        v = ef_add(v, r_in.numpy())
    saturated = np.abs(v) == np.float32(FLT_MAX)
    assert saturated.any() == kind.endswith("_saturating"), "saturation where the case does not expect it, or none"
    assert np.isfinite(decode(*_records_np(out, n, CHUNK)).reshape(-1)[saturated]).all(), "a saturated value decoded non-finite"
    assert_bits_equal(y, bf16_rne_bits(v), "out is v rounded to bf16")
    _check_identity(v, out, r_out, CHUNK, f"{kind} reduce P={n_src} local={with_local}")


@pytest.mark.parametrize("v", [448.0, 449.0, 3.3e38, float(np.finfo(np.float32).max), 2.0 ** -133, 2.0 ** -149,
                               -255.99 * 2.0 ** 120])
def test_identity_at_the_boundaries(v):
    """One value per block beside small neighbours: the 448 clamp, the e = 120 saturation (255.99 -> 240), an e4m3
    subnormal under e = -127 and an fp32 denormal; |d| <= 2|v| and the difference is exact."""
    x = np.zeros(CHUNK, np.float32)
    x.reshape(-1, 32)[:, 0] = v
    x.reshape(-1, 32)[:, 1:] = np.float32(v) * np.float32(2.0 ** -7) * np.linspace(-1, 1, 31, dtype=np.float32)
    recs, r = ops.ref_pack_fp8(torch.zeros(CHUNK, dtype=torch.bfloat16), CHUNK, residual=torch.from_numpy(x))
    v = np.zeros(CHUNK, np.float32) + x                      # what is quantised: 0 + x (-0 becomes +0)
    _check_identity(v, recs, r, CHUNK, "spread boundary")
    d = decode(*_records_np(recs, CHUNK, CHUNK)).reshape(-1).astype(np.float64)
    nz = d != 0
    assert np.all(np.abs(d[nz]) <= 2 * np.abs(v[nz].astype(np.float64))) and np.all(np.sign(d[nz]) == np.sign(v[nz]))


# ------------------------------------------------------------------ a zero residual
@pytest.mark.parametrize("kind", ["spread", "edge_saturating"])
def test_zero_residual_changes_only_the_sign_of_zero(kind):
    """Except where a sum of finite values overflows: without a residual it is Inf (its code NaN, its block's other
    codes +-0); with one it saturates to +-FLT_MAX and its block quantises finite.  Those blocks (the edge payload's
    "overflow" kind) are exempt, and their records with the residual must decode finite."""
    xs = dict(_payloads())[kind.removesuffix("_saturating")]
    x = xs[0]
    n = x.numel()
    zero = torch.zeros(n)

    def same_up_to_zero_sign(a, b, what, exempt=None):
        ca, sa = _records_np(a, n, CHUNK)
        cb, sb = _records_np(b, n, CHUNK)
        keep = np.ones(len(sa), bool) if exempt is None else ~exempt
        assert np.array_equal(sa[keep], sb[keep]), f"{what}: scale bytes differ"
        diff = (ca != cb) & keep[:, None]
        assert np.all((ca[diff] & 0x7F) == 0) and np.all((cb[diff] & 0x7F) == 0), f"{what}: a nonzero code differs"

    recs, _ = ops.ref_pack_fp8(x, CHUNK, residual=zero)
    same_up_to_zero_sign(recs, ops.ref_pack_fp8(x, CHUNK), "pack")
    src = ops.ref_pack_fp8(xs[1], CHUNK)
    y0, rec0 = ops.ref_reduce_fp8(src, 1, n, CHUNK, local=xs[2])
    y1, rec1, _ = ops.ref_reduce_fp8(src, 1, n, CHUNK, local=xs[2], residual=zero)
    loc, dec = xs[2].float().numpy(), decode(*_records_np(src, n, CHUNK)).reshape(-1)
    with np.errstate(over="ignore", invalid="ignore"):
        over = np.isinf(loc + dec) & np.isfinite(loc) & np.isfinite(dec)
    exempt = over.reshape(-1, 32).any(axis=1)
    assert exempt.any() == (kind != "spread"), "the edge payload's overflow kind must be exercised, spread must not"
    same_up_to_zero_sign(rec1, rec0, "reduce", exempt)
    d1 = decode(*_records_np(rec1, n, CHUNK))
    assert np.isfinite(d1[exempt]).all(), "a saturated block decoded non-finite"
    assert torch.equal(y0.float(), y1.float()) or torch.equal(torch.isnan(y0), torch.isnan(y1))


# ------------------------------------------------------------------ the ring with a residual per (rank, shard)
def ring_blocks_ef(xs, rs, trace=None):
    """The model's ring of one shard with error feedback.  ``xs[h]`` / ``rs[h]``: [B, 32] fp32, the input and the
    residual of the rank that quantises at hop h.  Returns (bf16 bits of the output, the new residuals per hop).
    ``trace`` receives per hop (the rounded addend sum or None, the quantised value v).  Both adds saturate
    (``ef_add``)."""
    xs, rs = np.asarray(xs, np.float32), np.asarray(rs, np.float32)
    new = np.empty_like(rs)
    codes = sc = None
    for h in range(len(xs)):
        with np.errstate(over="ignore", invalid="ignore"):
            a = xs[h] if h == 0 else ef_add(xs[h], decode(codes, sc))
            v = ef_add(a, rs[h])
            codes, sc = encode(v)
            r = v - decode(codes, sc)
        new[h] = np.where(np.isfinite(r), r, np.float32(0))
        if trace is not None:
            trace.append((None if h == 0 else a, v))
    return bf16_rne_bits(decode(codes, sc)), new


def ring_model_ef(xs, residuals, traces=None):
    """(bf16 bits [n], new residuals [N][n]) of one error-feedback run; rank (s + h) mod N quantises shard s at hop h."""
    N = len(xs)
    x = np.stack([t.float().numpy() for t in xs])
    r = np.stack([t.float().numpy() for t in residuals])
    m = x.shape[1] // N
    out = np.empty(x.shape[1], dtype=np.uint16)
    new = r.copy()
    for s in range(N):
        ranks = [(s + h) % N for h in range(N)]
        part = slice(s * m, (s + 1) * m)
        tr = [] if traces is not None else None
        bits, nr = ring_blocks_ef(x[ranks, part].reshape(N, -1, 32), r[ranks, part].reshape(N, -1, 32), tr)
        out[part] = bits.reshape(-1)
        for h, q in enumerate(ranks):
            new[q, part] = nr[h].reshape(-1)
        if traces is not None:
            traces.append((s, tr))
    return out, new


@pytest.mark.parametrize("N", range(2, 9))
def test_ring_model_with_residuals_equals_the_reference_over_three_runs(N):
    chunk = 8192
    n = N * 2 * chunk
    res_ref = [torch.zeros(n) for _ in range(N)]
    res_model = [torch.zeros(n) for _ in range(N)]
    for run in range(3):
        xs = spread(N, n, seed=300 + 10 * N + run)
        got, res_ref = ops.ref_allreduce_fp8(xs, chunk, residuals=res_ref)
        want, new = ring_model_ef(xs, res_model)
        res_model = [torch.from_numpy(r) for r in new]
        assert_bits_equal(got, want, f"N={N} run {run}")
        for q in range(N):
            assert np.array_equal(_f32_bits(res_ref[q].numpy()), _f32_bits(new[q])), f"N={N} run {run}: residual of rank {q}"
        assert any(bool((r != 0).any()) for r in res_ref), "the residuals stayed zero: the check is vacuous"


def test_ring_reference_without_residuals_is_unchanged():
    xs = spread(3, 3 * 8192, seed=9)
    plain = ops.ref_allreduce_fp8(xs, 8192)
    assert isinstance(plain, torch.Tensor)
    out, res = ops.ref_allreduce_fp8(xs, 8192, residuals=[torch.zeros(3 * 8192)] * 3)
    assert len(res) == 3 and all(r.dtype == torch.float32 for r in res)
    assert torch.equal(out.float().abs(), plain.float().abs())        # at most the sign of a zero differs


# ------------------------------------------------------------------ the bias goes away
@pytest.mark.parametrize("N", [2, 4, 8])
def test_error_feedback_removes_the_bias_of_a_fixed_input(N):
    """Each rank's input is the same for T = 64 runs.  Without feedback every run makes the same error; with it the
    error of the mean output is at most 1/8 of that, and at most the telescoping bound: the change of the summed
    residuals over T runs, divided by T, plus the rounding of the fp32 adds of every hop."""
    chunk, T = 8192, 64
    n = N * 2 * chunk
    xs = spread(N, n, seed=500 + N)
    exact = np.sum([x.double().numpy() for x in xs], axis=0)
    plain = ops.ref_allreduce_fp8(xs, chunk).double().numpy()
    err_plain = np.linalg.norm(plain - exact)
    assert err_plain > 0
    res = [torch.zeros(n) for _ in range(N)]
    r0 = np.sum([r.double().numpy() for r in res], axis=0)
    total = np.zeros(n)
    rounding = np.zeros(n)
    for t in range(T):
        out, res = ops.ref_allreduce_fp8(xs, chunk, residuals=res)
        total += out.double().numpy()
    res_model = [torch.zeros(n) for _ in range(N)]
    for t in range(T):                                       # the fp32-add rounding bound of every hop of every run
        traces = []
        _, new = ring_model_ef(xs, res_model, traces)
        res_model = [torch.from_numpy(r) for r in new]
        m = n // N
        for s, tr in traces:
            part = slice(s * m, (s + 1) * m)
            for a, v in tr:
                b = np.abs(v.astype(np.float64)).reshape(-1)
                if a is not None:
                    b = b + np.abs(a.astype(np.float64)).reshape(-1)
                rounding[part] += 2.0 ** -24 * b
    mean = total / T
    err_ef = np.linalg.norm(mean - exact)
    assert err_ef <= err_plain / 8, (err_ef, err_plain)
    rT = np.sum([r.double().numpy() for r in res], axis=0)
    bound = np.abs(r0 - rT) / T + rounding / T
    slack = 2.0 ** -50 * np.abs(mean)
    assert np.all(np.abs(mean - exact) <= bound + slack), f"max excess {np.max(np.abs(mean - exact) - bound)}"
    assert err_ef <= np.linalg.norm(r0 - rT) / T + np.linalg.norm(rounding) / T + np.linalg.norm(slack)
