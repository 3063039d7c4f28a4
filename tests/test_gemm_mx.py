"""K7: the block-scaled fp8 GEMM (e4m3 wgmma, block scales applied in registers) against a PyTorch fp32 reference of the
same op: dequantise both operands (e4m3 * 2^(scale - 127) per 32-element block), multiply in fp32.  The kernel's
only rounding beyond that is fp32 accumulation order and the bf16 store."""
import ctypes as C

import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W
from rocnrdma_b200.ops import gemm_mx as MX

pytestmark = pytest.mark.gpu


def _rand(rows, K, spread=True):
    x = torch.randn(rows, K, device="cuda")
    if spread:   # different magnitudes per block, so that a wrong scale byte (wrong row, wrong k, wrong operand) shows
        x = x * torch.exp2(torch.randint(-6, 7, (rows, K // 32, 1), device="cuda").float()).expand(rows, K // 32, 32).reshape(rows, K)
    return x.to(torch.bfloat16)


def _check(c, aq, as_, bq, bs, K):
    ref = MX.dequantize_mx(aq, as_) @ MX.dequantize_mx(bq, bs).T
    err = (c.float() - ref).abs().max().item()
    tol = 2e-2 * ref.abs().max().item() + 1e-3
    assert err <= tol, (err, tol)


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (128, 128, 512), (256, 384, 256), (1024, 512, 1024), (2048, 2304, 1152)])
def test_mxfp8_gemm_matches_dequantised_fp32_reference(ctx, M, N, K, cta_group):
    a, b = _rand(M, K), _rand(N, K)
    (aq, as_), (bq, bs) = MX.quantize_mx(a), MX.quantize_mx(b)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    r = ops.gemm_mxfp8(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group)
    assert r.ok, r.status
    _check(c, aq, as_, bq, bs, K)


@pytest.mark.parametrize("cta_group,M,N", [(1, 128, 128), (2, 256, 256), (2, 512, 768)])
def test_mxfp8_scale_bytes_are_applied_per_row_and_per_block(ctx, cta_group, M, N):
    """All data = 1.0 (e4m3 0x38); only the scales differ.  C[i][j] = sum_k 2^(sa[i][k] + sb[j][k]): any mix-up of row,
    k-block, operand -- or, in the pair kernel, of CTA and accumulator half -- in the scale-factor path changes the answer
    by powers of two."""
    K = 256
    aq = torch.full((M, K), 0x38, dtype=torch.uint8, device="cuda")
    bq = torch.full((N, K), 0x38, dtype=torch.uint8, device="cuda")
    ea = torch.randint(-3, 4, (M, K // 32), device="cuda")
    eb = torch.randint(-3, 4, (N, K // 32), device="cuda")
    as_, bs = (ea + 127).to(torch.uint8), (eb + 127).to(torch.uint8)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group).ok
    ref = 32.0 * (torch.exp2(ea.float()) @ torch.exp2(eb.float()).T)
    assert torch.allclose(c.float(), ref, rtol=1e-2, atol=0), (c.float() - ref).abs().max()


@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("M,N,K", [(200, 136, 160), (130, 72, 96), (64, 300, 32), (700, 520, 416)])
def test_mxfp8_ragged_shapes(ctx, M, N, K, cta_group):
    """TMA zero-fills the out-of-bounds rows and the K tail; the epilogue bounds-checks its stores."""
    a, b = _rand(M, K), _rand(N, K)
    (aq, as_), (bq, bs) = MX.quantize_mx(a), MX.quantize_mx(b)
    pad = torch.full((M + 1, N), 7.0, device="cuda", dtype=torch.bfloat16)     # a canary row behind C
    c = pad[:M]
    r = ops.gemm_mxfp8(ctx, MX.MxOperand.from_tensors(aq, as_), MX.MxOperand.from_tensors(bq, bs), c, cta_group=cta_group)
    assert r.ok, r.status
    _check(c, aq, as_, bq, bs, K)
    assert torch.all(pad[M] == 7.0), "the epilogue wrote past the last row"


def test_mxfp8_consumes_panel_records_of_the_gemm_epilogue(ctx):
    """K4 -> wire -> K7: GEMM 1 emits block-scaled fp8 panel records and RDMA-writes them; GEMM 2 on the receiving side
    uses the delivered records as its A operand, untouched."""
    M, K1, N1 = 512, 256, 512            # GEMM 1: X[M, N1] = P[M, K1] @ Q[N1, K1]^T, sent as fp8 panels
    N2 = 256                             # GEMM 2: Y[M, N2] = X @ R[N2, N1]^T
    p, q = _rand(M, K1, spread=False), _rand(N1, K1, spread=False)
    nb = (M // 128) * ops.panel_record_bytes(N1)
    rec = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    dst = torch.zeros_like(rec)
    rm, dm = ctx.reg_mr(rec), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    g1 = ops.gemm_send(ctx, p, q, rec, c_mr=rm, qp=qp, dst_mr=dm, out_fp8=True)
    ctx.engine_stop()
    assert g1.ok and torch.equal(rec, dst)
    r_ = _rand(N2, N1)
    rq, rs = MX.quantize_mx(r_)
    y = torch.zeros(M, N2, device="cuda", dtype=torch.bfloat16)
    a_op = MX.MxOperand.from_panel_records(dst, M, N1)
    assert ops.gemm_mxfp8(ctx, a_op, MX.MxOperand.from_tensors(rq, rs), y).ok
    x_deq = ops.dequant_fp8_panels(dst, M, N1)                         # what the records say X is
    ref = x_deq @ MX.dequantize_mx(rq, rs).T
    assert (y.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-3


def test_mxfp8_consumes_chunk_records_of_the_fused_pack(ctx):
    """K3 -> K7: a bf16 matrix packed into chunk records is a GEMM operand as it stands."""
    M, K, N = 512, 256, 128
    a = _rand(M, K)
    chunk = 128 * K * 2                                                 # two 128-row groups per record
    nb = ops.staging_bytes(a.numel(), chunk)
    stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    ops.pack_fp8_write(ctx, a.reshape(-1), ctx.reg_mr(stg), qp=None, chunk_elems=chunk)
    torch.cuda.synchronize()
    assert torch.equal(stg, ops.ref_pack_fp8(a.reshape(-1), chunk))
    b = _rand(N, K)
    bq, bs = MX.quantize_mx(b)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_chunk_records(stg, M, K, chunk), MX.MxOperand.from_tensors(bq, bs), c).ok
    aq, as_ = MX.quantize_mx(a)
    _check(c, aq, as_, bq, bs, K)


def test_mxfp8_starts_tiles_as_their_panels_arrive(ctx):
    """Receive-side fusion on one GPU: GEMM 1's fp8 panels travel through the wire (RDMA_WRITE_IMM per panel), a consumer
    kernel stamps each arrival, and GEMM 2 -- launched BEFORE anything has arrived -- starts each tile when the panel it
    reads is there.  Everything is resident at once (engine 16 SMs, GEMM 1 on 48, consumer 1, GEMM 2 on 64: 129 of 132).
    The receive buffer holds poison until a panel lands (e4m3 448 under scale 2^127), and the result must equal bit for
    bit the same call made after every panel is in place: a tile that read its panel early changes bits.
    tests/test_gpu_receive_fusion.py checks the same chain with exact operands at odd and ragged panel counts."""
    M, K1, N1, N2 = 1024, 512, 1024, 512
    p, q = _rand(M, K1, spread=False), _rand(N1, K1, spread=False)
    w = _rand(N2, N1)
    wq, ws = MX.quantize_mx(w)
    panels = M // 128
    nb = panels * ops.panel_record_bytes(N1)
    snd = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    rcv = torch.full((panels, nb // panels), 0xFE, dtype=torch.uint8, device="cuda")
    rcv[:, :128 * N1] = 0x7E
    rcv = rcv.reshape(-1)
    words = torch.zeros(panels + 8, dtype=torch.int64, device="cuda")     # zero words behind the arrival words
    stamps = words[:panels]
    y = torch.zeros(M, N2, device="cuda", dtype=torch.bfloat16)
    sm, rm = ctx.reg_mr(snd), ctx.reg_mr(rcv)
    qp = ctx.loopback_qp(depth=64)
    for _ in range(panels):
        qp.post_recv(rm, 0)
    _, s_recv, s_mm = ctx.streams(3)          # GEMM 1 itself runs on ctx.stream (streams[0])
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=5000)
    try:
        view, _ = ops.recv_consume(qp, panels, panels, stamps, timeout_ms=5000, sync=False, stream=s_recv)
        out2, _ = ops.gemm_mxfp8(ctx, MX.MxOperand.from_panel_records(rcv, M, N1), MX.MxOperand.from_tensors(wq, ws), y, grid=64,
                                 a_ready=stamps, timeout_ms=5000, sync=False, stream=s_mm)
        r1 = ops.gemm_send(ctx, p, q, snd, c_mr=sm, qp=qp, dst_mr=rm, out_fp8=True, with_imm=True, grid=48, timeout_ms=5000)
        s_recv.synchronize(); s_mm.synchronize()
    finally:
        ctx.engine_stop()
    assert r1.ok and r1.panels_posted == panels
    assert ops.parse_recv(view)["seen"] == panels
    assert torch.all(stamps != 0) and torch.all(words[panels:] == 0)
    assert torch.equal(snd, rcv)
    status = (C.c_int64 * 8).from_buffer(out2)[0]                       # read before the next call reuses the slot
    assert status == 0, f"on-arrival GEMM: {status}"
    y_after = torch.zeros_like(y)
    assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_panel_records(rcv, M, N1), MX.MxOperand.from_tensors(wq, ws), y_after).ok
    diff = (y.view(torch.int16) != y_after.view(torch.int16)).sum().item()
    assert diff == 0, f"{diff} elements differ between the product on arrival and after arrival"
    xq = rcv.reshape(panels, -1)[:, :128 * N1].reshape(M, N1)
    xs = rcv.reshape(panels, -1)[:, 128 * N1:].reshape(M, N1 // 32)
    _check(y, xq, xs, wq, ws, N1)


def test_mxfp8_consumes_ragged_panel_records(ctx):
    """K4 at a ragged M emits ceil(M / 128) whole records; K7 multiplies exactly the M rows that exist."""
    M, K1, N1, N2 = 300, 200, 288, 136
    p, q = _rand(M, K1, spread=False), _rand(N1, K1, spread=False)
    w = _rand(N2, N1)
    wq, ws = MX.quantize_mx(w)
    panels = -(-M // 128)
    rec = torch.zeros(panels * ops.panel_record_bytes(N1), dtype=torch.uint8, device="cuda")
    assert ops.gemm_send(ctx, p, q, rec, out_fp8=True).ok
    y = torch.zeros(M, N2, device="cuda", dtype=torch.bfloat16)
    for cg in (1, 2):
        y.zero_()
        assert ops.gemm_mxfp8(ctx, MX.MxOperand.from_panel_records(rec, M, N1), MX.MxOperand.from_tensors(wq, ws), y, cta_group=cg).ok
        r = rec.reshape(panels, -1)
        xq = r[:, :128 * N1].reshape(panels * 128, N1)[:M].contiguous()
        xs = r[:, 128 * N1:].reshape(panels * 128, N1 // 32)[:M].contiguous()
        _check(y, xq, xs, wq, ws, N1)
