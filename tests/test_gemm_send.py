"""K4: wgmma GEMM + fused RDMA write of finished panels, vs a plain fp32 PyTorch reference."""
import pytest
import torch

from rocnrdma_b200 import ops

pytestmark = pytest.mark.gpu


def _ref(a, b):
    return a.float() @ b.float().T


def _check(c, ref, K):
    # bf16 output: half an ulp of relative error, plus fp32 accumulation noise ~ sqrt(K) * eps
    err = (c.float() - ref).abs()
    tol = ref.abs() * 2.0 ** -8 + 1e-3 * (K ** 0.5)
    assert torch.all(err <= tol), f"max err {err.max().item()} (tol at that point {tol.flatten()[err.argmax()].item()})"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 256, 256), (256, 512, 512), (1024, 1024, 2048), (384, 768, 192)])
def test_gemm_compute_only_matches_fp32_reference(ctx, M, N, K):
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c)
    assert r.ok, r.status
    _check(c, _ref(a, b), K)


def test_gemm_identity_exposes_layout_bugs(ctx):
    # A = I (first 256 of K) so C must reproduce B^T's leading block exactly: catches swizzle/descriptor mistakes
    M, N, K = 256, 256, 256
    a = torch.eye(M, K, device="cuda:0").to(torch.bfloat16)
    b = (torch.arange(N * K, device="cuda:0").reshape(N, K) % 251).to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c)
    assert r.ok
    assert torch.equal(c, b.T[:M].contiguous())


def test_gemm_send_panels_arrive_and_match(ctx):
    M, N, K = 1024, 1024, 1024
    torch.manual_seed(7)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    d = torch.zeros_like(c)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, signal_every=4, grid=64)
    finally:
        ctx.engine_stop()
    assert r.ok and r.panels_posted == M // 128, r
    _check(c, _ref(a, b), K)
    assert torch.equal(c, d), "what arrived is not what the GEMM produced"
    cnt = qp.counters()
    assert cnt["n_wqe"] == M // 128 + 1 and cnt["n_err"] == 0 and cnt["n_db_order_violations"] == 0


def test_gemm_rejects_bad_shapes(ctx):
    # rows must be 16-byte multiples for TMA: N % 8, K % 8 (N % 32 for fp8 records); the measurement switches keep the tile rule
    a = torch.zeros(100, 68, device="cuda:0", dtype=torch.bfloat16)
    b = torch.zeros(256, 68, device="cuda:0", dtype=torch.bfloat16)
    c = torch.zeros(100, 256, device="cuda:0", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.gemm_send(ctx, a, b, c)
    a = torch.zeros(100, 64, device="cuda:0", dtype=torch.bfloat16)
    b = torch.zeros(260, 64, device="cuda:0", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.gemm_send(ctx, a, b, torch.zeros(100, 260, device="cuda:0", dtype=torch.bfloat16))
    b = torch.zeros(256, 64, device="cuda:0", dtype=torch.bfloat16)
    with pytest.raises(ValueError):
        ops.gemm_send(ctx, a, b, c, plain_stores=True)


RAGGED = [(100, 256, 64), (1000, 520, 328), (130, 8, 8), (384, 264, 72), (515, 1000, 4104), (257, 1032, 200)]


@pytest.mark.parametrize("cta_group", [1, 2, 3])
@pytest.mark.parametrize("M,N,K", RAGGED)
def test_gemm_ragged_shapes_match_fp32_reference(ctx, M, N, K, cta_group):
    """No tile multiples anywhere: TMA zero-fills the loads that hang over an edge and clips the stores.  Guard rows /
    columns around C prove nothing is written outside it."""
    torch.manual_seed(M * 7 + N * 3 + K + cta_group)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    buf = torch.full(((M + 2) * N + 64,), 7.0, device="cuda:0", dtype=torch.bfloat16)
    off = N + 8                                     # keeps the 16-byte alignment TMA needs
    c = buf[off:off + M * N].view(M, N)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=cta_group)
    assert r.ok, r.status
    _check(c, _ref(a, b), K)
    assert torch.all(buf[:off] == 7.0) and torch.all(buf[off + M * N:] == 7.0), "stored outside C"


@pytest.mark.parametrize("cta_group", [1, 2, 3])
def test_gemm_ragged_send_short_last_panel(ctx, cta_group):
    """M = 3 panels and 40 rows: four RDMA writes, the last one 40 rows long, nothing beyond it at the destination."""
    M, N, K = 424, 520, 200
    torch.manual_seed(5 + cta_group)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    d = torch.full((M + 16, N), 3.0, device="cuda:0", dtype=torch.bfloat16)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, cta_group=cta_group, grid=16)
    finally:
        ctx.engine_stop()
    assert r.ok and r.panels_posted == 4, r
    _check(c, _ref(a, b), K)
    assert torch.equal(d[:M], c) and torch.all(d[M:] == 3.0)


@pytest.mark.parametrize("cta_group", [1, 2, 3])
@pytest.mark.parametrize("M,N,K", [(300, 288, 200), (128, 32, 64), (700, 1056, 520)])
def test_gemm_ragged_fp8_records(ctx, M, N, K, cta_group):
    """fp8 epilogue through the staged TMA store at shapes that clip: whole records for ceil(M / 128) panels, columns
    beyond N never written (the byte after the last record stays untouched)."""
    torch.manual_seed(M + N + K + cta_group)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    P = -(-M // 128)
    nb = P * ops.panel_record_bytes(N)
    c = torch.full((nb + 256,), 0xAB, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, out_fp8=True, cta_group=cta_group)
    assert r.ok, r.status
    assert torch.all(c[nb:] == 0xAB), "stored beyond the last record"
    ref32 = _ref(a, b)
    ref_rec = ops.ref_fp8_panels(ref32)
    mism = (c[:nb] != ref_rec).float().mean().item()
    assert mism < 0.02, f"{mism:.4f} of the record bytes differ from the reference quantisation"
    got = ops.dequant_fp8_panels(c[:nb], M, N)
    blk = ref32.reshape(M, N // 32, 32).abs().amax(dim=2, keepdim=True).expand(-1, -1, 32).reshape(M, N)
    assert torch.all((got - ref32).abs() <= blk * (2.0 ** -4) * 1.05 + 1e-2)


def test_gemm_fp8_epilogue_records_match_reference_and_arrive(ctx):
    """Block-scaled fp8 send tile: the epilogue's records equal quantising the fp32 product, and they land."""
    M, N, K = 512, 1024, 512
    torch.manual_seed(11)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    nb = (M // 128) * ops.panel_record_bytes(N)
    c = torch.zeros(nb, dtype=torch.uint8, device="cuda:0")
    d = torch.zeros(nb, dtype=torch.uint8, device="cuda:0")
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, out_fp8=True, grid=32)
    finally:
        ctx.engine_stop()
    assert r.ok and r.panels_posted == M // 128
    assert torch.equal(c, d), "records at the destination differ from the send buffer"
    ref32 = _ref(a, b)
    ref_rec = ops.ref_fp8_panels(ref32)
    # the tensor core accumulates in a different order than the fp32 reference GEMM, so a value that
    # sits on a rounding boundary may fall either way: allow a small fraction of 1-ulp differences,
    # and require the dequantised result to be within the format's error bound
    mism = (c != ref_rec).float().mean().item()
    assert mism < 0.02, f"{mism:.4f} of the record bytes differ from the reference quantisation"
    got = ops.dequant_fp8_panels(d, M, N)
    blk = ref32.reshape(M, N // 32, 32).abs().amax(dim=2, keepdim=True).expand(-1, -1, 32).reshape(M, N)
    assert torch.all((got - ref32).abs() <= blk * (2.0 ** -4) * 1.05 + 1e-2)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (256, 512, 512), (1024, 1024, 2048), (512, 768, 192)])
def test_gemm_cta_pair_kernel_matches_fp32_reference(ctx, M, N, K):
    torch.manual_seed(M * 3 + N + K)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=2)
    assert r.ok, r.status
    _check(c, _ref(a, b), K)


def test_gemm_cta_pair_identity_layout(ctx):
    M, N, K = 512, 512, 512
    a = torch.eye(M, K, device="cuda:0").to(torch.bfloat16)
    b = (torch.arange(N * K, device="cuda:0").reshape(N, K) % 251).to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=2)
    assert r.ok
    assert torch.equal(c, b.T[:M].contiguous())


def test_gemm_cta_pair_send_panels(ctx):
    M, N, K = 1024, 1024, 1024
    torch.manual_seed(5)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda:0", dtype=torch.bfloat16)
    d = torch.zeros_like(c)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, signal_every=4, cta_group=2, grid=64)
    finally:
        ctx.engine_stop()
    assert r.ok and r.panels_posted == M // 128, r
    _check(c, _ref(a, b), K)
    assert torch.equal(c, d)


@pytest.mark.parametrize("cta_group,group_m", [(1, 1), (1, 3), (2, 1), (2, 3), (2, 16)])
def test_gemm_tile_rasterisation_orders(ctx, cta_group, group_m):
    """Grouped tile orders (incl. a group size that does not divide the M blocks) cover every tile exactly once."""
    M, N, K = 1280, 768, 128           # 10 M blocks / 5 pairs: ragged last group for group_m = 3
    torch.manual_seed(group_m)
    a = torch.randn(M, K, device="cuda:0").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda:0").to(torch.bfloat16)
    c = torch.full((M, N), float("nan"), device="cuda:0", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    r = ops.gemm_send(ctx, a, b, c, cta_group=cta_group, group_m=group_m, grid=12)
    assert r.ok
    _check(c, _ref(a, b), K)


@pytest.mark.parametrize("cta_group", [1, 2])
def test_gemm_epilogue_variants_agree_bit_for_bit(ctx, cta_group):
    """Staged TMA tensor stores (default) and per-thread row stores are two ways to write the same bf16 tile."""
    torch.manual_seed(11)
    M, N, K = 512, 768, 320
    a = torch.randn(M, K, device="cuda").bfloat16()
    b = torch.randn(N, K, device="cuda").bfloat16()
    c1 = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    c2 = torch.full((M, N), -7.0, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_send(ctx, a, b, c1, cta_group=cta_group).ok
    assert ops.gemm_send(ctx, a, b, c2, cta_group=cta_group, plain_stores=True).ok
    assert torch.equal(c1, c2)
    ref = a.float() @ b.float().t()
    assert (c1.float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item()


@pytest.mark.parametrize("M,N,K", [(512, 256, 64), (512, 512, 256), (1024, 768, 320), (2048, 1024, 1024)])
def test_gemm_wide_pair_kernel_matches_fp32_reference(ctx, M, N, K):
    """cta_group=3: the CTA-pair kernel on the schedule that can split the last wave along K (stream-K)."""
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    r = ops.gemm_send(ctx, a, b, c, cta_group=3)
    assert r.ok, r.status
    ref = a.float() @ b.float().T
    assert torch.allclose(c.float(), ref, rtol=2e-2, atol=0.5 * (K / 256) ** 0.5)


def test_gemm_wide_identity_layout(ctx):
    """B = I: C must equal A exactly -- every row of both CTAs of every cluster lands where it belongs."""
    M = N = K = 1024
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.eye(N, K, device="cuda").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    assert ops.gemm_send(ctx, a, b, c, cta_group=3, grid=6).ok          # 3 clusters over 16 tiles: uneven, several tiles per cluster
    assert torch.equal(c, a)


@pytest.mark.parametrize("out_fp8", [False, True])
def test_gemm_wide_send_panels(ctx, out_fp8):
    M, N, K = 1024, 512, 256
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    if out_fp8:
        nb = (M // 128) * ops.gemm.panel_record_bytes(N)
        c = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    else:
        c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    d = torch.zeros_like(c)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, cta_group=3, out_fp8=out_fp8, signal_every=2)
    ctx.engine_stop()
    assert r.ok and r.panels_posted == M // 128, (r.status, r.panels_posted)
    assert torch.equal(c, d)
    ref = a.float() @ b.float().T
    if out_fp8:
        assert torch.equal(d, ops.gemm.ref_fp8_panels(ref)) or torch.allclose(ops.gemm.dequant_fp8_panels(d, M, N), ref, rtol=0.08, atol=0.5)
    else:
        assert torch.allclose(d.float(), ref, rtol=2e-2, atol=0.5)


@pytest.mark.parametrize("M,N,K,grid", [(1024, 1024, 512, 6), (1536, 768, 1024, 10), (2560, 2048, 2048, 60), (512, 768, 4096, 4),
                                        (512, 768, 4096, 8), (4096, 4096, 1024, 148)])
def test_gemm_wide_stream_k_matches_fp32_reference(ctx, M, N, K, grid):
    """Where the 256x256 cluster tiles do not divide evenly among the clusters, the last wave is split along K between
    neighbouring clusters and folded back together through the fp32 workspace: same answer as the unsplit schedule (bit
    for bit is not required: different summation order), fp32-reference accuracy.  Where they do divide evenly (512 x 768
    over 2 clusters), stream-K must not split anything and the result equals the plain schedule's exactly.  The grid is
    clamped to the SM count, so 148 runs as many clusters as the GPU holds."""
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    c2 = torch.zeros_like(c)
    n_tiles = -(-M // 256) * -(-N // 256)
    clusters = min(grid, torch.cuda.get_device_properties(0).multi_processor_count, 2 * n_tiles) // 2
    partial_wave = n_tiles % clusters != 0
    for _ in range(2):                                               # twice: the epoch-stamped flags need no reset
        r = ops.gemm_send(ctx, a, b, c, cta_group=3, grid=grid, stream_k=True)
        assert r.ok, r.status
        assert r.stream_k == partial_wave, (n_tiles, clusters)
    r2 = ops.gemm_send(ctx, a, b, c2, cta_group=3, grid=grid, stream_k=False)
    assert r2.ok and not r2.stream_k
    ref = a.float() @ b.float().T
    tol = 0.5 * (K / 256) ** 0.5
    assert torch.allclose(c.float(), ref, rtol=2e-2, atol=tol)
    assert torch.allclose(c.float(), c2.float(), rtol=2e-2, atol=tol)
    if not partial_wave:
        assert torch.equal(c, c2)


def test_gemm_wide_stream_k_send_and_fp8(ctx):
    M, N, K = 1024, 768, 1024                                        # 12 tiles over 5 clusters: the last 2 are split along K
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    nb = (M // 128) * ops.gemm.panel_record_bytes(N)
    c = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    d = torch.zeros_like(c)
    cm, dm = ctx.reg_mr(c), ctx.reg_mr(d)
    qp = ctx.loopback_qp(depth=64)
    ctx.engine_start(ctas=8, idle_timeout_ms=3000)
    r = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, cta_group=3, out_fp8=True, grid=10, stream_k=True)
    ctx.engine_stop()
    assert r.ok and r.stream_k and r.panels_posted == M // 128 and torch.equal(c, d)
    ref = a.float() @ b.float().T
    assert torch.allclose(ops.gemm.dequant_fp8_panels(d, M, N), ref, rtol=0.08, atol=1.0)
