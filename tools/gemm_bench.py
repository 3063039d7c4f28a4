"""K4 bench: wgmma GEMM (compute only) vs cuBLAS, and GEMM+send fused vs GEMM-then-send."""
import json, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W
ctx = rn.Context(0)
rows = []
shapes = [(4096, 4096, 4096), (8192, 8192, 8192), (8192, 8192, 2048), (16384, 4096, 1024)]
bufs = {}
for (M, N, K) in shapes:
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16); b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16); d = torch.zeros_like(c)
    bufs[(M, N, K)] = (a, b, c, d, ctx.reg_mr(c), ctx.reg_mr(d))
qp = ctx.loopback_qp(depth=256, cq_depth=512)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
for (M, N, K) in shapes:
    a, b, c, d, cm, dm = bufs[(M, N, K)]
    flops = 2.0 * M * N * K
    # cuBLAS reference (library GEMM, for the roofline only)
    with torch.cuda.stream(ctx.stream):
        for _ in range(3): torch.matmul(a, b.T, out=c)
        ev[0].record()
        for _ in range(10): torch.matmul(a, b.T, out=c)
        ev[1].record(); ev[1].synchronize()
    cublas_tf = flops * 10 / (ev[0].elapsed_time(ev[1]) * 1e-3) / 1e12
    for _ in range(2): r = ops.gemm_send(ctx, a, b, c, cta_group=1)
    best = max(ops.gemm_send(ctx, a, b, c, cta_group=1).tflops for _ in range(5))
    for _ in range(2): ops.gemm_send(ctx, a, b, c, cta_group=2)
    best2 = max(ops.gemm_send(ctx, a, b, c, cta_group=2).tflops for _ in range(5))
    gm = {g: round(max(ops.gemm_send(ctx, a, b, c, cta_group=2, group_m=g).tflops for _ in range(3)), 1) for g in (1, 2, 4, 8, 16)}
    plain2 = max(ops.gemm_send(ctx, a, b, c, cta_group=2, plain_stores=True).tflops for _ in range(5))
    row = dict(M=M, N=N, K=K, group_m_sweep_2cta=gm, ours_2cta_plain_store_epilogue_tflops=round(plain2, 1), cublas_tflops=round(cublas_tf, 1), ours_1cta_tflops=round(best, 1), frac_1cta=round(best / cublas_tf, 3),
               ours_2cta_tflops=round(best2, 1), frac_2cta=round(best2 / cublas_tf, 3))
    by_ctas = {}
    for ectas in [16, 32]:
        ctx.engine_start(ctas=ectas, idle_timeout_ms=3000)
        grid = torch.cuda.get_device_properties(0).multi_processor_count - ectas
        ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, signal_every=4, grid=grid)
        f = min((ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=dm, signal_every=4, grid=grid) for _ in range(3)), key=lambda r: r.device_ns)
        # unfused: GEMM (compute only, same grid), then one GPU-posted write of C; best of 3
        unf_us = 1e30
        for _ in range(3):
            with torch.cuda.stream(ctx.stream):
                ev[0].record()
                ops.gemm_send(ctx, a, b, c, grid=grid, sync=False)
                ops.rdma_stream(qp, W.OP_RDMA_WRITE, cm, dm, min(2 * M * N, (1 << 31) - 65536), iters=1, sync=False)
                ev[1].record(); ev[1].synchronize()
            unf_us = min(unf_us, ev[0].elapsed_time(ev[1]) * 1e3)
        ctx.engine_stop()
        by_ctas[ectas] = dict(engine_ctas=ectas, fused_ok=f.ok, fused_us=round(f.device_ns / 1e3, 1), fused_tflops=round(f.tflops, 1),
                              compute_phase_us=round((f.t_compute_end_ns - f.t_start_ns) / 1e3, 1), unfused_us=round(unf_us, 1),
                              verify=bool(torch.equal(c, d)))
    best_e = min(by_ctas, key=lambda e: by_ctas[e]["fused_us"])
    row.update(by_ctas[best_e])
    row["fused_by_engine_ctas"] = by_ctas
    rows.append(row); print(row, flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/gemm_bench.json", "w"), indent=1)
