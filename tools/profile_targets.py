"""Short, profiler-friendly runs of each hot kernel (used under ncu; one GPU).

  gemm     wgmma GEMM, compute only, 4096^3
  pack     bf16 -> fp8 block-scaled pack, 256 Mi elements (pack only: the post needs a resident engine)
  engine   the DMA engine in one-shot mode: 4 host-posted 256 MiB RDMA writes, then it exits
  poster   K1 posting kernel against a resident engine is NOT profilable under ncu (kernel
           serialisation); its cost is in the WQE lifecycle trace instead (tools/latency_trace.py)
"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W
from rocnrdma_b200.ops import pack as P

what = sys.argv[1]
ctx = rn.Context(0)
if what in ("gemm", "gemm2"):
    M = N = K = 4096
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16); b = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    c = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    torch.cuda.synchronize()
    for _ in range(3):
        r = ops.gemm_send(ctx, a, b, c, cta_group=2 if what == "gemm2" else 1)
    print(what, r.ok, round(r.tflops, 1), "TFLOP/s")
elif what == "pack":
    n = 1 << 28
    x = torch.empty(n, dtype=torch.bfloat16, device="cuda"); ops.fill_bf16(x, 1, 1.0)
    st = torch.empty(P.staging_bytes(n, 1 << 22), dtype=torch.uint8, device="cuda")
    smr = ctx.reg_mr(st)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for i in range(3):
        with torch.cuda.stream(ctx.stream):
            ev[0].record(); P.pack_fp8_write(ctx, x, smr, qp=None, chunk_elems=1 << 22, sync=False); ev[1].record()
        ev[1].synchronize()
    us = ev[0].elapsed_time(ev[1]) * 1e3
    print("pack", round(us, 1), "us", round((2 * n + n + n / 32) / us / 1e3, 1), "GB/s HBM traffic")
elif what == "engine":
    msg = 256 << 20
    src = torch.empty(4 * msg, dtype=torch.uint8, device="cuda"); dst = torch.empty(4 * msg, dtype=torch.uint8, device="cuda")
    ops.fill_random(src, 5)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=16, mem=W.MEM_HOST_PINNED if len(sys.argv) > 2 and sys.argv[2] == 'host' else W.MEM_DEVICE)
    if os.environ.get("RN_TRACE"):
        qp.set_flags(trace=True)
    torch.cuda.synchronize()
    for rep in range(2):
        for i in range(4):
            qp.post_write(ms, md, msg, src_off=i * msg, dst_off=i * msg)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ctx.engine_run_oneshot(ctas=128)
        wcs = qp.scq.wait(4)
        assert not any(w.is_error for w in wcs)
        st = ctx.engine_stats()
        if os.environ.get("RN_TRACE"):
            for t in qp.read_trace(8):
                if t["claim"]:
                    print({k: round((v - st["t_start"]) / 1e3, 1) for k, v in t.items() if k in ("claim", "parsed", "copied", "cqe") and v})
        print("oneshot device time", (st["t_exit"] - st["t_start"]) / 1e3, "us", round(4 * msg / max(st["t_exit"] - st["t_start"], 1), 1), "GB/s")
    print("engine oneshot ok", ops.compare(src, dst) == 0)
