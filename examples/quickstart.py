"""The README quick start as a runnable script (one H100)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W

ctx = rn.Context(device=0)
# allocate and register BEFORE the engine starts: cudaMalloc waits for a resident persistent kernel (DESIGN.md 3.2)
src = torch.empty(1 << 28, dtype=torch.uint8, device="cuda"); dst = torch.empty_like(src)
x = torch.randn(1 << 24, device="cuda").bfloat16()
stg_buf = torch.empty(ops.staging_bytes(x.numel(), 1 << 22), dtype=torch.uint8, device="cuda")
a = torch.randn(4096, 4096, device="cuda").bfloat16(); b = torch.randn(4096, 4096, device="cuda").bfloat16()
c = torch.empty(4096, 4096, device="cuda", dtype=torch.bfloat16)
ms, md, stg, cm = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(stg_buf), ctx.reg_mr(c)   # what amdp2p exists to make possible
qp = ctx.loopback_qp()
torch.cuda.synchronize()

ctx.engine_start(ctas=128)
r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, 1 << 28, iters=8, window=4)   # posted by an SM
print(r.gbps, "GB/s device-timed")
r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, 65536, iters=4096, window=128, burst=16, signal_every=16,
                    slot_stride=65536, nslots=1024)                            # perftest's --post_list / --cq-mod
print(r.us_per_msg, "us per message")
ctx.engine_stop(); ctx.engine_start(ctas=64)
ops.pack_fp8_write(ctx, x, stg, qp=qp, dst_mr=md, chunk_elems=1 << 22)         # bf16 -> fp8 pack fused with the post
ctx.engine_stop(); ctx.engine_start(ctas=32)                                   # leave 100 of 132 SMs to the GEMM
g = ops.gemm_send(ctx, a, b, c, c_mr=cm, qp=qp, dst_mr=md, signal_every=4, grid=100)   # wgmma GEMM, one RDMA write per finished 128-row panel
print(g.tflops, "TFLOP/s including delivery")
ctx.engine_stop()
