"""Send side: a bf16 activation matrix is packed to block-scaled fp8 (one UE8M0 scale per 32 values) by the kernel that
also posts the RDMA writes (K3).  Receive side: the delivered records are the A operand of a tensor-core GEMM as they
stand (K7, e4m3 wgmma with the block scales applied in registers) -- no unpack pass, half the bytes of bf16 on the wire and in
HBM.  Loopback wire on one H100."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops  # noqa: E402
from rocnrdma_b200.ops import gemm_mx as MX  # noqa: E402

M, K, N = 4096, 4096, 4096
ctx = rn.Context(device=0)
x = torch.randn(M, K, device="cuda").bfloat16()                      # what the sender has
w = torch.randn(N, K, device="cuda").bfloat16()                      # the receiver's weights, quantised once
wq, ws = MX.quantize_mx(w)
chunk = 128 * K * 4                                                  # one record = 512 rows of x
nb = ops.staging_bytes(x.numel(), chunk)
stg = torch.zeros(nb, dtype=torch.uint8, device="cuda"); rcv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
y = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
smr, rmr = ctx.reg_mr(stg), ctx.reg_mr(rcv)
qp = ctx.loopback_qp(depth=64)
torch.cuda.synchronize()

ctx.engine_start(ctas=32)
p = ops.pack_fp8_write(ctx, x.reshape(-1), smr, qp=qp, dst_mr=rmr, chunk_elems=chunk)      # pack + post, one kernel
ctx.engine_stop()
assert p.ok
print(f"packed and delivered {x.numel() * 2 / 2**20:.0f} MiB of bf16 as {nb / 2**20:.0f} MiB of records in {p.device_ns / 1e3:.0f} us")

a = MX.MxOperand.from_chunk_records(rcv, M, K, chunk)                                       # the receive buffer IS the operand
r = ops.gemm_mxfp8(ctx, a, MX.MxOperand.from_tensors(wq, ws), y)
assert r.ok
xq, xs = MX.quantize_mx(x)
ref = MX.dequantize_mx(xq[:256], xs[:256]) @ MX.dequantize_mx(wq, ws).T
err = (y[:256].float() - ref).abs().max().item() / ref.abs().max().item()
print(f"y = dequant(records) @ dequant(w)^T: {r.tflops:.0f} TFLOP/s in the kernel, max rel. error vs the fp32 reference {err:.1e}")
ctx.close()
