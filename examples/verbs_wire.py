"""The ConnectX code path end to end: ``Context(wire="verbs")`` -- HBM registered with the HCA (dma-buf first, peer-memory
client second), the QP's mlx5dv send queue / doorbell / CQ mapped into the GPU, an sm_90a kernel posting RDMA writes into
them, and the two host-side baselines on the same MRs.

On a box with a ConnectX and rdma-core this runs against the NIC (loopback on one port).  Without one it uses the
in-tree mock provider (a host-thread NIC that executes the same mlx5 WQEs): set ROCNRDMA_VERBS_LIBDIR yourself, or let
this script do it when /dev/infiniband is absent.  Bandwidth against the mock is the mock's, not a NIC's.
"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if not os.environ.get("ROCNRDMA_VERBS_LIBDIR") and not os.path.exists("/dev/infiniband"):
    os.environ["ROCNRDMA_VERBS_LIBDIR"] = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rocnrdma_b200", "lib", "mock")
import torch  # noqa: E402
import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import _native as N, ops, wire as W  # noqa: E402

ctx = rn.Context(device=0, wire="verbs", nic=0)
print("NIC:", ctx.nic, "(mock provider)" if ctx.nic_is_mock else "")
n = 64 << 20
src = torch.empty(4 * n, dtype=torch.uint8, device="cuda"); dst = torch.zeros_like(src)
ops.fill_random(src, seed=7)
torch.cuda.synchronize()
ms, md = ctx.reg_mr(src, mode="auto"), ctx.reg_mr(dst, mode="auto")          # ibv_reg_dmabuf_mr, else ibv_reg_mr on the pointer
print("HBM registered through:", ms.mode, " lkey", hex(ms.lkey), " rkey", hex(md.rkey))

gq = ctx.loopback_qp(depth=32)                                                 # queues mapped into the GPU (VerbsQueuePair.to_gpu)
r = ops.rdma_stream(gq, W.OP_RDMA_WRITE, ms, md, n, iters=16, window=4, slot_stride=n, nslots=4, timeout_ms=10000)
assert r.ok and ops.compare(src, dst) == 0
print(f"P1  GPU-posted RDMA write : {r.gbps:8.1f} GB/s   (doorbell via CPU proxy: {gq.db_proxy})")

hq = ctx.loopback_qp(depth=32, mem=W.MEM_HOST_PINNED)                          # the same verbs, posted by the CPU
ns, ne = C.c_uint64(), C.c_uint32()
lib = N.load()
rc = lib.rn_verbs_host_stream(hq._vq, W.OP_RDMA_WRITE, ms.addr, ms.lkey, md.addr, md.rkey, n, 16, 4, n, 4, 10000, C.byref(ns), C.byref(ne))
assert rc == 0 and ne.value == 0
print(f"B2  host-posted on HBM MRs: {16 * n / ns.value:8.1f} GB/s")
print("NIC counters:", {k: v for k, v in gq.counters().items() if k in ("n_wqe", "n_err", "n_db_order_violations", "n_doorbells")})
ctx.close()
