"""BASELINE configs 2, 3 and 5: one H100 driving its own HCA in loopback.

    wl = Loopback(device=0, pool_bytes=1 << 30)
    wl.start(engine_ctas=128)
    wl.write(256 << 20, iters=8).gbps          # GPU-posted RDMA write (config 5 shape, per GPU)
    wl.read(1 << 20, iters=64)
    wl.fused_pack(1 << 28)                     # bf16 -> fp8 pack fused with the post (config 3)
    wl.stop()
"""
from __future__ import annotations

import torch

from .. import ops, wire as W
from ..api import Context, MemoryRegion


class Loopback:
    def __init__(self, device: int = 0, pool_bytes: int = 1 << 30, qp_depth: int = 256):
        self.ctx = Context(device)
        dev = torch.device("cuda", device)
        self.src = torch.empty(pool_bytes, dtype=torch.uint8, device=dev)
        self.dst = torch.empty(pool_bytes, dtype=torch.uint8, device=dev)
        ops.fill_random(self.src, seed=17 + device)
        self.ms, self.md = self.ctx.reg_mr(self.src), self.ctx.reg_mr(self.dst)
        self.qp = self.ctx.loopback_qp(depth=qp_depth)
        self.pool = pool_bytes
        torch.cuda.synchronize(dev)

    def start(self, engine_ctas: int = 128, idle_timeout_ms: int = 8000):
        self.ctx.engine_start(ctas=engine_ctas, idle_timeout_ms=idle_timeout_ms)

    def stop(self):
        self.ctx.engine_stop()

    def _stream(self, op, nbytes, iters, window):
        nslots = max(1, min(self.pool // nbytes, 4096))
        l, r = (self.ms, self.md) if op != W.OP_RDMA_READ else (self.md, self.ms)
        return ops.rdma_stream(self.qp, op, l, r, nbytes, iters=iters, window=window, slot_stride=nbytes, nslots=nslots)

    def write(self, nbytes: int, iters: int = 8, window: int = 8):
        return self._stream(W.OP_RDMA_WRITE, nbytes, iters, window)

    def read(self, nbytes: int, iters: int = 8, window: int = 8):
        return self._stream(W.OP_RDMA_READ, nbytes, iters, window)

    def fused_pack(self, n_elems: int, chunk_elems: int = 1 << 22, signal_every: int = 8):
        """bf16 view of the source pool -> fp8 records staged in the first half of dst, written to its second half."""
        nb = ops.staging_bytes(n_elems, chunk_elems)
        if 2 * n_elems > self.pool or 2 * nb > self.pool:
            raise ValueError("pool too small")
        x = self.src[:2 * n_elems].view(torch.bfloat16)
        stg = MemoryRegion(self.ctx, self.md.addr, nb, self.md.key, self.md.access)
        rmt = MemoryRegion(self.ctx, self.md.addr + self.pool // 2, nb, self.md.key, self.md.access)
        return ops.pack_fp8_write(self.ctx, x, stg, qp=self.qp, dst_mr=rmt, chunk_elems=chunk_elems, signal_every=signal_every)

    def verify(self, nbytes: int) -> bool:
        return ops.compare(self.src[:nbytes], self.dst[:nbytes]) == 0

    def close(self):
        self.ctx.close()
