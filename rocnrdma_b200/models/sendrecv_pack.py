"""2xH100: a bf16 tensor on GPU0 leaves as block-scaled fp8 records and is bf16 again on GPU1, with no host step in between.

GPU0 runs ``pack_fp8_write`` (K3); GPU1 runs ``unpack_fp8`` (K5), which waits on its receive CQ from the device and
unpacks every record the moment its RDMA_WRITE_IMM completion shows up.  Two data planes under the same control
plane, as for the GEMM (``models/sendrecv_gemm.py``):

  engine   records are staged in GPU0's registered buffer and moved by the DMA engine (RDMA semantics end to end)
  direct   the pack kernel's own coalesced stores go straight into GPU1's registered buffer over NVLink; the queue pair
           only carries a zero-length RDMA_WRITE_IMM per record, posted after a cumulative system-scope fence

Compared with: pack locally, then one GPU-posted RDMA write of all records, then unpack (three steps, one after the other).
"""
from __future__ import annotations

import time

import torch

from .. import ops, wire as W
from ..api import Context


def run(n_elems: int = 1 << 28, chunk_elems: int = 1 << 22, mode: str = "direct", gpus=(0, 1), reps: int = 3, engine_ctas: int = 0) -> dict:
    g0, g1 = gpus
    d0, d1 = torch.device("cuda", g0), torch.device("cuda", g1)
    tx, rx = Context(g0), Context(g1)
    tx.enable_peer(g1)
    x = torch.randn(n_elems, device=d0).to(torch.bfloat16)
    y = torch.zeros(n_elems, device=d1, dtype=torch.bfloat16)
    nb = ops.staging_bytes(n_elems, chunk_elems)
    stg = torch.zeros(nb, dtype=torch.uint8, device=d0)                  # local staging (engine mode, and the unfused baseline)
    rcv = torch.zeros(nb, dtype=torch.uint8, device=d1)
    n_rec = n_elems // chunk_elems
    smr, rmr = tx.reg_mr(stg), rx.reg_mr(rcv)
    direct = mode == "direct"
    peer_mr = tx.reg_mr(rcv) if direct else None                        # GPU1's buffer, registered with GPU0's HCA: peer mapping over NVLink
    cq_a = tx.create_cq(512)
    cq_b = rx.create_cq(max(512, 2 * n_rec))
    qa = tx.create_qp(cq_a, cq_a, 256, 16)
    qb = rx.create_qp(cq_b, cq_b, 16, max(256, 1 << max(n_rec - 1, 1).bit_length()))
    qa.connect(qb)
    qa.set_flags(sys_scope=True)
    if engine_ctas <= 0:
        engine_ctas = 8 if direct else 32                               # direct: the engine only carries the announcements
    _, s_rx = rx.streams(2)
    torch.cuda.synchronize(d0); torch.cuda.synchronize(d1)
    tx.engine_start(ctas=engine_ctas, idle_timeout_ms=5000)
    best = {"fused": None, "sequential": None}
    pack_ns = None
    status = None
    try:
        for it in range(2 * reps):
            fused = it % 2 == 1
            y.zero_(); torch.cuda.synchronize(d1)
            if fused:
                for _ in range(n_rec):                                   # receive buffers are posted ahead of time, as a receiver does
                    qb.post_recv(rmr, 0)
            t0 = time.perf_counter()
            if fused:
                view, _ = ops.unpack_fp8(rx, rcv, y, chunk_elems=chunk_elems, qp=qb, timeout_ms=5000, sync=False, stream=s_rx)
                pr = ops.pack_fp8_write(tx, x, peer_mr if direct else smr, qp=qa, dst_mr=rmr, chunk_elems=chunk_elems, with_imm=True,
                                        signal_every=4, direct=direct, timeout_ms=5000)
                s_rx.synchronize()
                up = ops.pack.parse_unpack(view)
                ok = pr.ok and up["status"] == "OK" and up["records_seen"] == n_rec
                status = {"pack": pr.status, "unpack": up}
                pack_ns = pr.device_ns
            else:
                ops.pack_fp8_write(tx, x, smr, chunk_elems=chunk_elems)                         # 1. pack into local staging
                r = ops.rdma_stream(qa, W.OP_RDMA_WRITE, smr, rmr, nb, iters=1, timeout_ms=5000)   # 2. one GPU-posted write of all records
                ops.unpack_fp8(rx, rcv, y, chunk_elems=chunk_elems)                             # 3. unpack on the peer
                ok = r.ok
            dt = (time.perf_counter() - t0) * 1e6
            if ok and (best["fused" if fused else "sequential"] is None or dt < best["fused" if fused else "sequential"]):
                best["fused" if fused else "sequential"] = dt
    finally:
        tx.engine_stop()
    ref_rec = ops.ref_pack_fp8(x[: 4 * chunk_elems], chunk_elems).to(d1)
    verified = bool(torch.equal(rcv[: ref_rec.numel()], ref_rec)) and bool(
        torch.equal(y[: 4 * chunk_elems], ops.ref_unpack_fp8(ref_rec, 4 * chunk_elems, chunk_elems)))
    out = {"mode": mode, "n_elems": n_elems, "chunk_elems": chunk_elems, "records": n_rec, "wire_bytes": nb, "engine_ctas": engine_ctas,
           "fused_us": best["fused"], "sequential_us": best["sequential"],
           "speedup": best["sequential"] / best["fused"] if best["fused"] and best["sequential"] else None,
           "pack_kernel_us": pack_ns / 1e3 if pack_ns else None, "source_gbps_fused": 2.0 * n_elems / (best["fused"] * 1e3) if best["fused"] else None,
           "verified": verified, "last_fused_status": status, "timing": "host wall clock, launch to completion on both GPUs, best of %d" % reps}
    tx.close(); rx.close()
    return out


if __name__ == "__main__":
    import json
    import sys
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 28
    for m in (sys.argv[2:] or ["engine", "direct"]):
        print(json.dumps(run(n, mode=m)))
