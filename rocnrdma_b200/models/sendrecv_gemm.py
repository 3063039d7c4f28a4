"""BASELINE config 4: 2xH100 send/recv, GPU0 -> wire -> GPU1, overlapped with the wgmma GEMM that
produces the send tile.

Two HCA contexts, one per GPU, connected QP to QP exactly as two nodes would be (the responder's MKey
table, receive ring and receive CQ live on GPU1 and are reached by GPU0's engine over NVLink).  GPU0
runs ``gemm_send`` with RDMA_WRITE_IMM: every finished 128-row panel is written into GPU1's registered
buffer and announced by a receive completion carrying the panel index; a consumer kernel on GPU1 polls
that receive CQ on the device.  No host involvement between the first launch and the last completion.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import ops, wire as W
from ..api import Context


@dataclass
class SendRecvResult:
    mode: str
    ok: bool
    fused_us: float
    compute_us: float
    first_post_us: float
    engine_ctas: int
    unfused_us: float
    tflops: float
    wire_gbps: float
    panels: int
    consumer: dict
    verified: bool


def run(M: int = 8192, N: int = 8192, K: int = 2048, engine_ctas: int = 0, gpus=(0, 1), reps: int = 3,
        mode: str = "engine") -> SendRecvResult:
    """mode="engine": panels are staged in GPU0's send buffer and moved by the DMA engine (RDMA semantics).
    mode="direct": the GEMM epilogue stores straight into GPU1's registered buffer over NVLink and only the
    per-panel completion signal (zero-length RDMA_WRITE_IMM) goes through the queue pair.
    mode="auto": direct for compute-heavy shapes (K >= 4096), engine otherwise."""
    if mode == "auto":
        # direct stores leave the SMs in bursts (all CTAs reach their epilogue together), the engine streams at NVLink
        # rate but costs 32 SMs: direct pays off once a tile's compute time covers its 64 KiB of output leaving the SM.
        # K >= 4096 is that point by estimate; the crossover has not been measured on H100 (it needs two GPUs)
        mode = "direct" if K >= 4096 else "engine"
    g0, g1 = gpus
    d0, d1 = torch.device("cuda", g0), torch.device("cuda", g1)
    tx, rx = Context(g0), Context(g1)
    tx.enable_peer(g1)
    a = torch.randn(M, K, device=d0).to(torch.bfloat16)
    b = torch.randn(N, K, device=d0).to(torch.bfloat16)
    c = torch.zeros(M, N, device=d0, dtype=torch.bfloat16)
    d = torch.zeros(M, N, device=d1, dtype=torch.bfloat16)
    panels = M // 128
    stamps = torch.zeros(panels, dtype=torch.int64, device=d1)
    cm, dm = tx.reg_mr(c), rx.reg_mr(d)
    cq_a = tx.create_cq(512)
    cq_b = rx.create_cq(max(512, 2 * panels))
    qa = tx.create_qp(cq_a, cq_a, 256, 16)
    qb = rx.create_qp(cq_b, cq_b, 16, max(256, 1 << (panels - 1).bit_length()))
    qa.connect(qb)
    qa.set_flags(sys_scope=True)                # the responder side of this QP lives on another GPU
    torch.cuda.synchronize(d0); torch.cuda.synchronize(d1)
    direct = mode == "direct"
    if engine_ctas <= 0:
        engine_ctas = 8 if direct else 32          # direct: the engine only carries the signals
    if direct:
        d_local = tx.reg_mr(d)                     # GPU1's buffer, registered with GPU0's HCA: peer mapping over NVLink
    tx.engine_start(ctas=engine_ctas, idle_timeout_ms=5000)
    grid = torch.cuda.get_device_properties(d0).multi_processor_count - engine_ctas
    best = None
    try:
        for rep in range(reps):
            for _ in range(panels):
                qb.post_recv(dm, 0)
            view, rstream = ops.recv_consume(qb, panels, panels, stamps, timeout_ms=5000, sync=False)
            if direct:
                r = ops.gemm_send(tx, a, b, d, c_mr=d_local, qp=qa, dst_mr=dm, signal_every=4, with_imm=True, direct=True,
                                  grid=grid, timeout_ms=5000)
            else:
                r = ops.gemm_send(tx, a, b, c, c_mr=cm, qp=qa, dst_mr=dm, signal_every=4, with_imm=True, grid=grid, timeout_ms=5000)
            rstream.synchronize()
            cons = ops.parse_recv(view)
            if best is None or r.device_ns < best[0].device_ns:
                best = (r, cons)
        # unfused reference on the same wire: GEMM, then one GPU-posted write of C
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        with torch.cuda.stream(tx.stream):
            ev[0].record()
            ops.gemm_send(tx, a, b, c, grid=grid, sync=False)
            ops.rdma_stream(qa, W.OP_RDMA_WRITE, cm, dm, 2 * M * N, iters=1, sync=False, timeout_ms=5000)
            ev[1].record()
        ev[1].synchronize()
        unfused_us = ev[0].elapsed_time(ev[1]) * 1e3
    finally:
        tx.engine_stop()
    r, cons = best
    if direct:
        ops.gemm_send(tx, a, b, c)                 # reference product computed locally for the comparison
    verified = bool(torch.equal(c.cpu(), d.cpu()))
    out = SendRecvResult(mode=mode, ok=r.ok and cons["status"] == "OK" and cons["seen"] == panels, fused_us=r.device_ns / 1e3,
                         compute_us=(r.t_compute_end_ns - r.t_start_ns) / 1e3,
                         first_post_us=(r.t_first_post_ns - r.t_start_ns) / 1e3, engine_ctas=engine_ctas, unfused_us=unfused_us, tflops=r.tflops,
                         wire_gbps=r.wire_gbps, panels=panels, consumer=cons, verified=verified)
    tx.close(); rx.close()
    return out


def run_chain(M: int = 8192, N1: int = 8192, K1: int = 2048, N2: int = 8192, gpus=(0, 1), reps: int = 3, engine_ctas: int = 32) -> dict:
    """Two GEMMs chained across two GPUs with the wire between them fused into both.

    GPU0: ``X[M, N1] = P @ Q^T`` (K4): the epilogue emits block-scaled fp8 panel records and RDMA-writes each finished
    128-row panel (RDMA_WRITE_IMM) into GPU1's registered buffer.  GPU1: ``Y[M, N2] = X @ W^T`` (K7) multiplies the records
    where they landed; given the arrival words that a receive-CQ consumer kernel stamps, it starts every tile as soon
    as the panel it reads is there -- so GEMM 2 runs while GEMM 1 is still producing and the wire is still moving.
    Compared with the same three steps run one after the other.  Host wall clock around launch .. completion (two
    devices, no common device clock), best of ``reps``."""
    import time
    from ..ops import gemm_mx as MX
    g0, g1 = gpus
    d0, d1 = torch.device("cuda", g0), torch.device("cuda", g1)
    tx, rx = Context(g0), Context(g1)
    tx.enable_peer(g1)
    p = torch.randn(M, K1, device=d0).to(torch.bfloat16)
    q = torch.randn(N1, K1, device=d0).to(torch.bfloat16)
    w = torch.randn(N2, N1, device=d1).to(torch.bfloat16)
    wq, ws = MX.quantize_mx(w)
    panels = M // 128
    nb = panels * ops.panel_record_bytes(N1)
    snd = torch.zeros(nb, dtype=torch.uint8, device=d0)
    rcv = torch.zeros(nb, dtype=torch.uint8, device=d1)
    stamps = torch.zeros(panels, dtype=torch.int64, device=d1)
    y = torch.zeros(M, N2, device=d1, dtype=torch.bfloat16)
    sm, rm = tx.reg_mr(snd), rx.reg_mr(rcv)
    cq_a = tx.create_cq(512)
    cq_b = rx.create_cq(max(512, 2 * panels))
    qa = tx.create_qp(cq_a, cq_a, 256, 16)
    qb = rx.create_qp(cq_b, cq_b, 16, max(256, 1 << (panels - 1).bit_length()))
    qa.connect(qb)
    qa.set_flags(sys_scope=True)
    _, s_recv, s_mm = rx.streams(3)
    a_op, b_op = MX.MxOperand.from_panel_records(rcv, M, N1), MX.MxOperand.from_tensors(wq, ws)
    torch.cuda.synchronize(d0); torch.cuda.synchronize(d1)
    tx.engine_start(ctas=engine_ctas, idle_timeout_ms=5000)
    grid1 = torch.cuda.get_device_properties(d0).multi_processor_count - engine_ctas
    best = {"fused": None, "sequential": None}
    try:
        for mode in ("sequential", "fused", "sequential", "fused") * max(1, (reps + 1) // 2):
            stamps.zero_()
            torch.cuda.synchronize(d1)
            for _ in range(panels):
                qb.post_recv(rm, 0)
            t0 = time.perf_counter()
            view, _ = ops.recv_consume(qb, panels, panels, stamps, timeout_ms=5000, sync=False, stream=s_recv)
            if mode == "fused":
                # 146 CTAs: the consumer kernel keeps its SM; every tile waits for its own panel
                ops.gemm_mxfp8(rx, a_op, b_op, y, grid=146, a_ready=stamps, timeout_ms=5000, sync=False, stream=s_mm)
                r1 = ops.gemm_send(tx, p, q, snd, c_mr=sm, qp=qa, dst_mr=rm, out_fp8=True, with_imm=True, signal_every=4, grid=grid1, timeout_ms=5000)
            else:
                r1 = ops.gemm_send(tx, p, q, snd, c_mr=sm, qp=qa, dst_mr=rm, out_fp8=True, with_imm=True, signal_every=4, grid=grid1, timeout_ms=5000)
                s_recv.synchronize()
                ops.gemm_mxfp8(rx, a_op, b_op, y, sync=False, stream=s_mm)
            s_recv.synchronize(); s_mm.synchronize()
            dt = (time.perf_counter() - t0) * 1e6
            ok = r1.ok and ops.parse_recv(view)["seen"] == panels
            if ok and (best[mode] is None or dt < best[mode]):
                best[mode] = dt
    finally:
        tx.engine_stop()
    xq = rcv.reshape(panels, -1)[:256 // 128, :128 * N1].reshape(256, N1)
    xs = rcv.reshape(panels, -1)[:256 // 128, 128 * N1:].reshape(256, N1 // 32)
    ref = MX.dequantize_mx(xq, xs) @ MX.dequantize_mx(wq, ws).T
    verified = bool(torch.equal(snd.cpu(), rcv.cpu())) and (y[:256].float() - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-3
    out = {"shape": {"M": M, "N1": N1, "K1": K1, "N2": N2}, "fused_us": best["fused"], "sequential_us": best["sequential"],
           "speedup": (best["sequential"] / best["fused"]) if best["fused"] and best["sequential"] else None, "verified": verified,
           "wire_bytes": nb, "panels": panels, "engine_ctas": engine_ctas,
           "what": "GPU0 GEMM (fp8 panel records, per-panel RDMA_WRITE_IMM over NVLink) -> GPU1 block-scaled GEMM on the records in place; "
                   "fused = GEMM 2 starts tiles on panel arrival; host wall clock"}
    tx.close(); rx.close()
    return out


if __name__ == "__main__":
    import json
    import sys
    shape = tuple(int(x) for x in sys.argv[1:4]) if len(sys.argv) >= 4 else (8192, 8192, 2048)
    if len(sys.argv) > 4 and sys.argv[4] == "chain":
        print(json.dumps(run_chain(shape[0], shape[1], shape[2], int(sys.argv[5]) if len(sys.argv) > 5 else shape[1])))
        sys.exit(0)
    res = run(*shape, mode=sys.argv[4] if len(sys.argv) > 4 else "engine", engine_ctas=int(sys.argv[5]) if len(sys.argv) > 5 else 0)
    print(json.dumps(res.__dict__))
