"""What the fp8 reduce costs alone and what it buys in a ring hop, one JSON record on stdout.

    python tools/reduce_bench.py [--ctas 32] [--reps 3] [--out FILE]

* alone: ops.reduce_fp8 at 2^26 elements in 64 K3 records of 2^20 per source, for P in {1, 2, 4, 8}, with and without a
  bf16 addend, into bf16 or into K3 records; HBM bytes read and written over kernel time (CUDA events), as a share of
  cudaMemcpyAsync D2D (bytes read and written) measured in the same run.  P = 1 without an addend into bf16 moves the
  bytes K5 moves, so it is timed against unpack_fp8 on the same records, alternated.
* ring hop: K3 packs x0 and WRITE_IMMs each record over a loopback QP, recv_consume stamps the arrival words, and
  reduce_fp8(ready=, local=x1) re-packs each sum and WRITEs it over a second loopback QP as it completes, against the same
  steps one after the other on one stream (K3 and its drain, then the reduce, then rdma_stream of its records).  The time
  runs from K3's first post to the last forwarded completion (device timers).
  SMs: engine --ctas + consumer 1 + reduce 48 + K3 48 (129 at the default).
Every run is alternated --reps times after one warm-up round, min-max over the runs, and every result is checked
against ref_reduce_fp8 or the sequential run.  The card's name and power limit are read in the same run.  Needs a GPU.
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops, wire as W  # noqa: E402
from tools.pull_bench import _spread, gpu_info  # noqa: E402


def _timed(fn, stream):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        e0.record(stream)
        out = fn()
        e1.record(stream)
    e1.synchronize()
    return out, e0.elapsed_time(e1) * 1e6      # ns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("reduce_bench needs a GPU")
    TMO = 20000
    chunk, n = 1 << 20, 1 << 26
    n_rec, rec = n // chunk, ops.record_bytes(chunk)
    nb = n_rec * rec
    P_MAX = 8
    if a.ctas + 1 + 48 + 48 > 132:
        sys.exit(f"--ctas {a.ctas}: the engine, the consumer, the reduce and K3 must all be resident on the 132 SMs")
    out = {"bench": "reduce", "n_elems": n, "chunk_elems": chunk, "engine_ctas": a.ctas,
           "sm_sum": {"ring_hop": a.ctas + 1 + 48 + 48}, **gpu_info()}
    ctx = rn.Context(0)
    try:
        g = torch.Generator(device="cuda").manual_seed(7)
        xs = [torch.randn(n, device="cuda", generator=g).to(torch.bfloat16) for _ in range(P_MAX)]
        recs = torch.cat([ops.ref_pack_fp8(x, chunk) for x in xs])
        local = torch.randn(n, device="cuda", generator=g).to(torch.bfloat16)
        y = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        stg = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        smr = ctx.reg_mr(stg)
        cp_src, cp_dst = torch.empty(nb * 4, dtype=torch.uint8, device="cuda"), torch.empty(nb * 4, dtype=torch.uint8, device="cuda")
        s = ctx.stream
        torch.cuda.synchronize()
        checks = {}
        alone = {}
        configs = [(p, loc, o) for p in (1, 2, 4, 8) for loc in (False, True) for o in ("bf16", "fp8")]
        memcpy, k5, k5_ref = [], [], []
        for rep in range(a.reps + 1):
            keep = rep > 0
            _, ns = _timed(lambda: cp_dst.copy_(cp_src), s)
            if keep:
                memcpy.append(2 * cp_src.numel() / ns)
            for p, loc, o in configs:
                key = f"P{p}_{'local' if loc else 'nolocal'}_{o}"
                r, ns = _timed(lambda: ops.reduce_fp8(ctx, recs, p, n, chunk, local=local if loc else None,
                                                      out=y if o == "bf16" else None, out_mr=smr if o == "fp8" else None,
                                                      stream=s, sync=False), s)
                if keep:      # HBM bytes read and written: the sources, the addend, the output
                    alone.setdefault(key, []).append((p * nb + (2 * n if loc else 0) + (2 * n if o == "bf16" else nb)) / ns)
                if rep == a.reps:       # check the last run of each configuration
                    want_y, want_r = ops.ref_reduce_fp8(recs, p, n, chunk, local=local if loc else None)
                    good = ops.parse_reduce(r[0]).ok
                    good &= bool(torch.equal(y.view(torch.int16), want_y.view(torch.int16))) if o == "bf16" else bool(torch.equal(stg, want_r))
                    checks[key] = good
                if p == 1 and not loc and o == "bf16":
                    _, ns5 = _timed(lambda: ops.unpack_fp8(ctx, recs[:nb], y, chunk, stream=s, sync=False), s)
                    if keep:
                        k5.append(ns5 / 1e3)
                        k5_ref.append(ns / 1e3)
                    if rep == a.reps:
                        checks["k5_same_bits"] = bool(torch.equal(y.view(torch.int16), ops.ref_unpack_fp8(recs[:nb], n, chunk).view(torch.int16)))
        mc = min(memcpy)
        out["memcpy_d2d_GBps"] = _spread(memcpy)
        out["alone_GBps"] = {k: {**_spread(v), "share_of_memcpy": [round(min(v) / max(memcpy), 3), round(max(v) / mc, 3)]}
                             for k, v in alone.items()}
        out["P1_bf16_vs_unpack_us"] = {"reduce_fp8": _spread(k5_ref), "unpack_fp8": _spread(k5)}

        # ---- ring hop
        x0, x1 = xs[0], xs[1]
        want_fwd = ops.ref_reduce_fp8(ops.ref_pack_fp8(x0, chunk), 1, n, chunk, local=x1)[1]
        stg0 = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        land1 = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        land2 = {k: torch.zeros(nb, dtype=torch.uint8, device="cuda") for k in ("fused", "sequential")}
        m0, l1 = ctx.reg_mr(stg0), ctx.reg_mr(land1)
        l2 = {k: ctx.reg_mr(v) for k, v in land2.items()}
        words = torch.zeros(n_rec, dtype=torch.int64, device="cuda")
        qp1, qp2 = ctx.loopback_qp(depth=256), ctx.loopback_qp(depth=256)
        _, s_recv, s_red = ctx.streams(3)
        with torch.cuda.stream(s_recv):
            words.zero_()
        torch.cuda.synchronize()
        hop = {"fused": [], "sequential": []}
        for rep in range(a.reps + 1):
            keep = rep > 0
            for kind in ("fused", "sequential"):
                for _ in range(n_rec):
                    qp1.post_recv(l1, 0)
                with torch.cuda.stream(s_recv):
                    words.zero_()
                s_recv.synchronize()
                ctx.engine_start(ctas=a.ctas, idle_timeout_ms=TMO)
                try:
                    if kind == "fused":
                        cv, _ = ops.recv_consume(qp1, n_rec, n_rec, words, timeout_ms=TMO, sync=False, stream=s_recv)
                        rv, _ = ops.reduce_fp8(ctx, land1, 1, n, chunk, local=x1, out_mr=smr, qp=qp2, dst_mr=l2[kind], ready=words,
                                               grid=48, timeout_ms=TMO, sync=False, stream=s_red)
                        pr = ops.pack_fp8_write(ctx, x0, m0, qp=qp1, dst_mr=l1, chunk_elems=chunk, with_imm=True, grid=48,
                                                timeout_ms=TMO, stream=s)
                        s_recv.synchronize(); s_red.synchronize()
                        rr = ops.parse_reduce(rv)
                        good = pr.ok and rr.ok and rr.records_posted == n_rec and ops.parse_recv(cv)["status"] == "OK"
                        t = rr.t_end_ns - pr.t_first_post_ns
                    else:
                        cv, _ = ops.recv_consume(qp1, n_rec, n_rec, words, timeout_ms=TMO, sync=False, stream=s_recv)
                        pr = ops.pack_fp8_write(ctx, x0, m0, qp=qp1, dst_mr=l1, chunk_elems=chunk, with_imm=True, grid=48,
                                                timeout_ms=TMO, stream=s)
                        s_recv.synchronize()
                        rr = ops.reduce_fp8(ctx, land1, 1, n, chunk, local=x1, out_mr=smr, grid=48, timeout_ms=TMO, stream=s)
                        st = ops.rdma_stream(qp2, W.OP_RDMA_WRITE, smr, l2[kind], rec, iters=n_rec, window=16, slot_stride=rec,
                                             nslots=n_rec, timeout_ms=TMO, stream=s)
                        good = pr.ok and rr.ok and st.ok
                        t = max(st.t_end_ns) - pr.t_first_post_ns
                finally:
                    ctx.engine_stop()
                checks[f"ring_{kind}_status"] = checks.get(f"ring_{kind}_status", True) and bool(good)
                checks[f"ring_{kind}_exact"] = checks.get(f"ring_{kind}_exact", True) and bool(torch.equal(land2[kind], want_fwd))
                land2[kind].zero_()
                if keep:
                    hop[kind].append(t / 1e3)
        out["ring_hop_us"] = {k: _spread(v) for k, v in hop.items()}
        out["checks"] = checks
        out["verified"] = all(checks.values())
    finally:
        ctx.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")
    return 0 if out.get("verified") else 1


if __name__ == "__main__":
    sys.exit(main())
