#!/usr/bin/env python
"""NVLink ring: every rank GPU-posts RDMA writes into the next rank's HBM (one process per GPU, QPs connected
through CUDA IPC).  Device-timed, max over ranks.  Launch: torchrun --nproc-per-node N bench/ring.py"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops, parallel, wire as W  # noqa: E402
from rocnrdma_b200.config import parse_sweep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64k:1g:x16")
    ap.add_argument("--engine-ctas", type=int, default=32)
    ap.add_argument("--out", default="gpurun_out/ring.json")
    a = ap.parse_args()
    rank, lr, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    dev = torch.device("cuda", lr)
    sizes = parse_sweep(a.sizes)
    pool = max(max(sizes), 1 << 30)
    ctx = rn.Context(lr)
    src = torch.empty(pool, dtype=torch.uint8, device=dev); dst = torch.zeros(pool, dtype=torch.uint8, device=dev)
    ops.fill_random(src, 100 + rank)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    cq = ctx.create_cq(512)
    qp = ctx.create_qp(cq, cq, 256, 256)
    torch.cuda.synchronize()
    nxt, remote = parallel.connect_ring(ctx, qp, [md])
    rmd = remote[md.key] if md.key in remote else list(remote.values())[0]
    dist.barrier(device_ids=[lr]); torch.cuda.synchronize()
    ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=10000)
    rows = []
    for size in sizes:
        iters = int(max(8, min(1024, (8 << 30) // size)))
        nslots = max(1, min(pool // size, 1024))
        ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, rmd, size, iters=min(iters, 16), window=8, slot_stride=size, nslots=nslots, timeout_ms=5000)
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, rmd, size, iters=iters, window=8, slot_stride=size, nslots=nslots, timeout_ms=5000)
        rows.append(dict(bytes=size, ok=r.ok, ns=r.device_ns, iters=iters))
    ctx.engine_stop()
    torch.cuda.synchronize()
    dist.barrier(device_ids=[lr])
    # the previous rank wrote src(prev) into my dst: verify the first slot region against its generator
    prev = (rank - 1) % world
    expect = torch.empty(min(pool, 64 << 20), dtype=torch.uint8, device=dev)
    ops.fill_random(expect, 100 + prev)
    torch.cuda.synchronize()
    ok = bool(torch.equal(expect, dst[:expect.numel()])) if world > 1 else True
    t = torch.tensor([r["ns"] for r in rows] + [0.0 if ok else 1.0], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        out = []
        for r, ns in zip(rows, t.tolist()):
            out.append(dict(bytes=r["bytes"], per_gpu_gbps=round(r["bytes"] * r["iters"] / ns, 1),
                            aggregate_gbps=round(world * r["bytes"] * r["iters"] / ns, 1)))
            print(json.dumps(out[-1]), flush=True)
        res = dict(world=world, engine_ctas=a.engine_ctas, verified=t.tolist()[-1] == 0.0, rows=out,
                   roofline_per_gpu_gbps=450.0, note="H100 SXM NVLink 4: 450 GB/s per direction per GPU (data sheet, not measured)")
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)
        print("verified", res["verified"])
    dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
