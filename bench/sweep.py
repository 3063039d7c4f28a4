#!/usr/bin/env python
"""Message-size sweep, 1 KB - 1 GB (BASELINE.json configs 1, 2, 3, 5 on one GPU):

  gpu_posted      P1  sm_90a kernel posts WQEs + polls the CQ on the device (device-timed, %globaltimer)
  gpu_posted_read P1  same, RDMA READ
  host_posted     B2  CPU posts on host-resident rings and polls (the ib_write_bw-on-a-peermem-MR shape; host-timed)
  host_dram       B0  host MR -> host MR write, host-posted (plumbing check, no GPU memory)
  host_staged     B1  cudaMemcpy D2H -> host-MR write -> cudaMemcpy H2D per message (host-timed)

Every path goes through the same software HCA engine (DESIGN.md section 2: no ConnectX is exposed to the
container), so the comparison isolates WHO posts and WHERE the bytes travel, not the wire."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import _native as N, ops, wire as W  # noqa: E402
from rocnrdma_b200.config import parse_sweep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1k:1g:x4")
    ap.add_argument("--engine-ctas", type=int, default=96)
    ap.add_argument("--out", default="gpurun_out/sweep.json")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    sizes = parse_sweep(a.sizes)
    dev = torch.device("cuda", a.device)
    torch.cuda.set_device(dev)
    from rocnrdma_b200.utils.affinity import bind_to_gpu
    bind_to_gpu(a.device)
    ctx = rn.Context(a.device)
    lib = N.load()
    big = max(sizes)
    pool = max(big, 1 << 30)
    src = torch.empty(pool, dtype=torch.uint8, device=dev); dst = torch.empty(pool, dtype=torch.uint8, device=dev)
    ops.fill_random(src, 11)
    hbytes = min(big, 1 << 30)
    ha = torch.empty(hbytes, dtype=torch.uint8).pin_memory(); hb = torch.empty(hbytes, dtype=torch.uint8).pin_memory()
    ha.random_(0, 255)
    ms, md, mha, mhb = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(ha), ctx.reg_mr(hb)
    qd = ctx.loopback_qp(depth=256)                                   # device rings: GPU-posted
    qh = ctx.loopback_qp(depth=256, mem=W.MEM_HOST_PINNED)            # host rings: host-posted
    qmulti = [qd] + [ctx.loopback_qp(depth=256) for _ in range(7)]    # 8 QPs, one posting warp each: message-rate scaling
    torch.cuda.synchronize()
    ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=10000)
    rows = []
    try:
        for size in sizes:
            iters = int(max(8, min(4096, (8 << 30) // size)))
            nslots = max(1, min(pool // size, 4096))
            win = 16
            row = {"bytes": size, "iters": iters}
            for name, op, l, r in (("gpu_posted", W.OP_RDMA_WRITE, ms, md), ("gpu_posted_read", W.OP_RDMA_READ, md, ms)):
                ops.rdma_stream(qd, op, l, r, size, iters=min(iters, 32), window=win, slot_stride=size, nslots=nslots)
                res = ops.rdma_stream(qd, op, l, r, size, iters=iters, window=win, slot_stride=size, nslots=nslots, timeout_ms=5000)
                row[name] = {"ok": res.ok, "gbps": round(res.gbps, 3), "us_per_msg": round(res.us_per_msg, 3)}
            # perftest-style posting: --post_list 16 --cq-mod 16, 128 outstanding (ib_write_bw's own default is cq-mod 100)
            for name, op, l, r in (("gpu_posted_burst", W.OP_RDMA_WRITE, ms, md), ("gpu_posted_read_burst", W.OP_RDMA_READ, md, ms)):
                kw = dict(window=128, burst=16, signal_every=16, slot_stride=size, nslots=nslots)
                ops.rdma_stream(qd, op, l, r, size, iters=min(iters, 128), **kw)
                res = ops.rdma_stream(qd, op, l, r, size, iters=iters, timeout_ms=5000, **kw)
                row[name] = {"ok": res.ok, "gbps": round(res.gbps, 3), "us_per_msg": round(res.us_per_msg, 3)}
            if size <= (4 << 20):
                # 8 QPs x (post_list 16, cq-mod 16, 128 outstanding); QP q works on its own 1/8 of the pool
                per = pool // 8
                kw = dict(window=128, burst=16, signal_every=16, slot_stride=size, nslots=max(1, min(per // size, 512)), stride=per)
                ops.rdma_stream(qmulti, W.OP_RDMA_WRITE, ms, md, size, iters=min(iters, 128), **kw)
                res = ops.rdma_stream(qmulti, W.OP_RDMA_WRITE, ms, md, size, iters=iters, timeout_ms=5000, **kw)
                row["gpu_posted_burst_8qp"] = {"ok": res.ok, "gbps": round(res.gbps, 3), "us_per_msg": round(res.device_ns / 1e3 / max(sum(res.done), 1), 4),
                                               "mmsgs_per_s": round(sum(res.done) / max(res.device_ns, 1) * 1e3, 2)}
            lat = ops.rdma_stream(qd, W.OP_RDMA_WRITE, ms, md, size, iters=min(iters, 64), window=1, slot_stride=size, nslots=nslots)
            row["gpu_posted"]["latency_us"] = round(lat.us_per_msg, 2)
            ns, err = C.c_uint64(), C.c_uint32()
            hiters = int(max(8, min(1024, (4 << 30) // size)))
            for name, l, r, cap in (("host_posted", ms, md, pool), ("host_dram", mha, mhb, hbytes)):
                if size > cap:
                    continue
                hs = max(1, min(cap // size, 1024))
                N.check(lib.rn_host_stream(qh._q, W.OP_RDMA_WRITE, l.addr, l.lkey, r.addr, r.rkey, size, min(hiters, 16), win, size, hs, 10000,
                                           C.byref(ns), C.byref(err)), name)
                N.check(lib.rn_host_stream(qh._q, W.OP_RDMA_WRITE, l.addr, l.lkey, r.addr, r.rkey, size, hiters, win, size, hs, 20000,
                                           C.byref(ns), C.byref(err)), name)
                row[name] = {"ok": err.value == 0, "gbps": round(size * hiters / ns.value, 3), "us_per_msg": round(ns.value / 1e3 / hiters, 3)}
            if size <= hbytes:
                siters = int(max(4, min(256, (1 << 30) // size)))
                N.check(lib.rn_host_staged_stream(qh._q, src.data_ptr(), dst.data_ptr(), mha.addr, mha.lkey, mhb.addr, mhb.rkey, size, 2,
                                                  size, nslots, 10000, C.byref(ns)), "host_staged")
                N.check(lib.rn_host_staged_stream(qh._q, src.data_ptr(), dst.data_ptr(), mha.addr, mha.lkey, mhb.addr, mhb.rkey, size, siters,
                                                  size, nslots, 30000, C.byref(ns)), "host_staged")
                row["host_staged"] = {"ok": True, "gbps": round(size * siters / ns.value, 3), "us_per_msg": round(ns.value / 1e3 / siters, 3)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    finally:
        ctx.engine_stop()
    ok = ops.compare(src[:min(pool, 1 << 30)], dst[:min(pool, 1 << 30)]) == 0
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    json.dump({"engine_ctas": a.engine_ctas, "verify": ok, "rows": rows, "counters": {"device_qp": qd.counters(), "host_qp": qh.counters()}},
              open(a.out, "w"), indent=1)
    print("verify", ok)


if __name__ == "__main__":
    main()
