"""What the fence flag costs on the software HCA, one JSON record on stdout.

    python tools/fence_bench.py [--ctas 32] [--reps 3] [--out FILE]

On one device-posted loopback QP, engine on --ctas CTAs, alternated --reps times:
* (a) RDMA WRITE message rate at 4 KiB and 1 MiB, window 16, with fence_every 0 (no fence), 8 and 1 (every WRITE
  fenced): ops.rdma_stream, GB/s and microseconds per message;
* (b) latency of a WRITE followed by a READ of the same bytes (4 KiB and 1 MiB): the READ fenced, both under one
  doorbell (ops.write_read mode "fenced"), against the WRITE signaled, its completion awaited, then the READ (mode
  "wait": what ordering costs without the fence).  Mean and best microseconds per pair.

Times come from the device timers (%globaltimer).  The card's name and power limit are read in the same run and recorded
beside the numbers.  Needs a GPU.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops, wire as W  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clk = ([s.strip() for s in q.stdout.strip().split(",")] + ["?", "?", "?"])[:3] if q.returncode == 0 else ("?", "?", "?")
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit": power, "max_sm_clock": clk}


def _spread(xs):
    return {"min": round(min(xs), 3), "max": round(max(xs), 3), "runs": [round(x, 3) for x in xs]} if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fence_bench needs a GPU")
    sizes = (4 << 10, 1 << 20)
    fences = (0, 8, 1)
    iters = {4 << 10: 20000, 1 << 20: 2000}
    pairs = {4 << 10: 2000, 1 << 20: 500}
    nslots = 64
    rec = {"bench": "fence", "engine_ctas": a.ctas, "window": 16, **gpu_info()}
    ctx = rn.Context(0)
    try:
        big = max(sizes)
        src = torch.empty(nslots * big, dtype=torch.uint8, device="cuda:0")
        dst = torch.zeros(nslots * big, dtype=torch.uint8, device="cuda:0")
        back = torch.zeros(big, dtype=torch.uint8, device="cuda:0")
        ops.fill_random(src, seed=3)
        ms, md, mb = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(back)
        qp = ctx.loopback_qp(depth=256)
        torch.cuda.synchronize()
        rate = {f"{n}B": {f"fence_every_{f}": {"gbps": [], "us_per_msg": []} for f in fences} for n in sizes}
        lat = {f"{n}B": {m: {"mean_us": [], "min_us": []} for m in ("fenced", "wait")} for n in sizes}
        ok = True
        ctx.engine_start(ctas=a.ctas, idle_timeout_ms=5000)
        try:
            for rep in range(a.reps + 1):                 # rep 0 warms up every shape
                for n in sizes:
                    for f in fences:
                        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, n, iters=iters[n] if rep else 256, window=16,
                                            slot_stride=n, nslots=nslots, timeout_ms=20000, fence_every=f)
                        ok = ok and r.ok
                        if rep:
                            d = rate[f"{n}B"][f"fence_every_{f}"]
                            d["gbps"].append(r.gbps); d["us_per_msg"].append(r.us_per_msg)
                    for m in ("fenced", "wait"):
                        w = ops.write_read(qp, ms, md, mb, n, iters=pairs[n] if rep else 32, mode=m, timeout_ms=20000)
                        ok = ok and w["status"] == "OK"
                        if rep:
                            d = lat[f"{n}B"][m]
                            d["mean_us"].append(w["mean_ns"] / 1e3); d["min_us"].append(w["min_ns"] / 1e3)
        finally:
            ctx.engine_stop()
        ok = ok and torch.equal(back[:big], dst[:big])
        st = ctx.engine_stats()
        rec["ok"] = bool(ok and st["fatal"] == 0)
        rec["n_fence_waits"] = qp.counters()["n_fence_waits"]
        rec["write_rate"] = {k: {f: {x: _spread(v) for x, v in d.items()} for f, d in fd.items()} for k, fd in rate.items()}
        rec["write_then_read_latency"] = {k: {m: {x: _spread(v) for x, v in d.items()} for m, d in md_.items()}
                                          for k, md_ in lat.items()}
    finally:
        ctx.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
