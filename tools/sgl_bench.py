"""What a two-entry gather costs on the software HCA, one JSON record on stdout.

    python tools/sgl_bench.py [--ctas 32] [--reps 3] [--out FILE]

On one device-posted QP, engine on --ctas CTAs, at 64 B, 4 KiB and 1 MiB per message, alternated --reps times:
* gather:  one WRITE of n bytes whose scatter-gather list is two entries of n/2 in two buffers (ops.gather_stream);
* single:  one WRITE of n bytes from one buffer (ops.rdma_stream);
* halves:  two WRITEs of n/2, both from the first buffer, into the two halves of the destination slot (ops.rdma_stream,
           bursts of two WQEs).
Window 1 (latency: one message in flight; halves keeps one pair in flight, and there the poster's window rule, a burst at
most half the window, rings one doorbell per WRITE) and window 16 with bursts of 8 (rate: halves keeps 32 WQEs in flight
and rings one doorbell per 16).  Microseconds per message of n bytes from the device timers (first post to last
completion), min-max over the runs.  The card's name and power limit are read in the same run.  Needs a GPU.
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
    return {"min": round(min(xs), 4), "max": round(max(xs), 4), "runs": [round(x, 4) for x in xs]} if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sgl_bench needs a GPU")
    sizes = {64: 4000, 4096: 4000, 1 << 20: 400}           # bytes per message: messages per run
    # (label, window, burst): halves runs twice the WQEs at the same number of messages in flight
    modes = (("latency_w1", 1, 1), ("rate_w16_b8", 16, 8))
    nslots = 64
    rec = {"bench": "sgl", "engine_ctas": a.ctas, **gpu_info()}
    ctx = rn.Context(0)
    try:
        cap = max(sizes) * nslots
        a0 = torch.randint(0, 256, (cap,), dtype=torch.uint8, device="cuda:0")
        a1 = torch.randint(0, 256, (cap,), dtype=torch.uint8, device="cuda:0")
        dst = torch.zeros(cap, dtype=torch.uint8, device="cuda:0")
        m0, m1, md = ctx.reg_mr(a0), ctx.reg_mr(a1), ctx.reg_mr(dst)
        qp = ctx.loopback_qp(depth=256)
        torch.cuda.synchronize()
        ok = True
        res = {f"{n}B_{label}": {"gather": [], "single": [], "halves": []} for n in sizes for label, _, _ in modes}

        def run(kind, n, iters, window, burst):
            h = n // 2
            if kind == "gather":
                return ops.gather_stream(qp, W.OP_RDMA_WRITE, m0, m1, md, n, h, iters=iters, window=window, burst=burst,
                                         slot_stride=n, nslots=nslots, timeout_ms=20000)
            if kind == "single":
                return ops.rdma_stream(qp, W.OP_RDMA_WRITE, m0, md, n, iters=iters, window=window, burst=burst, slot_stride=n,
                                       nslots=nslots, timeout_ms=20000)
            # two WRITEs of n/2 per message: 2 * iters WQEs of h bytes into consecutive halves of the same slots
            return ops.rdma_stream(qp, W.OP_RDMA_WRITE, m0, md, h, iters=2 * iters, window=2 * window, burst=2 * burst,
                                   signal_every=2, slot_stride=h, nslots=2 * nslots, timeout_ms=20000)

        ctx.engine_start(ctas=a.ctas, idle_timeout_ms=10000)
        try:
            for rep in range(a.reps + 1):                     # rep 0 warms up every shape
                for n, iters in sizes.items():
                    for label, window, burst in modes:
                        for kind in ("gather", "single", "halves"):
                            r = run(kind, n, iters, window, burst)
                            ok = ok and r.ok
                            if rep:
                                per_msg = r.device_ns / 1e3 / iters
                                res[f"{n}B_{label}"][kind].append(per_msg)
        finally:
            ctx.engine_stop()
        st = ctx.engine_stats()
        rec["ok"] = ok and st["fatal"] == 0
        rec["us_per_msg"] = {k: {kind: _spread(v) for kind, v in d.items()} for k, d in res.items()}
    finally:
        ctx.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
