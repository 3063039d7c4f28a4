"""How close the software HCA's engine gets to its own copy loop, and where the difference goes.

In one process, alternating and repeated (--reps), at each engine CTA count (--ctas):
  (a) ceiling: the engine's TMA copy loop with nothing around it (rn_k_engine_ceiling: each CTA streams one long
      contiguous span, no claims, no chunk boundaries, no completion bookkeeping);
  (b) engine:  the persistent engine on bench.py's shape (256 MiB RDMA WRITEs, window 8, 4 rotating slots);
  (c) memcpy:  cudaMemcpyAsync device-to-device on the same buffers (once per repetition; uses no SMs).
Reports median / min / max GB/s of each, the engine as a fraction of the ceiling, and the per-chunk dead time
derived from (a) and (b): the engine cuts a 256 MiB WQE into granules of max(chunk_bytes, bytes / (8 x CTAs)), so a
CTA moves one granule in granule / (rate / CTAs); the dead time is the engine's time per granule minus the ceiling's.
The card name, power limit and max SM clock are read (nvidia-smi --query-gpu, read-only) in the same run.

--profile adds, once per CTA count after the timed runs, one profiled run of each (the engine under RN_ENGINE_PROFILE=1,
the ceiling kernel with a profile buffer): where the mover's time went, as µs per granule summed over the CTAs' movers
and divided by the granules moved (Context.engine_mover_profile; bucket names in api.MOVER_PROFILE_FIELDS).  "issue" is
what is left of the mover's total after every wait: issuing loads and stores, polling, bookkeeping.

    python tools/engine_pipeline.py [--ctas 8,16,32,64] [--reps 3] [--profile] [--out results.json]

The result is printed as JSON; --out also writes it to a file.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MSG = 256 << 20
NSLOTS = 4
KSUB = 16384


def granule(nbytes: int, ctas: int, chunk_bytes: int = 512 << 10) -> int:
    """The engine's work granule for one WQE (write_resolved in csrc/hca/engine.cuh)."""
    target = 8 * ctas
    want = -(-nbytes // target)
    want = -(-want // KSUB) * KSUB
    return max(chunk_bytes, want)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, sm = [v.strip() for v in out[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": sm}
    except Exception as e:      # the numbers still stand; say why the card is not named
        return {"error": str(e)[:120]}


def summary(xs):
    return {"median": round(statistics.median(xs), 1), "min": round(min(xs), 1), "max": round(max(xs), 1),
            "runs": [round(x, 1) for x in xs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", default="8,16,32,64")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=0.4, help="approximate length of each timed window")
    ap.add_argument("--profile", action="store_true", help="also profile where the mover's time goes (engine and ceiling)")
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    args = ap.parse_args()

    import torch
    import rocnrdma_b200 as rn
    from rocnrdma_b200 import _native as N, ops, wire as W

    ctas_list = [int(x) for x in args.ctas.split(",")]
    lib = N.load()
    ctx = rn.Context(device=0, wire="softhca")
    dev = torch.device("cuda", 0)
    src = torch.empty(MSG * NSLOTS, dtype=torch.uint8, device=dev)
    dst = torch.zeros(MSG * NSLOTS, dtype=torch.uint8, device=dev)
    fatal = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.fill_random(src, seed=7)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64)
    stream = ctx.stream
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = MSG * NSLOTS
    torch.cuda.synchronize()

    nf = len(rn.api.MOVER_PROFILE_FIELDS)
    prof = torch.zeros(max(ctas_list) * nf, dtype=torch.int64, device=dev)

    def ceiling(n: int, profile: bool = False) -> float:
        span = total // n // KSUB * KSUB
        pp = prof.data_ptr() if profile else 0
        launch = lambda: N.check(lib.rn_k_engine_ceiling(stream.cuda_stream, src.data_ptr(), dst.data_ptr(), span, n,
                                                         fatal.data_ptr(), pp), "engine_ceiling")
        launch()
        launch()
        stream.synchronize()
        iters = max(2, int(args.seconds * 40e9 * n / (span * n)))
        ev0.record(stream)
        for _ in range(iters):
            launch()
        ev1.record(stream)
        ev1.synchronize()
        assert int(fatal.item()) == 0, "ceiling kernel: a bulk load never landed"
        return iters * span * n / (ev0.elapsed_time(ev1) * 1e-3) / 1e9

    def engine(n: int, profile: bool = False) -> float:
        os.environ["RN_ENGINE_PROFILE"] = "1" if profile else "0"
        ctx.engine_start(ctas=n, idle_timeout_ms=20000)
        kw = dict(window=8, slot_stride=MSG, nslots=NSLOTS, stream=stream, timeout_ms=20000)
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, MSG, iters=8, **kw)
        assert r.ok, r.status
        iters = max(16, int(args.seconds * 40e9 * n / MSG))
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, MSG, iters=iters, **kw)
        ctx.engine_stop()
        st = ctx.engine_stats()
        assert r.ok and st["fatal"] == 0, (r.status, st)
        return r.gbps

    def per_granule(rows, n_granules: float) -> dict:
        """Bucket ns summed over the movers, as µs per granule moved."""
        tot = {k: sum(r[k] for r in rows) for k in rn.api.MOVER_PROFILE_FIELDS}
        out = {k[:-3]: round(tot[k] / n_granules / 1e3, 3) for k in rn.api.MOVER_PROFILE_FIELDS if k.endswith("_ns")}
        waits = sum(v for k, v in out.items() if k != "total")
        out["issue"] = round(out["total"] - waits, 3)
        out["chunks"] = tot["chunks"]
        return out

    def profile(n: int) -> dict:
        g = granule(MSG, n)
        prof.zero_()
        gb_c = ceiling(n, profile=True)         # rows are those of the last launch: n spans
        span = total // n // KSUB * KSUB
        ceil_rows = rn.api.mover_profile_rows(prof[:n * nf].cpu().tolist())
        gb_e = engine(n, profile=True)
        eng_rows = ctx.engine_mover_profile()
        os.environ.pop("RN_ENGINE_PROFILE", None)
        n_chunks = sum(r["chunks"] for r in eng_rows)
        assert n_chunks == ctx.engine_stats()["n_bulk_chunks"], (n_chunks, ctx.engine_stats())
        return {"ctas": n, "granule_bytes": g,
                "ceiling": {"gbps": round(gb_c, 1), "us_per_granule": per_granule(ceil_rows, n * span / g)},
                "engine": {"gbps": round(gb_e, 1), "us_per_granule": per_granule(eng_rows, n_chunks)}}

    def memcpy() -> float:
        with torch.cuda.stream(stream):
            for s in range(NSLOTS):
                dst[s * MSG:(s + 1) * MSG].copy_(src[s * MSG:(s + 1) * MSG], non_blocking=True)
            ev0.record(stream)
            n = 64
            for i in range(n):
                s = i % NSLOTS
                dst[s * MSG:(s + 1) * MSG].copy_(src[s * MSG:(s + 1) * MSG], non_blocking=True)
            ev1.record(stream)
        ev1.synchronize()
        return n * MSG / (ev0.elapsed_time(ev1) * 1e-3) / 1e9

    runs = {("ceiling", n): [] for n in ctas_list}
    runs.update({("engine", n): [] for n in ctas_list})
    runs[("memcpy", 0)] = []
    for rep in range(args.reps):
        for n in ctas_list:
            runs[("ceiling", n)].append(ceiling(n))
            runs[("engine", n)].append(engine(n))
            print(f"rep {rep} ctas {n}: ceiling {runs[('ceiling', n)][-1]:.1f} GB/s, engine {runs[('engine', n)][-1]:.1f} GB/s",
                  flush=True)
        runs[("memcpy", 0)].append(memcpy())
        print(f"rep {rep}: memcpy d2d {runs[('memcpy', 0)][-1]:.1f} GB/s", flush=True)

    profiles = []
    if args.profile:
        for n in ctas_list:
            profiles.append(profile(n))
            p = profiles[-1]
            print(f"profile ctas {n}: ceiling {p['ceiling']['us_per_granule']}", flush=True)
            print(f"profile ctas {n}: engine  {p['engine']['us_per_granule']}", flush=True)

    rows = []
    for n in ctas_list:
        a, b = summary(runs[("ceiling", n)]), summary(runs[("engine", n)])
        g = granule(MSG, n)
        t_a = g / (a["median"] * 1e9 / n) * 1e6
        t_b = g / (b["median"] * 1e9 / n) * 1e6
        rows.append({"ctas": n, "ceiling_gbps": a, "engine_gbps": b, "engine_frac_of_ceiling": round(b["median"] / a["median"], 3),
                     "ceiling_over_engine": round(a["median"] / b["median"], 3), "granule_bytes": g,
                     "us_per_granule_ceiling": round(t_a, 2), "us_per_granule_engine": round(t_b, 2),
                     "dead_us_per_chunk": round(t_b - t_a, 2)})
    out = {"card": card(), "msg_bytes": MSG, "window": 8, "nslots": NSLOTS, "reps": args.reps,
           "memcpy_d2d_gbps": summary(runs[("memcpy", 0)]), "rows": rows}
    if profiles:
        out["mover_profile"] = profiles
    ctx.close()
    print(json.dumps(out, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
