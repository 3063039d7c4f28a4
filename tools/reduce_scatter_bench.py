"""The fp8 ring reduce-scatter and the GEMM-reduce-scatter with N ranks simulated on one GPU, by host wall clock.

For N in (2, 4), M = 8192 rows, a total K of 8192 (each rank holds K_l = K / N) and Nb in (4096, 8192):
  fused       ``run_gemm``: each rank's panels are reduced with the landed sum and posted on as its GEMM finishes them
  unfused     every rank's ``gemm_send`` (bf16 C [M, Nb]) in its default variant (CTA pairs), then ``run`` on the C's
  unfused1    the same with ``gemm_send(cta_group=1)``: the single-CTA tile body the fused kernel also runs
  run         ``run`` alone, on the C's the unfused path made
The four alternate, ``--reps`` times each, after one warm-up; min-max per configuration.  Every output is checked
against ``ops.ref_reduce_scatter_fp8`` afterwards.  Every rank shares the one GPU (its SMs, its HBM and the software HCA's
engine), so this says nothing about N GPUs.  Prints one JSON line per configuration, the card name and power limit
first."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops  # noqa: E402
from rocnrdma_b200.parallel import reduce_scatter_fp8 as RS  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [v.strip() for v in q.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), f"unknown ({e})"
    return dict(gpu=name, power_limit=power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engine-ctas", type=int, default=16)
    ap.add_argument("--worlds", default="2,4")
    ap.add_argument("--nbs", default="4096,8192")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    ctx = rn.Context(0, wire="softhca")
    M, K = 8192, 8192
    for N in [int(v) for v in args.worlds.split(",")]:
        Kl = K // N
        g = torch.Generator().manual_seed(N)
        # small integers: every partial is exact, so the reference is exact whatever the order of the adds
        a_cpu = [torch.randint(-2, 3, (M, Kl), generator=g).to(torch.bfloat16) for _ in range(N)]
        a = [t.cuda() for t in a_cpu]
        for Nb in [int(v) for v in args.nbs.split(",")]:
            chunk = 128 * Nb
            plans = [RS.RingReduceScatterFp8(ctx, (M // N) * Nb, chunk, q, N, engine_ctas=args.engine_ctas) for q in range(N)]
            RS.link_in_process(plans)
            b_cpu = [torch.randint(-2, 3, (Nb, Kl), generator=g).to(torch.bfloat16) for _ in range(N)]
            b = [t.cuda() for t in b_cpu]
            outs_f = [torch.zeros(M // N, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
            outs_u = [torch.zeros((M // N) * Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
            cs = [torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
            torch.cuda.synchronize()

            def fused():
                return RS.run_gemm_in_process(plans, a, b, outs_f)

            def unfused():
                for p, x, y, c in zip(plans, a, b, cs):
                    ops.gemm_send(ctx, x, y, c, grid=p.grid, stream=p.main_stream, sync=False, scratch_slot=p.scratch_slot)
                return RS.run_in_process(plans, [c.reshape(-1) for c in cs], outs_u)

            def unfused1():
                for p, x, y, c in zip(plans, a, b, cs):
                    ops.gemm_send(ctx, x, y, c, cta_group=1, grid=p.grid, stream=p.main_stream, sync=False,
                                  scratch_slot=p.scratch_slot)
                return RS.run_in_process(plans, [c.reshape(-1) for c in cs], outs_u)

            def run():
                return RS.run_in_process(plans, [c.reshape(-1) for c in cs], outs_u)

            times = {"fused": [], "unfused": [], "unfused1": [], "run": []}
            ctx.engine_start(ctas=args.engine_ctas, idle_timeout_ms=10000)
            try:
                for fn in (fused, unfused, unfused1, run):
                    fn()
                for _ in range(args.reps):
                    for name, fn in (("fused", fused), ("unfused", unfused), ("unfused1", unfused1), ("run", run)):
                        t0 = time.perf_counter()
                        res = fn()
                        times[name].append((time.perf_counter() - t0) * 1e3)
                        bad = [(r.rank, r.status, r.failed) for r in res if not r.ok]
                        assert not bad, (name, bad)
            finally:
                ctx.engine_stop()
            parts = [(x.float() @ y.float().T).reshape(-1) for x, y in zip(a_cpu, b_cpu)]
            want_f = ops.ref_reduce_scatter_fp8(parts, chunk)
            want_u = ops.ref_reduce_scatter_fp8([c.cpu().reshape(-1) for c in cs], chunk)
            fused_ok = all(torch.equal(o.cpu().reshape(-1).view(torch.int16), w.view(torch.int16)) for o, w in zip(outs_f, want_f))
            unfused_ok = all(torch.equal(o.cpu().view(torch.int16), w.view(torch.int16)) for o, w in zip(outs_u, want_u))
            line = dict(N=N, M=M, K=K, K_l=Kl, Nb=Nb, chunk=chunk, grid=plans[0].grid, engine_ctas=args.engine_ctas,
                        reps=args.reps, fused_matches_reference=fused_ok, unfused_matches_reference=unfused_ok)
            for name, t in times.items():
                line[f"{name}_ms_min"], line[f"{name}_ms_max"] = round(min(t), 3), round(max(t), 3)
            print(json.dumps(line), flush=True)
            del plans
    ctx.close()


if __name__ == "__main__":
    main()
