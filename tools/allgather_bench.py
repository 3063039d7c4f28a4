"""The fp8 ring all-gather and the all-gather GEMM with N ranks simulated on one GPU, by host wall clock.

For N in (2, 4), a total M of 8192 rows, K = 4096 and Nb in (4096, 8192):
  fused       ``run_gemm``: K7 walks each rank's records as they land (``a_ready`` + ``a_order``)
  serial      the same launches with K7 started only after every rank's gather has ended (host wait in between)
  gather      ``run`` alone (bf16 out), every output checked against ``ops.ref_allgather_fp8`` afterwards
The three alternate, ``--reps`` times each, after one warm-up; min-max per configuration.  Every rank shares the one GPU
(its SMs, its HBM and the software HCA's engine), so this says nothing about N GPUs.  Prints one JSON line per
configuration, the card name and power limit first."""
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
from rocnrdma_b200.ops import gemm_mx as MX  # noqa: E402
from rocnrdma_b200.parallel import allgather_fp8 as AG  # noqa: E402
from rocnrdma_b200.parallel.ring_fp8 import _run_ranks  # noqa: E402


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
    M, K = 8192, 4096
    chunk = 256 * K
    for N in [int(v) for v in args.worlds.split(",")]:
        rows = M // N
        plans = [AG.RingAllgatherFp8(ctx, rows * K, chunk, q, N, engine_ctas=args.engine_ctas) for q in range(N)]
        AG.link_in_process(plans)
        g = torch.Generator().manual_seed(N)
        xs_cpu = [torch.randn(rows, K, generator=g).to(torch.bfloat16) for _ in range(N)]
        xs = [x.cuda() for x in xs_cpu]
        outs = [torch.zeros(M * K, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
        for Nb in [int(v) for v in args.nbs.split(",")]:
            bq, bs = MX.quantize_mx(torch.randn(Nb, K, device="cuda").to(torch.bfloat16))
            b = MX.MxOperand.from_tensors(bq, bs)
            cs = [torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
            c_serial = [torch.zeros_like(c) for c in cs]
            a_ops = [MX.MxOperand.from_chunk_records(p.records(), M, K, chunk) for p in plans]
            torch.cuda.synchronize()

            def fused():
                return AG.run_gemm_in_process(plans, xs, [b] * N, cs)

            def serial():
                res = _run_ranks(plans, [lambda p=p, x=x: p._enqueue_gather(x.reshape(-1)) for p, x in zip(plans, xs)],
                                 True, ())
                for p, a, c in zip(plans, a_ops, c_serial):
                    ops.gemm_mxfp8(ctx, a, b, c, grid=p.grid, stream=p.compute_stream, sync=False,
                                   scratch_slot=p.scratch_slot, cta_group=1, a_ready=p.words, a_order=p.a_order)
                for p in plans:
                    p.compute_stream.synchronize()
                return res

            def gather():
                return AG.run_in_process(plans, xs, outs)

            times = {"fused": [], "serial": [], "gather": []}
            ctx.engine_start(ctas=args.engine_ctas, idle_timeout_ms=10000)
            try:
                for fn in (fused, serial, gather):
                    fn()
                for _ in range(args.reps):
                    for name, fn in (("fused", fused), ("serial", serial), ("gather", gather)):
                        t0 = time.perf_counter()
                        res = fn()
                        times[name].append((time.perf_counter() - t0) * 1e3)
                        bad = [(r.rank, r.status, r.failed) for r in res if not r.ok]
                        assert not bad, (name, bad)
            finally:
                ctx.engine_stop()
            want, want_rec = ops.ref_allgather_fp8([x.reshape(-1) for x in xs_cpu], chunk)
            gather_ok = all(torch.equal(o.cpu().view(torch.int16), want.view(torch.int16)) for o in outs)
            records_ok = all(torch.equal(p.records().cpu(), want_rec) for p in plans)
            c_same = all(torch.equal(c.view(torch.int16), cs[0].view(torch.int16)) for c in cs + c_serial)
            line = dict(N=N, M=M, K=K, Nb=Nb, rows_per_rank=rows, chunk=chunk, grid=plans[0].grid,
                        engine_ctas=args.engine_ctas, reps=args.reps, gather_matches_reference=gather_ok,
                        records_match_reference=records_ok, c_identical_on_every_rank_and_path=c_same)
            for name, t in times.items():
                line[f"{name}_ms_min"], line[f"{name}_ms_max"] = round(min(t), 3), round(max(t), 3)
            line["gemm_tflops_fused_best"] = round(N * 2.0 * M * Nb * K / (min(times["fused"]) * 1e-3) / 1e12, 1)
            print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
