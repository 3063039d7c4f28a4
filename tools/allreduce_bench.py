"""The fp8 ring all-reduce (``parallel.ring_fp8``), timed.  Needs a GPU.

One GPU (``python tools/allreduce_bench.py``): N = 2, 4 and 8 simulated ranks in one context, 2^26 bf16 elements each.
The fused run (every hop started on the device) alternates with a host-stepped run of the same launches that
synchronises every rank's main stream after each step.  Every output is checked against ``ops.ref_allreduce_fp8``.

Under torchrun with two or more GPUs (``torchrun --nproc-per-node G tools/allreduce_bench.py``): one rank per GPU through
``connect_ring``, alternated with ``torch.distributed.all_reduce`` of the same bf16 tensors over NCCL, run while no
engine is resident.

With ``--error-feedback`` (one GPU): the fused run without error feedback alternates with the fused run with it
(``RingAllreduceFp8(error_feedback=True)``, its residuals threaded from run to run), each output checked against
``ops.ref_allreduce_fp8`` for its mode (with ``residuals=`` for the second).

Times are host wall clock around work that ends in a stream synchronise, plus the device span of the fused run (first
launch start to last launch end).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import rocnrdma_b200 as rn  # noqa: E402
from rocnrdma_b200 import ops  # noqa: E402
from rocnrdma_b200.parallel import ring_fp8 as RF  # noqa: E402
from tools.pull_bench import _spread, gpu_info  # noqa: E402


def _inputs(N, n, seed, device="cuda"):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    return [(torch.randn(n, generator=g) * 4).to(torch.bfloat16).to(device) for _ in range(N)]


def _timed_run(ctx, plans, xs, outs, a):
    for o in outs:
        o.zero_()
    torch.cuda.synchronize()
    ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=a.timeout_ms)
    try:
        t0 = time.perf_counter()
        res = RF.run_in_process(plans, xs, outs)
        dt = time.perf_counter() - t0
    finally:
        ctx.engine_stop()
    return res, dt


def one_gpu_error_feedback(a):
    """Alternate the ring without and with error feedback; the same inputs, every output checked."""
    ctx = rn.Context(0, wire="softhca")
    rows = []
    for N in a.ranks:
        n = a.elems
        modes = {}
        for ef in (False, True):
            plans = [RF.RingAllreduceFp8(ctx, n, a.chunk, q, N, timeout_ms=a.timeout_ms, engine_ctas=a.engine_ctas,
                                         error_feedback=ef) for q in range(N)]
            RF.link_in_process(plans)
            modes[ef] = plans
        xs = _inputs(N, n, seed=N)
        outs = [torch.zeros_like(x) for x in xs]
        want_off = ops.ref_allreduce_fp8(xs, a.chunk)
        ref_res = [torch.zeros(n, dtype=torch.float32, device="cuda") for _ in range(N)]
        times = {False: [], True: []}
        device = {False: [], True: []}
        launches = {False: {}, True: {}}
        for rep in range(a.reps + 1):                      # rep 0 warms both up and is not recorded
            for ef in (False, True):
                if ef:
                    want, ref_res = ops.ref_allreduce_fp8(xs, a.chunk, residuals=ref_res)
                else:
                    want = want_off
                res, dt = _timed_run(ctx, modes[ef], xs, outs, a)
                bad = [(r.rank, r.status, r.failed) for r in res if not r.ok]
                if bad:
                    raise SystemExit(f"N={N} error_feedback={ef}: {bad}")
                for q, o in enumerate(outs):
                    if not torch.equal(o.view(torch.int16), want.view(torch.int16)):
                        raise SystemExit(f"N={N} error_feedback={ef}: rank {q} differs from ref_allreduce_fp8")
                if ef:
                    for q, p in enumerate(modes[ef]):
                        if not torch.equal(p.residual.view(torch.int32), ref_res[q].view(torch.int32)):
                            raise SystemExit(f"N={N}: rank {q}'s residual differs from ref_allreduce_fp8")
                if rep:
                    times[ef].append(dt * 1e3)
                    device[ef].append(max(r.total_ns for r in res) / 1e6)
                    # rank 0's launches of its last run in this mode: where the time went
                    launches[ef] = {l.name: round(l.device_ns / 1e6, 3) for l in res[0].launches if l.name != "receive"}
        row = dict(ranks=N, elems=n, chunk=a.chunk, ef_off_ms=_spread(times[False]), ef_on_ms=_spread(times[True]),
                   ef_off_device_ms=_spread(device[False]), ef_on_device_ms=_spread(device[True]),
                   ef_off_launch_ms=launches[False], ef_on_launch_ms=launches[True],
                   outputs_checked=True, residuals_checked=True)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del modes, xs, outs, want, want_off, ref_res
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    ctx.close()
    return rows


def one_gpu(a):
    ctx = rn.Context(0, wire="softhca")
    rows = []
    for N in a.ranks:
        n = a.elems
        plans = [RF.RingAllreduceFp8(ctx, n, a.chunk, q, N, timeout_ms=a.timeout_ms, engine_ctas=a.engine_ctas)
                 for q in range(N)]
        RF.link_in_process(plans)
        xs = _inputs(N, n, seed=N)
        outs = [torch.zeros_like(x) for x in xs]
        want = ops.ref_allreduce_fp8(xs, a.chunk)
        torch.cuda.synchronize()
        fused, stepped, device = [], [], []
        for rep in range(a.reps + 1):                      # rep 0 warms both up and is not recorded
            for mode in ("fused", "stepped"):
                for o in outs:
                    o.zero_()
                torch.cuda.synchronize()
                ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=a.timeout_ms)
                try:
                    t0 = time.perf_counter()
                    if mode == "fused":
                        res = RF.run_in_process(plans, xs, outs)
                    else:
                        for p in plans:
                            p.start_consumer()
                        for i in range(2 * N):
                            for p, x, o in zip(plans, xs, outs):
                                p.enqueue_main(x, o, steps=(i,))
                            for p in plans:
                                p.main_stream.synchronize()
                        for p in plans:
                            p.synchronize()
                        res = [p.result() for p in plans]
                    dt = time.perf_counter() - t0
                finally:
                    ctx.engine_stop()
                bad = [(r.rank, r.status, r.failed) for r in res if not r.ok]
                if bad:
                    raise SystemExit(f"N={N} {mode}: {bad}")
                for q, o in enumerate(outs):
                    if not torch.equal(o.view(torch.int16), want.view(torch.int16)):
                        raise SystemExit(f"N={N} {mode}: rank {q} differs from ref_allreduce_fp8")
                if rep:
                    (fused if mode == "fused" else stepped).append(dt * 1e3)
                    if mode == "fused":
                        device.append(max(r.total_ns for r in res) / 1e6)
        row = dict(ranks=N, elems=n, chunk=a.chunk, fused_ms=_spread(fused), stepped_ms=_spread(stepped),
                   fused_device_ms=_spread(device), outputs_checked=True)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del plans, xs, outs, want
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    ctx.close()
    return rows


def multi_gpu(a):
    import torch.distributed as dist
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    ctx = rn.Context(dev, wire="softhca")
    for peer in range(torch.cuda.device_count()):
        if peer != dev:
            ctx.enable_peer(peer)
    plan = RF.RingAllreduceFp8(ctx, a.elems, a.chunk, rank, world, timeout_ms=a.timeout_ms, engine_ctas=a.engine_ctas)
    plan.connect()
    xs = _inputs(world, a.elems, seed=world, device="cpu")
    want = ops.ref_allreduce_fp8(xs, a.chunk)
    x = xs[rank].to(f"cuda:{dev}")
    out = torch.zeros_like(x)
    y = x.clone()
    torch.cuda.synchronize()
    ring, nccl = [], []
    for rep in range(a.reps + 1):
        dist.barrier()
        ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=a.timeout_ms)
        try:
            t0 = time.perf_counter()
            r = plan.run(x, out)
            dt = time.perf_counter() - t0
        finally:
            ctx.engine_stop()
        if not r.ok or not torch.equal(out.cpu().view(torch.int16), want.view(torch.int16)):
            raise SystemExit(f"rank {rank}: {r.status} {r.failed}, or the output differs from ref_allreduce_fp8")
        dist.barrier()
        y.copy_(x)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        dist.all_reduce(y)
        torch.cuda.synchronize()
        d2 = time.perf_counter() - t1
        if rep:
            ring.append(dt * 1e3)
            nccl.append(d2 * 1e3)
    if rank == 0:
        print(json.dumps(dict(world=world, elems=a.elems, chunk=a.chunk, ring_fp8_ms=_spread(ring),
                              nccl_bf16_all_reduce_ms=_spread(nccl), **gpu_info())), flush=True)
    ctx.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--elems", type=int, default=1 << 26)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engine-ctas", type=int, default=16)
    ap.add_argument("--timeout-ms", type=int, default=5000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--error-feedback", action="store_true",
                    help="alternate the ring without and with error feedback (one GPU)")
    a = ap.parse_args()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        return multi_gpu(a)
    info = gpu_info()
    print(json.dumps(info), flush=True)
    rows = one_gpu_error_feedback(a) if a.error_feedback else one_gpu(a)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(rows=rows, **info), f, indent=1)


if __name__ == "__main__":
    main()
