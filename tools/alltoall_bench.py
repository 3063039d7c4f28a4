"""The fp8 all-to-all and the all-to-all GEMM with N ranks simulated on one GPU, by host wall clock.

For N in (2, 4, 8), each rank holding x of M = 8192 rows and K = 4096 (M / N rows per destination), 256-row records,
Nb in (4096, 8192):
  fused       ``run_gemm``: K7 walks each rank's records as they land (``a_ready`` + ``a_order``)
  serial      the same launches with K7 started only after every rank's exchange has ended (host wait in between)
  scatter     ``run`` alone (bf16 out)
  compose     what a user can write without the scatter pack: per rank, N - 1 ``pack_fp8_write`` launches, one per
              destination, to ``staging_off = q R rec`` (their immediates collide, so nothing may read before the host
              wait), one more into the own slot, then a host wait and one plain unpack of the landing region
The four alternate, ``--reps`` times each, after one warm-up; min-max per configuration; every output, record and C is
checked against ``ops.ref_alltoall_fp8`` (C against K7 on the reference's records).  Then the engine's cost of idle queue
pairs: a ring all-gather (``run``, N = 4, the same bytes per rank) timed without and then with the 112 queue pairs of an
8-rank mesh created and connected but idle.  Every rank shares the one GPU, so this says nothing about N GPUs.  Prints
one JSON line per configuration, the card name and power limit first.

Under torchrun (one process per GPU, ``WORLD_SIZE`` > 1) each rank connects its plan with ``connect()`` and runs
``run`` ``--reps`` times, checking every output against the reference."""
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
from rocnrdma_b200.parallel import allgather_fp8 as AG, alltoall_fp8 as A2A  # noqa: E402
from rocnrdma_b200.parallel.ring_fp8 import _run_ranks  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [v.strip() for v in q.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), f"unknown ({e})"
    return dict(gpu=name, power_limit=power)


def _compose(p, x, out):
    """The enqueue of one rank's composed all-to-all: N - 1 pack_fp8_write launches plus the own slot's, on the main
    stream; the unpack runs after the host wait (see main)."""
    q, R, rec = p.rank, p.R, p.rec
    ms = p.main_stream
    ms.wait_event(p._cleared)
    for k, d in enumerate(A2A.phase_order(q, p.world)):
        shard = x[d * p.shard:(d + 1) * p.shard]
        post = {} if d == q else dict(qp=p.send_qps[d], dst_mr=p.remote_landings[d], with_imm=True)
        mr = p.landing_mr if d == q else p.staging_mr
        v, _ = ops.pack_fp8_write(p.ctx, shard, mr, chunk_elems=p.chunk, staging_off=q * R * rec, grid=p.grid,
                                  timeout_ms=p.timeout_ms, stream=ms, sync=False, scratch_slot=p.scratch_slot,
                                  result_off=p._res(3 + k), **post)
        p._views.append((f"pack {d}", "pack", v))


def one_gpu(a):
    print(json.dumps(card()), flush=True)
    ctx = rn.Context(0, wire="softhca")
    M, K = 8192, 4096
    chunk = 256 * K
    for N in [int(v) for v in a.worlds.split(",")]:
        rows = M // N
        plans = [A2A.AllToAllFp8(ctx, rows * K, chunk, q, N, engine_ctas=a.engine_ctas) for q in range(N)]
        A2A.link_in_process(plans)
        g = torch.Generator().manual_seed(N)
        xs_cpu = [torch.randn(M, K, generator=g).to(torch.bfloat16) for _ in range(N)]
        xs = [x.cuda() for x in xs_cpu]
        xf = [x.reshape(-1) for x in xs]
        outs = [torch.zeros(M * K, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
        outs_c = [torch.zeros_like(o) for o in outs]
        want, want_rec = ops.ref_alltoall_fp8([x.reshape(-1) for x in xs_cpu], chunk)
        for Nb in [int(v) for v in a.nbs.split(",")]:
            bq, bs = MX.quantize_mx(torch.randn(Nb, K, device="cuda").to(torch.bfloat16))
            b = MX.MxOperand.from_tensors(bq, bs)
            cs = [torch.zeros(M, Nb, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
            c_serial = [torch.zeros_like(c) for c in cs]
            a_ops = [MX.MxOperand.from_chunk_records(p.records(), M, K, chunk) for p in plans]
            torch.cuda.synchronize()

            def fused():
                return A2A.run_gemm_in_process(plans, xs, [b] * N, cs)

            def serial():
                res = _run_ranks(plans, [lambda p=p, x=x: p._enqueue_scatter(x) for p, x in zip(plans, xf)], True, ())
                for p, ao, c in zip(plans, a_ops, c_serial):
                    ops.gemm_mxfp8(ctx, ao, b, c, grid=p.grid, stream=p.compute_stream, sync=False,
                                   scratch_slot=p.scratch_slot, cta_group=1, a_ready=p.words, a_order=p.a_order)
                for p in plans:
                    p.compute_stream.synchronize()
                return res

            def scatter():
                return A2A.run_in_process(plans, xf, outs)

            def compose():
                res = _run_ranks(plans, [lambda p=p, x=x, o=o: _compose(p, x, o) for p, x, o in zip(plans, xf, outs_c)],
                                 True, ())
                # the composed packs report no per-destination counts: a clean run leaves nothing for the next one
                assert all(r.ok for r in res), [(r.rank, r.status, r.failed) for r in res]
                for p in plans:
                    p._stale_cqes = p._rq_backlog = 0
                    p._backlogs = [0] * N
                for p, o in zip(plans, outs_c):
                    ops.unpack_fp8(ctx, p.landing, o, chunk, grid=p.grid, stream=p.compute_stream, sync=False,
                                   scratch_slot=p.scratch_slot, result_off=p._res(3))
                for p in plans:
                    p.compute_stream.synchronize()
                return res

            runs = (("fused", fused), ("serial", serial), ("scatter", scatter), ("compose", compose))
            times = {name: [] for name, _ in runs}
            ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=10000)
            try:
                for _, fn in runs:
                    fn()
                for _ in range(a.reps):
                    for name, fn in runs:
                        t0 = time.perf_counter()
                        res = fn()
                        times[name].append((time.perf_counter() - t0) * 1e3)
                        bad = [(r.rank, r.status, r.failed) for r in res if not r.ok]
                        assert not bad, (name, bad)
            finally:
                ctx.engine_stop()
            out_ok = all(torch.equal(o.cpu().view(torch.int16), w.view(torch.int16)) for o, w in zip(outs, want))
            compose_ok = all(torch.equal(o.cpu().view(torch.int16), w.view(torch.int16)) for o, w in zip(outs_c, want))
            records_ok = all(torch.equal(p.records().cpu(), r) for p, r in zip(plans, want_rec))
            c_ref = [torch.zeros_like(c) for c in cs]
            for q in range(N):
                ao = MX.MxOperand.from_chunk_records(want_rec[q].cuda(), M, K, chunk)
                assert ops.gemm_mxfp8(ctx, ao, b, c_ref[q], cta_group=1).ok
            c_ok = all(torch.equal(c.view(torch.int16), r.view(torch.int16)) for c, r in zip(cs + c_serial, c_ref + c_ref))
            line = dict(N=N, M=M, K=K, Nb=Nb, rows_per_destination=rows, chunk=chunk, grid=plans[0].grid,
                        engine_ctas=a.engine_ctas, reps=a.reps, out_matches_reference=out_ok,
                        composed_out_matches_reference=compose_ok, records_match_reference=records_ok,
                        c_matches_k7_on_reference_records=c_ok)
            for name, t in times.items():
                line[f"{name}_ms_min"], line[f"{name}_ms_max"] = round(min(t), 3), round(max(t), 3)
            print(json.dumps(line), flush=True)
    ctx.close()
    idle_qps(a)


def idle_qps(a):
    """A ring all-gather of N = 4 (8192 x 4096 bf16 per rank in all), timed without and then with an 8-rank mesh's
    112 queue pairs created and connected but idle, in a context of its own (the plans above hold its queue pairs)."""
    ctx = rn.Context(0, wire="softhca")
    N, M, K = 4, 8192, 4096
    chunk, rows = 256 * K, M // 4
    plans = [AG.RingAllgatherFp8(ctx, rows * K, chunk, q, N, engine_ctas=a.engine_ctas) for q in range(N)]
    AG.link_in_process(plans)
    xs = [torch.randn(rows * K, device="cuda").to(torch.bfloat16) for _ in range(N)]
    outs = [torch.zeros(N * rows * K, dtype=torch.bfloat16, device="cuda") for _ in range(N)]
    torch.cuda.synchronize()

    def timed():
        t = []
        ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=10000)
        try:
            AG.run_in_process(plans, xs, outs)
            for _ in range(a.reps):
                t0 = time.perf_counter()
                res = AG.run_in_process(plans, xs, outs)
                t.append((time.perf_counter() - t0) * 1e3)
                assert all(r.ok for r in res), [(r.rank, r.status) for r in res]
        finally:
            ctx.engine_stop()
        return t

    without = timed()
    mesh = [A2A._mesh_qps(ctx, q, 8, 7 * 4, 4, 256) for q in range(8)]
    for s in range(8):
        for d in range(8):
            if s != d:
                mesh[s][0][d].connect(mesh[d][1][s])
    torch.cuda.synchronize()
    with_idle = timed()
    want = ops.ref_allgather_fp8([x.cpu() for x in xs], chunk)[0]
    ok = all(torch.equal(o.cpu().view(torch.int16), want.view(torch.int16)) for o in outs)
    print(json.dumps(dict(idle_qps=112, allgather_N=N, rows_per_rank=rows, K=K, chunk=chunk, reps=a.reps,
                          out_matches_reference=ok, without_idle_ms_min=round(min(without), 3),
                          without_idle_ms_max=round(max(without), 3), with_idle_ms_min=round(min(with_idle), 3),
                          with_idle_ms_max=round(max(with_idle), 3))), flush=True)
    ctx.close()


def multi_gpu(a):
    import torch.distributed as dist
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    ctx = rn.Context(dev, wire="softhca")
    for peer in range(torch.cuda.device_count()):
        if peer != dev:
            ctx.enable_peer(peer)
    K, rows, chunk = 4096, 1024, 256 * 4096
    plan = A2A.AllToAllFp8(ctx, rows * K, chunk, rank, world, timeout_ms=5000, engine_ctas=a.engine_ctas)
    plan.connect()
    g = torch.Generator().manual_seed(world)
    xs = [torch.randn(world * rows * K, generator=g).to(torch.bfloat16) for _ in range(world)]
    want = ops.ref_alltoall_fp8(xs, chunk)[0][rank]
    x = xs[rank].to(f"cuda:{dev}")
    out = torch.zeros_like(x)
    torch.cuda.synchronize()
    t = []
    for rep in range(a.reps + 1):
        dist.barrier()
        ctx.engine_start(ctas=a.engine_ctas, idle_timeout_ms=5000)
        try:
            t0 = time.perf_counter()
            r = plan.run(x, out)
            dt = time.perf_counter() - t0
        finally:
            ctx.engine_stop()
        if not r.ok or not torch.equal(out.cpu().view(torch.int16), want.view(torch.int16)):
            raise SystemExit(f"rank {rank}: {r.status} {r.failed}, or the output differs from ref_alltoall_fp8")
        if rep:
            t.append(dt * 1e3)
    if rank == 0:
        print(json.dumps(dict(world=world, rows_per_destination=rows, K=K, chunk=chunk, run_ms_min=round(min(t), 3),
                              run_ms_max=round(max(t), 3), **card())), flush=True)
    ctx.close()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--engine-ctas", type=int, default=16)
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--nbs", default="4096,8192")
    a = ap.parse_args()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        return multi_gpu(a)
    one_gpu(a)


if __name__ == "__main__":
    main()
