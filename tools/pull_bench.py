"""What pulling records with arrival words costs and buys on the software HCA, one JSON record on stdout.

    python tools/pull_bench.py [--ctas 32] [--reps 3] [--out FILE]

One device-posted loopback QP, engine on --ctas SMs, alternated --reps times after one warm-up round:
* stamping: ops.read_records (one arrival word per record) against ops.rdma_stream(OP_RDMA_READ) moving the same
  records, 64 KiB, 1 MiB and 4 MiB each, 256 MiB per run, window 16: GB/s from the device timers (first post to last
  completion);
* K5: read_records, then unpack_fp8(ready=) unpacking each record as it lands on a second stream, against read_records
  followed by unpack_fp8 on one stream, at 2^26 bf16 elements in 64 K3 chunk records (a permutation of the source's);
* K7: read_records of the 32 K4 panel records of a 4096 x 4096 fp8 operand, then gemm_mxfp8(a_ready=) multiplying them
  by a 4096 x 4096 operand as they land, against the pull followed by the GEMM on one stream.  The GEMM runs as 96
  single CTAs (cta_group 1): every CTA of a kernel that waits on the poster must be resident before the poster is
  launched, and 48 two-CTA clusters do not all find a place beside the engine, so the cluster left waiting holds the
  poster's launch back until the resident tiles give up.
SMs: engine --ctas + poster 1 + K5 64 (97 at the default), or + K7 96 (129).
K5 and K7 times run from the pull's first post to the consumer's end (device timers), min-max over the runs.  Each
result is checked against the same computation run after arrival.  The card's name and power limit are read in the
same run.  Needs a GPU.
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
from rocnrdma_b200.ops import gemm_mx as MX, launch as L  # noqa: E402


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
        sys.exit("pull_bench needs a GPU")
    TMO = 20000
    total = 256 << 20
    sizes = (64 << 10, 1 << 20, 4 << 20)
    chunk, n_elems = 1 << 20, 1 << 26
    n_chunks, crec = n_elems // chunk, ops.record_bytes(chunk)
    M = N_ = K = 4096
    prec = ops.panel_record_bytes(K)
    n_panels = M // 128
    if a.ctas + 1 + 96 > 132:
        sys.exit(f"--ctas {a.ctas}: the engine, the poster and K7's 96 CTAs must all be resident on the 132 SMs")
    rec = {"bench": "pull", "engine_ctas": a.ctas, "window": 16, "sm_sum": {"k5": a.ctas + 1 + 64, "k7": a.ctas + 1 + 96},
           **gpu_info()}
    ctx = rn.Context(0)
    try:
        g = torch.Generator(device="cuda").manual_seed(5)
        src = torch.randint(0, 256, (total,), dtype=torch.uint8, device="cuda", generator=g)
        dst = torch.zeros(total, dtype=torch.uint8, device="cuda")
        sm, dm = ctx.reg_mr(src), ctx.reg_mr(dst)
        words = torch.zeros(max(total // min(sizes), n_chunks, n_panels), dtype=torch.int64, device="cuda")
        # K5: K3 records of seeded bf16 and a permutation
        x = torch.randn(n_elems, device="cuda", generator=g).to(torch.bfloat16)
        crecs = ops.ref_pack_fp8(x, chunk)
        perm = torch.randperm(n_chunks, device="cuda", generator=g).to(torch.int32)
        want5 = ops.ref_unpack_fp8(crecs.view(n_chunks, crec)[perm.long()].reshape(-1), n_elems, chunk)
        y5 = {k: torch.empty(n_elems, dtype=torch.bfloat16, device="cuda") for k in ("on_arrival", "after_pull")}
        cm = ctx.reg_mr(crecs)
        land5 = dst[:n_chunks * crec]
        # K7: panel records of a 4096 x 4096 operand, B from tensors
        prs = ops.ref_fp8_panels(torch.randn(M, K, device="cuda", generator=g))
        pm = ctx.reg_mr(prs)
        land7 = dst[:n_panels * prec]
        bq, bs = MX.quantize_mx(torch.randn(N_, K, device="cuda", generator=g))
        a_op, b_op = MX.MxOperand.from_panel_records(land7, M, K), MX.MxOperand.from_tensors(bq, bs)
        y7 = {k: torch.empty(M, N_, dtype=torch.bfloat16, device="cuda") for k in ("on_arrival", "after_pull")}
        qp = ctx.loopback_qp(depth=256)
        s_pull, s_use = ctx.streams(2)
        with torch.cuda.stream(s_pull):
            words.zero_()                                     # loaded before any engine is resident
        torch.cuda.synchronize()
        res = {f"stamp_{s >> 10}KiB": {"read_records": [], "rdma_stream_read": []} for s in sizes}
        res["k5_2^26"] = {"on_arrival": [], "after_pull": []}
        res["k7_4096^3_panels"] = {"on_arrival": [], "after_pull": []}
        checks = {k: True for k in ("stamp_read_records", "stamp_rdma_stream_read", "k5_on_arrival_words", "k5_after_pull_words",
                                    "k5_on_arrival_exact", "k5_after_pull_exact", "k7_on_arrival_words", "k7_after_pull_words",
                                    "k7_same_bits")}

        def zero_words():
            # zeroed on the pull stream and finished before the consumer starts: no allocation, no device-wide
            # synchronise while the engine runs
            with torch.cuda.stream(s_pull):
                words.zero_()
            s_pull.synchronize()

        for rep in range(a.reps + 1):                         # rep 0 warms up every shape
            keep = rep > 0
            ctx.engine_start(ctas=a.ctas, idle_timeout_ms=TMO)
            try:
                for s in sizes:
                    n = total // s
                    for kind in ("read_records", "rdma_stream_read"):
                        if kind == "read_records":
                            zero_words()
                            r = ops.read_records(qp, sm, dm, s, n, ready=words, window=16, timeout_ms=TMO, stream=s_pull)
                            good, ns = r["status"] == "OK" and r["done"] == n, r["device_ns"]
                        else:
                            r = ops.rdma_stream(qp, W.OP_RDMA_READ, dm, sm, s, iters=n, window=16, slot_stride=s, nslots=n,
                                                timeout_ms=TMO, stream=s_pull)
                            good, ns = r.ok, r.device_ns
                        checks[f"stamp_{kind}"] &= good
                        if keep:
                            res[f"stamp_{s >> 10}KiB"][kind].append(total / max(ns, 1))
                # K5
                for kind in ("on_arrival", "after_pull"):
                    zero_words()
                    if kind == "on_arrival":
                        uv, _ = ops.unpack_fp8(ctx, land5, y5[kind], chunk, ready=words[:n_chunks], grid=64, timeout_ms=TMO,
                                               sync=False, stream=s_use)
                        pv, _ = ops.read_records(qp, cm, dm, crec, n_chunks, indices=perm, ready=words, window=16,
                                                 timeout_ms=TMO, sync=False, stream=s_pull)
                        s_pull.synchronize(); s_use.synchronize()
                    else:
                        pv, _ = ops.read_records(qp, cm, dm, crec, n_chunks, indices=perm, ready=words, window=16,
                                                 timeout_ms=TMO, sync=False, stream=s_pull)
                        uv, _ = ops.unpack_fp8(ctx, land5, y5[kind], chunk, grid=64, timeout_ms=TMO, sync=False, stream=s_pull)
                        s_pull.synchronize()
                    p, u = ops.parse_read_records(pv), ops.parse_unpack(uv)
                    checks[f"k5_{kind}_words"] &= p["status"] == "OK" and p["done"] == n_chunks and u["status"] == "OK"
                    if keep:
                        res["k5_2^26"][kind].append((u["t_end_ns"] - p["t_start_ns"]) / 1e3)
                # K7
                for kind in ("on_arrival", "after_pull"):
                    zero_words()
                    if kind == "on_arrival":
                        gv, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y7[kind], grid=96, cta_group=1, a_ready=words[:n_panels], timeout_ms=TMO,
                                               sync=False, stream=s_use)
                        pv, _ = ops.read_records(qp, pm, dm, prec, n_panels, ready=words, window=16, timeout_ms=TMO,
                                                 sync=False, stream=s_pull)
                        s_pull.synchronize(); s_use.synchronize()
                    else:
                        pv, _ = ops.read_records(qp, pm, dm, prec, n_panels, ready=words, window=16, timeout_ms=TMO,
                                                 sync=False, stream=s_pull)
                        gv, _ = ops.gemm_mxfp8(ctx, a_op, b_op, y7[kind], grid=96, cta_group=1, timeout_ms=TMO, sync=False,
                                               stream=s_pull)
                        s_pull.synchronize()
                    p, gw = ops.parse_read_records(pv), L.decode(gv)
                    checks[f"k7_{kind}_words"] &= p["status"] == "OK" and p["done"] == n_panels and gw["status"] == "OK"
                    if keep:
                        res["k7_4096^3_panels"][kind].append((gw["t_end_ns"] - p["t_start_ns"]) / 1e3)
            finally:
                ctx.engine_stop()
            for kind in ("on_arrival", "after_pull"):       # the engine is gone: full-device work is safe again
                checks[f"k5_{kind}_exact"] &= bool(torch.equal(y5[kind].view(torch.int16), want5.view(torch.int16)))
            checks["k7_same_bits"] &= bool(torch.equal(y7["on_arrival"].view(torch.int16), y7["after_pull"].view(torch.int16)))
        for key, d in res.items():
            unit = "GB/s" if key.startswith("stamp") else "us"
            rec[key] = {k: {**_spread(v), "unit": unit} for k, v in d.items()}
        rec["checks"] = checks
        rec["verified"] = all(checks.values())
    finally:
        ctx.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")
    return 0 if rec.get("verified") else 1


if __name__ == "__main__":
    sys.exit(main())
