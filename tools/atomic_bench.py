"""Remote atomics and put-with-signal on the software HCA, one JSON record on stdout.

    python tools/atomic_bench.py [--ctas 32] [--out FILE]

* device-posted FETCH_AND_ADD, microseconds per atomic: 1 QP (window 16, bursts of 8), 32 QPs on one shared word,
  32 QPs on distinct words;
* put-with-signal (RDMA WRITE + FA on a signal word, one doorbell) at 64 B and 4 KiB: latency (window 1) and rate
  (window 16), with the receiver waiting on the signal (ops.signal_wait) -- against RDMA WRITE_WITH_IMM + a receive
  consumer (ops.recv_consume) on the same kind of QP and the same engine size.

The card's name and power limit are read in the same run and recorded beside the numbers.  Needs a GPU.
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


def fa_rates(ctx, ctas):
    nq, it1, itn = 32, 20000, 2000
    target = torch.zeros(nq, dtype=torch.int64, device="cuda:0")
    fetch = torch.zeros(max(it1, nq * itn), dtype=torch.int64, device="cuda:0")
    mt, mf = ctx.reg_mr(target), ctx.reg_mr(fetch)
    qps = [ctx.loopback_qp(depth=64) for _ in range(nq)]
    torch.cuda.synchronize()
    out = {}
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        ops.atomic_stream(qps[0], "fa", mt, mf, 256, window=16, burst=8)                  # warm-up
        r = ops.atomic_stream(qps[0], "fa", mt, mf, it1, window=16, burst=8, timeout_ms=10000)
        out["fa_1qp_w16_b8_us_per_atomic"] = round(r.us_per_msg, 4) if r.ok else None
        for name, stride in (("fa_32qp_shared_word", 0), ("fa_32qp_distinct_words", 8)):
            r = ops.atomic_stream(qps, "fa", mt, mf, itn, target_stride=stride, window=16, burst=8, timeout_ms=10000)
            total = sum(r.done)
            out[name] = {"ok": r.ok, "us_per_atomic_aggregate": round(r.device_ns / 1e3 / max(total, 1), 4),
                         "us_per_atomic_per_qp": round(r.us_per_msg, 4), "matomics_per_s": round(total / max(r.device_ns, 1) * 1e3, 3)}
    finally:
        ctx.engine_stop()
    return out


def signalling(ctx, ctas, nbytes):
    n_lat, n_rate = 1000, 4000
    src = torch.empty(nbytes * n_rate, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros_like(src)
    ops.fill_random(src, seed=5)
    sig = torch.zeros(2, dtype=torch.int64, device="cuda:0")     # one signal word per run: nothing is reset while the engine runs
    fetch = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    ms, md, msig, mf = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(sig), ctx.reg_mr(fetch)
    qp_sig = ctx.loopback_qp(depth=256)
    qp_imm = ctx.loopback_qp(depth=8192)
    torch.cuda.synchronize()
    res = {}
    ctx.engine_start(ctas=ctas, idle_timeout_ms=5000)
    try:
        for k, (label, n, window) in enumerate((("latency", n_lat, 1), ("rate", n_rate, 16))):
            # put-with-signal, receiver waiting on the signal word
            view, wst = ops.signal_wait(ctx, (sig.data_ptr() + 8 * k, 8), n, timeout_ms=5000, stream=ctx.aux_stream, sync=False)
            r = ops.put_signal(qp_sig, ms, md, nbytes, msig, sig_off=8 * k, fetch_mr=mf, iters=n, window=window, slot_stride=nbytes,
                               nslots=n, timeout_ms=10000)
            wst.synchronize()
            w = ops.parse_signal_wait(view)
            ps = {"ok": r.ok and w["status"] == "OK" and w["seen"] == n, "sender_us_per_msg": round(r.us_per_msg, 4),
                  "receiver_us_per_msg": round((w["t_end_ns"] - r.t_start_ns[0]) / 1e3 / n, 4)}
            # WRITE_WITH_IMM + receive consumer (pre-posts its own n receive WQEs) on the same engine
            view, rst = ops.recv_consume(qp_imm, n, timeout_ms=5000, stream=ctx.aux_stream, sync=False, prepost_mr=md,
                                         prepost_bytes=0)
            r2 = ops.rdma_stream(qp_imm, W.OP_RDMA_WRITE_IMM, ms, md, nbytes, iters=n, window=window, slot_stride=nbytes,
                                 nslots=n, timeout_ms=10000)
            rst.synchronize()
            c = ops.parse_recv(view)
            wi = {"ok": r2.ok and c["status"] == "OK" and c["seen"] == n, "sender_us_per_msg": round(r2.us_per_msg, 4),
                  "receiver_us_per_msg": round((c["t_end_ns"] - r2.t_start_ns[0]) / 1e3 / n, 4)}
            res[label] = {"window": window, "messages": n, "put_signal": ps, "write_imm_recv": wi}
    finally:
        ctx.engine_stop()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("atomic_bench needs a GPU")
    rec = {"bench": "atomics", "engine_ctas": a.ctas, **gpu_info()}
    ctx = rn.Context(0)
    try:
        rec.update(fa_rates(ctx, a.ctas))
        rec["put_signal_vs_write_imm"] = {f"{nb}B": signalling(ctx, a.ctas, nb) for nb in (64, 4096)}
    finally:
        ctx.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
