"""Inline puts against gather WRITEs on the software HCA, one JSON record on stdout.

    python tools/inline_bench.py [--ctas 32] [--reps 3] [--out FILE]

On one device-posted QP, engine on --ctas CTAs, alternated --reps times:
* 8-byte inline puts (ops.put_inline, payload read from an unregistered tensor into the WQE) against 8-byte RDMA WRITEs
  from a registered buffer (ops.rdma_stream): window 1 (latency) and window 16 with bursts of 8 (rate);
* inline put with a signal (ops.put_inline with sig_mr) against put-with-signal (ops.put_signal), 8 bytes, window 1 and
  16, each with the receiver waiting on its signal word (ops.signal_wait).

Microseconds per message from the device timers (first post to last completion).  The card's name and power limit are
read in the same run and recorded beside the numbers.  Needs a GPU.
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
    xs = [x for x in xs if x is not None]
    return {"min": round(min(xs), 4), "max": round(max(xs), 4), "runs": [round(x, 4) for x in xs]} if xs else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inline_bench needs a GPU")
    nbytes, n_lat, n_rate = 8, 2000, 20000
    modes = (("latency_w1", n_lat, 1, 1), ("rate_w16_b8", n_rate, 16, 8))
    rec = {"bench": "inline", "engine_ctas": a.ctas, "nbytes": nbytes, **gpu_info()}
    ctx = rn.Context(0)
    try:
        values = torch.randint(0, 256, (n_rate, nbytes), dtype=torch.uint8, device="cuda:0")   # never registered
        src = values.clone().view(-1)
        dst = torch.zeros(n_rate * nbytes, dtype=torch.uint8, device="cuda:0")
        nsig = 2 * len(modes) * (a.reps + 1)
        sig = torch.zeros(nsig, dtype=torch.int64, device="cuda:0")       # a fresh signal word per run: nothing is reset
        fetch = torch.zeros(64, dtype=torch.int64, device="cuda:0")
        ms, md, msig, mf = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(sig), ctx.reg_mr(fetch)
        qp = ctx.loopback_qp(depth=256)
        torch.cuda.synchronize()
        res = {m[0]: {"inline": [], "gather": [], "inline_signal_sender": [], "put_signal_sender": [],
                      "inline_signal_receiver": [], "put_signal_receiver": []} for m in modes}
        ok = True
        word = 0

        def signalled(run, label, n, window):
            nonlocal word, ok
            view, wst = ops.signal_wait(ctx, (sig.data_ptr() + 8 * word, 8), n, timeout_ms=5000, stream=ctx.aux_stream, sync=False)
            r = run(word)
            word += 1
            wst.synchronize()
            w = ops.parse_signal_wait(view)
            ok = ok and r.ok and w["status"] == "OK" and w["seen"] == n
            return r.us_per_msg, (w["t_end_ns"] - r.t_start_ns[0]) / 1e3 / n

        ctx.engine_start(ctas=a.ctas, idle_timeout_ms=5000)
        try:
            ops.put_inline(qp, values, md, nbytes, iters=256, nslots=256, window=16, burst=8)        # warm-up
            ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, nbytes, iters=256, window=16, burst=8, slot_stride=nbytes, nslots=256)
            for rep in range(a.reps + 1):                 # rep 0 is a warm-up of every shape
                for label, n, window, burst in modes:
                    r1 = ops.put_inline(qp, values, md, nbytes, iters=n, nslots=n, window=window, burst=burst, timeout_ms=10000)
                    r2 = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, nbytes, iters=n, window=window, burst=burst,
                                         slot_stride=nbytes, nslots=n, timeout_ms=10000)
                    ok = ok and r1.ok and r2.ok
                    s1 = signalled(lambda k: ops.put_inline(qp, values, md, nbytes, iters=n, nslots=n, sig_mr=msig, sig_off=8 * k,
                                                            fetch_mr=mf, window=window, timeout_ms=10000), label, n, window)
                    s2 = signalled(lambda k: ops.put_signal(qp, ms, md, nbytes, msig, sig_off=8 * k, fetch_mr=mf, iters=n,
                                                            window=window, slot_stride=nbytes, nslots=n, timeout_ms=10000),
                                   label, n, window)
                    if rep == 0:
                        continue
                    d = res[label]
                    d["inline"].append(r1.us_per_msg)
                    d["gather"].append(r2.us_per_msg)
                    d["inline_signal_sender"].append(s1[0]); d["inline_signal_receiver"].append(s1[1])
                    d["put_signal_sender"].append(s2[0]); d["put_signal_receiver"].append(s2[1])
        finally:
            ctx.engine_stop()
        st = ctx.engine_stats()
        rec["ok"] = ok and st["fatal"] == 0
        rec["us_per_msg"] = {label: {k: _spread(v) for k, v in d.items()} for label, d in res.items()}
    finally:
        ctx.close()
    line = json.dumps(rec)
    print(line)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
