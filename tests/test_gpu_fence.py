"""The fence flag on one H100: a fenced work request moves no byte before every earlier one of its QP has finished.

Directed programs run every dependent pair (WRITE then fenced READ of the same bytes, WRITE then fenced WRITE over part
of them, READ then fenced WRITE / SEND of what it fetched, WRITE then fenced atomic on the written word) at 16 KiB, 4 MiB
and 64 MiB on 1, 3 and 32 engine CTAs, with queues and data in device or pinned host memory, pre-posted before a one-shot
engine (batch claims) or posted while it runs (single claims), and are checked byte for byte against the RC model
(tests/rc_model.py, with the fenced WRs of tests/rc_fence_model.py).  Device posters set the flag too:
``ops.rdma_stream(fence_every=...)`` and a kernel calling ``dev::rdma_write`` then ``dev::rdma_read(..., fence=true)``.  Random fenced programs run on the software HCA configs of
test_gpu_rc_model.py and on the mock ConnectX with data in HBM.  The per-QP count of fenced WQEs that found their gate
closed (``n_fence_waits``) is summed over the run, so the tests provably made the engine hold work back."""
import numpy as np
import pytest
import torch

import rc_fence_model as F
import rc_model as M
from rc_fence_model import FWR as WR
from rc_model import MR, Buf, Program, QpProg, Recv
from rocnrdma_b200 import ops, wire as W
from test_gpu_rc_model import CONFIGS

pytestmark = pytest.mark.gpu

K, MiB = 1 << 10, 1 << 20
GATE_WAITS = []          # n_fence_waits of every softhca run in this module


class _CountingWire(M.SoftHcaWire):
    def finish(self, prog):
        out = super().finish(prog)
        GATE_WAITS.append(sum(c["n_fence_waits"] for c in out["counters"]))
        return out


def _pairs_program(n, ctas, chunk, data_mem, bad_first=False):
    """Every dependent pair on one loopback QP, n bytes each; the overlapping WRITE pair and the SEND pair are misaligned
    (generic copy), the others aligned (TMA when n >= 4 KiB).  bad_first: the program starts with a WRITE whose rkey is
    wrong, so everything behind it, fenced or not, is flushed."""
    g = 64
    rng = np.random.default_rng(n + ctas)
    src = rng.integers(0, 256, 2 * n + 4 * K, dtype=np.uint8)
    # DST layout: [r0 | back0 | r1 (mis 1) | m2 | o2 | m3 (mis 8) | recv3], each followed by a gap
    offs, top = [], 64
    for mis in (0, 0, 1, 0, 0, 8, 0):
        start = (top + 15) // 16 * 16 + mis
        offs.append(start)
        top = start + n + g
    bufs = {"SRC": Buf("SRC", src, data_mem), "DST": Buf("DST", rng.integers(0, 256, top + 64, dtype=np.uint8), data_mem),
            "ATOM": Buf("ATOM", np.zeros(64, np.uint8), "dev"), "FETCH": Buf("FETCH", np.full(64, 0xEE, np.uint8), data_mem)}
    mrs = {"src": MR("src", "SRC", 0, src.size, M.ACC_ALL, "local"), "srcr": MR("srcr", "SRC", 0, src.size, M.ACC_ALL, "remote"),
           "dst": MR("dst", "DST", 0, top + 64, M.ACC_ALL, "remote"), "dstl": MR("dstl", "DST", 0, top + 64, M.ACC_ALL, "local"),
           "atom": MR("atom", "ATOM", 0, 64, M.ACC_ALL, "remote"), "fetch": MR("fetch", "FETCH", 0, 64, M.ACC_ALL, "local")}
    r0, back0, r1, m2, o2, m3, rv3 = offs
    wrs = [WR("WRITE", n, "src", 0, "dst", r0, signaled=False), WR("READ", n, "dstl", back0, "dst", r0, fence=True),
           WR("WRITE", n, "src", 16, "dst", r1, signaled=False),
           WR("WRITE", n // 2, "src", n + 32, "dst", r1 + n // 4, fence=True),
           WR("READ", n, "dstl", m2, "srcr", n, signaled=False), WR("WRITE", n, "dstl", m2, "dst", o2, fence=True),
           WR("READ", n, "dstl", m3, "srcr", 8, signaled=False), WR("SEND", n, "dstl", m3, fence=True),
           WR("WRITE", 8, "src", 64, "atom", 0, signaled=False), WR("FA", 8, "fetch", 0, "atom", 0, add=5, fence=True)]
    if bad_first:
        wrs.insert(0, WR("WRITE", n, "src", 0, "dst", r0, bad_rkey=True, fault="bad_rkey"))
    prog = Program(n, {"wire": "softhca", "ctas": ctas, "chunk_bytes": chunk}, bufs, mrs,
                   [QpProg(0, wrs, [Recv("dst", rv3, n)])])
    M.run_model(prog)
    return prog


DIRECTED = [(n, c) for n in (16 * K, 4 * MiB, 64 * MiB) for c in (1, 3, 32)]


@pytest.mark.parametrize("n,ctas", DIRECTED, ids=[f"{n // K}K-c{c}" for n, c in DIRECTED])
def test_every_dependent_pair(n, ctas):
    i = DIRECTED.index((n, ctas))
    qmem = ("host", "dev")[i % 2]
    oneshot = i % 3 != 1
    dmem = "dev" if n > 4 * MiB else ("host", "dev")[(i // 2) % 2]
    before = len(GATE_WAITS)
    prog = _pairs_program(n, ctas, 64 * K, dmem)
    wire = F.with_fences(_CountingWire(0, ctas, 64 * K, qmem, oneshot))
    try:
        M.run_program(prog, wire, timeout_s=60)
    finally:
        wire.close()
    print(f"{n} B, {ctas} CTAs, queues {qmem}, data {dmem}, {'oneshot' if oneshot else 'live'}: "
          f"{GATE_WAITS[before]} fenced WQEs found their gate closed")
    if oneshot:
        # pre-posted: each fenced WQE is committed in a batch, before its predecessor can have retired
        assert GATE_WAITS[before] >= 1


@pytest.mark.parametrize("oneshot", [True, False])
def test_fenced_wrs_behind_a_fault_are_flushed(oneshot):
    prog = _pairs_program(64 * K, 3, 16 * K, "dev", bad_first=True)
    assert all(c.status != "OK" for c in M.run_model(prog).qps[0].req)
    wire = F.with_fences(_CountingWire(0, 3, 16 * K, "dev", oneshot))
    try:
        M.run_program(prog, wire)
    finally:
        wire.close()


def test_engine_does_not_idle_out_while_a_gated_wqe_waits(ctx):
    """One CTA, a 1 ms idle watchdog: a 512 MiB WRITE keeps the fenced READ behind it waiting far longer than that."""
    n = 512 * MiB
    src = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(n, dtype=torch.uint8, device="cuda:0")
    back = torch.zeros(64 * K, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=7)
    ms, md, mb = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(back)
    cq = ctx.create_cq(64, W.MEM_HOST_PINNED)
    qp = ctx.create_qp(cq, cq, 64, 64, W.MEM_HOST_PINNED, chunk_bytes=n)
    qp.connect()
    torch.cuda.synchronize()
    qp.post_write(ms, md, n, signaled=False)
    qp.post_read(mb, md, 64 * K, remote_off=n - 64 * K, fence=True)
    ctx.engine_start(ctas=1, idle_timeout_ms=1)
    try:
        got = []
        import time
        t0 = time.monotonic()
        while not got and time.monotonic() - t0 < 20:
            got = cq.poll(4)
    finally:
        ctx.engine_stop()
    st = ctx.engine_stats()
    assert st["fatal"] == 0 and st["running_ctas"] == 0, st
    assert len(got) == 1 and not got[0].is_error, got
    assert torch.equal(back, src[n - 64 * K:])
    c = qp.counters()
    assert c["n_fence_waits"] == 1 and c["n_wqe"] == 2
    GATE_WAITS.append(c["n_fence_waits"])


@pytest.mark.parametrize("fence_every", [1, 8])
def test_stream_poster_sets_the_fence(ctx, fence_every):
    nbytes, n = 256 * K, 64
    src = torch.empty(n * nbytes, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(n * nbytes, dtype=torch.uint8, device="cuda:0")
    ops.fill_random(src, seed=fence_every)
    ms, md = ctx.reg_mr(src), ctx.reg_mr(dst)
    qp = ctx.loopback_qp(depth=64, chunk_bytes=64 * K)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=32, idle_timeout_ms=3000)
    try:
        r = ops.rdma_stream(qp, W.OP_RDMA_WRITE, ms, md, nbytes, iters=n, window=16, slot_stride=nbytes, nslots=n,
                            timeout_ms=5000, fence_every=fence_every)
    finally:
        ctx.engine_stop()
    assert r.ok and r.done == [n], r.status
    assert torch.equal(src, dst)
    c = qp.counters()
    print(f"fence_every {fence_every}: {c['n_fence_waits']} of {n // fence_every} fenced WRITEs waited")
    assert c["n_err"] == 0 and c["n_wqe"] == n and c["n_fence_waits"] <= n // fence_every
    GATE_WAITS.append(c["n_fence_waits"])


@pytest.mark.parametrize("mode", ["fenced", "wait", "one_call"])
@pytest.mark.parametrize("nbytes", [16 * K, 4 * MiB])
def test_device_posted_write_then_fenced_read(ctx, mode, nbytes):
    """A kernel posts WRITE src -> dst and then the READ dst -> back; with a fresh source each round, back must equal it."""
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(nbytes, dtype=torch.uint8, device="cuda:0")
    back = torch.zeros(nbytes, dtype=torch.uint8, device="cuda:0")
    ms, md, mb = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(back)
    qp = ctx.loopback_qp(depth=64, chunk_bytes=64 * K)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=32, idle_timeout_ms=3000)
    try:
        for k in range(4):
            ops.fill_random(src, seed=100 + k, stream=ctx.stream)
            ctx.stream.synchronize()
            r = ops.write_read(qp, ms, md, mb, nbytes, iters=1, mode=mode)
            assert r["status"] == "OK" and r["done"] == 1, r
            assert torch.equal(back, src), (mode, k)
    finally:
        ctx.engine_stop()
    c = qp.counters()
    assert c["n_err"] == 0
    GATE_WAITS.append(c["n_fence_waits"])


@pytest.mark.parametrize("ctas,prof,chunk,qmem,dmem,oneshot", CONFIGS,
                         ids=[f"c{c}-{'prof-' if p else ''}k{k // K}-q{q}-d{d}-{'oneshot' if o else 'live'}" for c, p, k, q, d, o in CONFIGS])
def test_random_fenced_programs_on_the_softhca(monkeypatch, ctas, prof, chunk, qmem, dmem, oneshot):
    if prof:
        monkeypatch.setenv("RN_ENGINE_PROFILE", "1")
    else:
        monkeypatch.delenv("RN_ENGINE_PROFILE", raising=False)
    cfg = {"wire": "softhca", "max_wrs": 100, "max_len": 4 << 20, "big_budget": 12 << 20, "ctas": ctas,
           "chunk_bytes": chunk, "data_mem": dmem, "allow_rnr": not oneshot, "fences": True}
    s = M.replay_seed()
    for seed in [s] if s is not None else [70_000 + 100 * CONFIGS.index((ctas, prof, chunk, qmem, dmem, oneshot)) + i
                                           for i in range(M.soak_seeds(2))]:
        F.check_seed(seed, cfg, lambda: _CountingWire(0, ctas, chunk, qmem, oneshot))


def test_random_fenced_programs_on_the_mock_connectx_with_hbm():
    cfg = {"wire": "verbs", "max_wrs": 80, "max_len": 1 << 20, "big_budget": 4 << 20, "allow_rnr": True, "fences": True}
    s = M.replay_seed()
    for seed in [s] if s is not None else [90_000 + i for i in range(M.soak_seeds(4))]:
        F.check_seed(seed, cfg, lambda: M.VerbsWire(device=0))


def test_the_gate_held_work_back():
    """Across this module's softhca runs, fenced WQEs found their gate closed."""
    print(f"gate closed for {sum(GATE_WAITS)} fenced WQEs over {len(GATE_WAITS)} runs")
    assert sum(GATE_WAITS) > 0
