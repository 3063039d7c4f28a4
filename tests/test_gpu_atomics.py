"""GPU tier: 8-byte RDMA atomics through the software HCA (and the mock ConnectX) on an H100 -- host- and device-posted
fetch-and-add / compare-and-swap, exactly-once under contention, in-order execution, put-with-signal ordering against
multi-chunk writes, the error paths, and a signal landing on a peer GPU."""
import pytest
import torch

import rocnrdma_b200 as rn
from rocnrdma_b200 import ops, wire as W

pytestmark = pytest.mark.gpu
H = W.MEM_HOST_PINNED


def _words(vals, dev="cuda:0"):
    return torch.tensor(vals, dtype=torch.int64, device=dev)


def test_host_posted_fetch_add_and_cmp_swap_on_device_memory(ctx):
    target, fetch = _words([40, 7]), _words([0, 0, 0, 0])
    mt, mf = ctx.reg_mr(target), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        qp.post_fetch_add(mf, mt, 2)
        qp.post_cmp_swap(mf, mt, compare=7, swap=99, local_off=8, remote_off=8)
        qp.post_cmp_swap(mf, mt, compare=7, swap=5, local_off=16, remote_off=8)      # no longer 7: left alone
        wcs = qp.scq.wait(3)
    finally:
        ctx.engine_stop()
    assert [w.status for w in wcs] == ["OK"] * 3 and all(w.byte_cnt == 8 for w in wcs)
    assert [w.wqe_opcode for w in wcs] == [W.OP_ATOMIC_FA, W.OP_ATOMIC_CS, W.OP_ATOMIC_CS]
    assert fetch.tolist() == [40, 7, 99, 0]
    assert target.tolist() == [42, 99]


def test_device_posted_fetch_add_contention_is_exactly_once(ctx):
    nq, iters = 32, 1024
    target, fetch = _words([0]), torch.full((nq * iters,), -1, dtype=torch.int64, device="cuda:0")
    mt, mf = ctx.reg_mr(target), ctx.reg_mr(fetch)
    qps = [ctx.loopback_qp(depth=64) for _ in range(nq)]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.atomic_stream(qps, "fa", mt, mf, iters, add=1, window=16, burst=8, timeout_ms=5000)
    finally:
        ctx.engine_stop()
    assert r.ok and r.done == [iters] * nq, r.status
    assert int(target.item()) == nq * iters
    assert torch.equal(torch.sort(fetch).values, torch.arange(nq * iters, device="cuda:0"))
    # one QP's fetched values grow: its atomics executed in its posting order
    per_qp = fetch.view(nq, iters)
    assert bool((per_qp[:, 1:] > per_qp[:, :-1]).all())


def test_chained_cmp_swap_executes_in_order(ctx):
    n = 2048
    target, fetch = _words([0]), torch.full((n,), -1, dtype=torch.int64, device="cuda:0")
    mt, mf = ctx.reg_mr(target), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=64)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=16, idle_timeout_ms=3000)
    try:
        r = ops.atomic_stream(qp, "cs", mt, mf, n, chain=True, window=16, burst=8, timeout_ms=5000)
    finally:
        ctx.engine_stop()
    assert r.ok and r.done == [n], r.status
    assert torch.equal(fetch, torch.arange(n, device="cuda:0")), "a CS found the word at a value other than its compare"
    assert int(target.item()) == n


def test_put_with_signal_never_signals_before_the_data(ctx):
    """64 slots of 4 MiB, each written once and followed by FA(+1) on the signal word; the receiver compares slot k
    with its source the moment the signal reaches k + 1.  An atomic executed when it is claimed (instead of at
    retirement, behind the multi-chunk WRITE before it) shows up here as mismatching words."""
    nslots, slot = 64, 4 << 20
    src = torch.empty(nslots * slot, dtype=torch.uint8, device="cuda:0")
    dst = torch.zeros(nslots * slot, dtype=torch.uint8, device="cuda:0")
    sig, fetch = _words([0]), _words([0] * nslots)
    ops.fill_random(src, seed=4242)
    ms, md, msig, mf = ctx.reg_mr(src), ctx.reg_mr(dst), ctx.reg_mr(sig), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=256)
    stamps = torch.zeros(nslots, dtype=torch.int64, device="cuda:0")
    torch.cuda.synchronize()
    ctx.engine_start(ctas=32, idle_timeout_ms=3000)
    try:
        wview, wst = ops.signal_wait(ctx, sig, nslots, stamps=stamps, timeout_ms=4000, stream=ctx.aux_stream, sync=False,
                                     check=(dst, src, slot, slot))
        r = ops.put_signal(qp, ms, md, slot, msig, fetch_mr=mf, iters=nslots, slot_stride=slot, nslots=nslots, timeout_ms=5000)
        wst.synchronize()
        w = ops.parse_signal_wait(wview)
    finally:
        ctx.engine_stop()
    assert r.ok and r.done == [nslots], r.status
    assert w["status"] == "OK" and w["seen"] == nslots, w
    assert w["mismatches"] == 0, f"{w['mismatches']} 16-byte words read before their WRITE landed"
    assert int(sig.item()) == nslots and fetch.tolist() == list(range(nslots))
    assert ops.compare(src, dst) == 0
    assert bool((stamps[1:] >= stamps[:-1]).all()) and int(stamps[0]) > 0


@pytest.mark.parametrize("case", ["no_remote_atomic", "misaligned", "length", "revoked"])
def test_atomic_error_paths_flush_and_fail_the_qp(ctx, case):
    target, fetch = _words([5, 0]), _words([0, 0])
    access = W.ACC_ALL & ~W.ACC_REMOTE_ATOMIC if case == "no_remote_atomic" else W.ACC_ALL
    mt, mf = ctx.reg_mr(target, access=access), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=16, mem=H)
    want = {"no_remote_atomic": "REMOTE_ACCESS_ERR", "misaligned": "REMOTE_INVAL_REQ_ERR", "length": "LOCAL_LENGTH_ERR",
            "revoked": "REMOTE_ACCESS_ERR"}[case]
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        if case == "revoked":
            mt.revoke()
        if case == "length":
            qp.post_raw(W.OP_ATOMIC_FA, mf.addr, mf.lkey, mt.addr, mt.rkey, nbytes=4)
        else:
            qp.post_fetch_add(mf, mt, 1, remote_off=4 if case == "misaligned" else 0)
        qp.post_fetch_add(mf, mt, 1, local_off=8)
        wcs = qp.scq.wait(2)
    finally:
        ctx.engine_stop()
    assert wcs[0].is_error and wcs[0].status == want, wcs[0]
    assert wcs[1].is_error and wcs[1].status == "WR_FLUSH_ERR"
    assert qp.state == "ERR"
    assert target.tolist() == [5, 0] and fetch.tolist() == [0, 0]


def test_atomic_on_pinned_host_memory(ctx):
    """Executed where the device reports native host atomics, REMOTE_OP_ERR (and a failed QP) where it does not."""
    target = torch.tensor([10], dtype=torch.int64).pin_memory()
    fetch = _words([0])
    mt, mf = ctx.reg_mr(target), ctx.reg_mr(fetch)
    qp = ctx.loopback_qp(depth=16, mem=H)
    torch.cuda.synchronize()
    ctx.engine_start(ctas=4, idle_timeout_ms=3000)
    try:
        qp.post_fetch_add(mf, mt, 3)
        qp.post_fetch_add(mf, mt, 3)
        wcs = qp.scq.wait(2)
    finally:
        ctx.engine_stop()
    if ctx.host_native_atomics:
        assert [w.status for w in wcs] == ["OK", "OK"]
        assert int(target[0]) == 16 and int(fetch.item()) == 13
    else:
        assert wcs[0].status == "REMOTE_OP_ERR" and wcs[1].status == "WR_FLUSH_ERR" and qp.state == "ERR"
        assert int(target[0]) == 10


def test_device_posted_fetch_add_into_mock_connectx_queues():
    vctx = rn.Context(device=0, wire="verbs", nic=0)
    try:
        assert vctx.nic_is_mock
        n = 64
        target, fetch = _words([100]), torch.full((n,), -1, dtype=torch.int64, device="cuda:0")
        torch.cuda.synchronize()
        mt, mf = vctx.reg_mr(target), vctx.reg_mr(fetch)
        qp = vctx.loopback_qp(depth=16)
        assert qp.on_gpu
        r = ops.atomic_stream(qp, "fa", mt, mf, n, add=2, window=8, burst=4, timeout_ms=5000)
        assert r.ok and r.done == [n], r.status
        assert int(target.item()) == 100 + 2 * n
        assert torch.equal(fetch, 100 + 2 * torch.arange(n, device="cuda:0"))
        c = qp.counters()
        assert c["n_err"] == 0 and c["n_wqe"] == n and c["n_db_order_violations"] == 0, c
    finally:
        vctx.close()


@pytest.mark.multigpu
def test_fetch_add_onto_peer_gpu_with_signal_wait_there():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    n = 512
    ctx0, ctx1 = rn.Context(0), rn.Context(1)
    try:
        target = _words([0], dev="cuda:1")
        fetch = torch.full((n,), -1, dtype=torch.int64, device="cuda:0")
        mt, mf = ctx0.reg_mr(target), ctx0.reg_mr(fetch)          # peer HBM: registration maps it over NVLink
        qp = ctx0.loopback_qp(depth=64)
        qp.set_flags(sys_scope=True)
        torch.cuda.synchronize(0); torch.cuda.synchronize(1)
        ctx0.engine_start(ctas=16, idle_timeout_ms=3000)
        try:
            wview, wst = ops.signal_wait(ctx1, target, n, timeout_ms=4000, sync=False)
            r = ops.atomic_stream(qp, "fa", mt, mf, n, window=16, burst=8, timeout_ms=5000)
            wst.synchronize()
            w = ops.parse_signal_wait(wview)
        finally:
            ctx0.engine_stop()
        assert r.ok and r.done == [n], r.status
        assert w["status"] == "OK" and w["seen"] == n, w
        assert int(target.item()) == n
        assert torch.equal(fetch, torch.arange(n, device="cuda:0"))
    finally:
        ctx0.close()
        ctx1.close()
