"""Scatter-gather work requests in the RC reference model and on the mock ConnectX on host DRAM.

Hand-worked programs check the model itself on every opcode that takes a list, an error in entry 1's key, a flushed
gather, a gather SEND longer than its receive, a gather SEND whose entry 1 fails (it takes no receive), a dropped
zero-length entry whose key is never looked at, and a hand-built two-segment WQE whose zero-length segment is.  The same
programs then run on the mock ConnectX.  ``cfg["sgl"]`` makes the generator of tests/rc_sgl_model.py splice list WRs
into rc_model's random programs, which run on two mock NICs against the model; with the option off it must produce
exactly the programs rc_model always did (the digests of tests/test_rc_fence.py, taken before either option existed)."""
import hashlib

import numpy as np
import pytest

import rc_model as M
import rc_sgl_model as S
from rc_model import MR, Buf, Program, QpProg, Recv
from rc_sgl_model import GWR
from test_rc_fence import DIGEST_CFGS, program_digest

K = 1 << 10


@pytest.mark.parametrize("name", sorted(DIGEST_CFGS))
def test_generator_without_sgl_is_unchanged(name):
    cfg, want = DIGEST_CFGS[name]
    h = hashlib.sha256()
    for seed in range(12):
        h.update(program_digest(S.generate(seed, cfg)).encode())
    assert h.hexdigest() == want


def _prog(wrs, recvs=(), cfg=None):
    src = (np.arange(8192) % 251 + 1).astype(np.uint8)
    bufs = {"q0.SRC": Buf("q0.SRC", src), "q0.DST": Buf("q0.DST", np.zeros(8192, np.uint8))}
    mrs = {"src": MR("src", "q0.SRC", 0, 8192, M.ACC_ALL, "local"), "srcr": MR("srcr", "q0.SRC", 0, 8192, M.ACC_ALL, "remote"),
           "dst": MR("dst", "q0.DST", 0, 4096, M.ACC_ALL, "remote"), "dstl": MR("dstl", "q0.DST", 4096, 4096, M.ACC_ALL, "local"),
           "ro": MR("ro", "q0.DST", 6144, 1024, M.NO_LOCAL_WRITE, "local")}
    return Program(0, dict({"wire": "verbs", "ctas": 1, "chunk_bytes": 1 << 16}, **(cfg or {})), bufs, mrs,
                   [QpProg(0, list(wrs), list(recvs))])


def G(op, n0, n1, lmr="src", loff=0, lmr1="src", loff1=0, rmr=None, roff=0, **kw):
    return GWR(op, n0 + n1, lmr, loff, rmr, roff, sgl=True, lmr1=lmr1, loff1=loff1, n1=n1, **kw)


SRC = (np.arange(8192) % 251 + 1).astype(np.uint8)


def test_model_every_opcode():
    p = _prog([G("WRITE", 10, 20, loff=100, loff1=500, rmr="dst", roff=7),
               G("WRITE_IMM", 5, 3, loff=1, loff1=2, rmr="dst", roff=100, imm=9),
               G("READ", 30, 40, lmr="dstl", loff=0, lmr1="dstl", loff1=200, rmr="srcr", roff=1000),
               G("SEND", 6, 4, loff=50, loff1=60), G("SEND_IMM", 1, 2, loff=70, loff1=80, imm=5)],
              [Recv("dst", 0, 8), Recv("dst", 200, 16), Recv("dst", 300, 3)])
    o = S.run_model(p)
    d = o.mem["q0.DST"]
    assert d[7:17].tolist() == SRC[100:110].tolist() and d[17:37].tolist() == SRC[500:520].tolist()
    assert d[100:105].tolist() == SRC[1:6].tolist() and d[105:108].tolist() == SRC[2:5].tolist()
    assert d[4096:4126].tolist() == SRC[1000:1030].tolist() and d[4296:4336].tolist() == SRC[1030:1070].tolist()
    assert d[200:210].tolist() == SRC[50:56].tolist() + SRC[60:64].tolist() and d[300:303].tolist() == [SRC[70]] + SRC[80:82].tolist()
    q = o.qps[0]
    assert [(c.status, c.byte_cnt) for c in q.req] == [("OK", 30), ("OK", 8), ("OK", 70), ("OK", 10), ("OK", 3)]
    assert [(c.recv, c.kind, c.byte_cnt) for c in q.resp] == [(0, "WR_IMM", 8), (1, "SEND", 10), (2, "SEND_IMM", 3)]


def test_model_entry_one_errors_and_flush():
    p = _prog([G("WRITE", 8, 8, rmr="dst", signaled=False), G("WRITE", 8, 8, rmr="dst", roff=64, bad_lkey1=True),
               G("WRITE", 8, 8, rmr="dst", roff=128)])
    q = S.run_model(p).qps[0]
    assert [c.status for c in q.req] == ["LOCAL_PROT_ERR", "WR_FLUSH_ERR"] and q.state == "ERR"
    d = S.run_model(p).mem["q0.DST"]
    assert d[:16].any() and not d[64:144].any()                  # the failing and the flushed gather wrote nothing
    q = S.run_model(_prog([G("READ", 8, 8, lmr="dstl", lmr1="ro", rmr="srcr")])).qps[0]
    assert [c.status for c in q.req] == ["LOCAL_ACCESS_ERR"]


def test_model_gather_send_checks():
    # longer than its receive: fails on the total, the receive is consumed in error
    q = S.run_model(_prog([G("SEND", 10, 10)], [Recv("dst", 0, 19)])).qps[0]
    assert [c.status for c in q.req] == ["REMOTE_INVAL_REQ_ERR"] and [(c.recv, c.status) for c in q.resp] == [(0, "REMOTE_INVAL_REQ_ERR")]
    # entry 1's key fails at the requester: no receive is taken
    q = S.run_model(_prog([G("SEND", 10, 10, bad_lkey1=True)], [Recv("dst", 0, 64)])).qps[0]
    assert [c.status for c in q.req] == ["LOCAL_PROT_ERR"] and q.resp == []


def test_model_zero_length_segments():
    # dropped by the poster: its bad key is never looked at
    q = S.run_model(_prog([G("WRITE", 16, 0, rmr="dst", bad_lkey1=True)])).qps[0]
    assert [c.status for c in q.req] == ["OK"]
    # kept in a hand-built WQE: checked over an empty range
    q = S.run_model(_prog([G("WRITE", 0, 16, rmr="dst", raw=True, bad_lkey=True)])).qps[0]
    assert [c.status for c in q.req] == ["LOCAL_PROT_ERR"]
    q = S.run_model(_prog([G("WRITE", 0, 16, loff1=3, rmr="dst", roff=5, raw=True)]))
    assert [c.status for c in q.qps[0].req] == ["OK"] and q.mem["q0.DST"][5:21].tolist() == SRC[3:19].tolist()


def test_model_total_past_the_limit_takes_no_receive():
    n = (1 << 29) + 8
    q = S.run_model(_prog([G("SEND", n, n)], [Recv("dst", 0, 64)])).qps[0]
    assert [c.status for c in q.req] == ["LOCAL_LENGTH_ERR"] and q.resp == []


def test_generator_reaches_every_opcode_and_fault():
    ops, faults, raw = set(), set(), 0
    for wire in ("verbs", "softhca"):
        cfg = dict(SGL_CFG, wire=wire, max_msg=M.MAX_MSG)
        for seed in range(40):
            for q in S.generate(seed, cfg).qps:
                for w in q.wrs:
                    if S.is_sgl(w):
                        ops.add(w.op)
                        faults.add(w.fault)
                        raw += w.raw
    assert ops == set(S.SGL_OPS) and set(S.SGL_FAULTS) <= faults and raw > 0, (ops, faults, raw)


@pytest.fixture(scope="module")
def verbs_lib():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    if lib.rn_verbs_available() < 2 or lib.rn_verbs_is_mock() != 1:
        pytest.fail("the mock rdma-core provider did not load: " + lib.rn_verbs_why().decode(errors="replace"))
    return lib


DIRECTED = {
    "every_opcode": ([G("WRITE", 10, 20, loff=100, loff1=500, rmr="dst", roff=7, signaled=False),
                      G("WRITE_IMM", 5, 3, loff=1, loff1=2, rmr="dst", roff=100, imm=9),
                      G("READ", 30, 40, lmr="dstl", loff=0, lmr1="dstl", loff1=200, rmr="srcr", roff=1000),
                      G("SEND", 6, 4, loff=50, loff1=60), G("SEND_IMM", 1, 2, loff=70, loff1=80, imm=5),
                      G("WRITE", 0, 16, loff1=3, rmr="dst", roff=400, raw=True),
                      G("SEND", 0, 12, loff1=9, raw=True),
                      G("WRITE", 16, 0, rmr="dst", roff=500, bad_lkey1=True)],
                     [Recv("dst", 0, 8), Recv("dst", 200, 16), Recv("dst", 300, 3), Recv("dst", 600, 12)]),
    "entry1_key_then_flush": ([G("WRITE", 8, 8, rmr="dst"), G("WRITE", 8, 8, rmr="dst", roff=64, bad_lkey1=True),
                               G("WRITE", 8, 8, rmr="dst", roff=128), G("SEND", 4, 4)], [Recv("dst", 300, 64)]),
    "read_entry1_read_only": ([G("READ", 8, 8, lmr="dstl", lmr1="ro", rmr="srcr")], []),
    "send_too_long": ([G("SEND", 10, 10)], [Recv("dst", 0, 19)]),
    "send_entry1_key": ([G("SEND", 10, 10, bad_lkey1=True)], [Recv("dst", 0, 64)]),
    "raw_zero_segment_key": ([G("WRITE", 0, 16, rmr="dst", raw=True, bad_lkey=True)], []),
    "too_long": ([G("SEND", (1 << 29) + 8, (1 << 29) + 8)], [Recv("dst", 0, 64)]),
}


@pytest.mark.parametrize("name", sorted(DIRECTED))
def test_mock_connectx_runs_directed_programs(verbs_lib, name):
    wrs, recvs = DIRECTED[name]
    p = _prog([GWR(**vars(w)) for w in wrs], recvs, {"max_msg": M.MAX_MSG})
    wire = M.VerbsWire(device=None)
    try:
        S.run_program(p, wire)
    finally:
        wire.close()


SGL_CFG = {"wire": "verbs", "max_wrs": 60, "max_len": 1 << 18, "big_budget": 1 << 20, "allow_rnr": True, "sgl": True,
           "ctas": 3, "chunk_bytes": 20 * K + 16}


def test_mock_connectx_matches_the_model_on_sgl_programs(verbs_lib):
    for seed in (M.replay_seed(),) if M.replay_seed() is not None else range(M.soak_seeds(40)):
        S.check_seed(seed, dict(SGL_CFG, max_msg=M.MAX_MSG), lambda: M.VerbsWire(device=None))
