"""Fenced work requests in the RC reference model and on the mock ConnectX on host DRAM.

``cfg["fences"]`` makes the program generator of tests/rc_fence_model.py splice dependent pairs whose later WR is fenced
into rc_model's random programs: a WRITE and a fenced READ of the same bytes, a WRITE and a fenced WRITE over part of
them, a READ and a fenced WRITE or SEND of what it fetched, a WRITE and a fenced atomic on the written word.  With the
option off it must produce exactly the programs rc_model always did (the digests below were taken before the fence
existed), so the model tests keep their coverage."""
import dataclasses
import hashlib

import pytest

import rc_fence_model as F
import rc_model as M
from rc_fence_model import FWR
from rc_model import MR, Buf, Program, QpProg, Recv
from rocnrdma_b200 import api

K = 1 << 10
DIGEST_CFGS = {
    "mock": ({"wire": "verbs", "max_wrs": 60, "max_len": 1 << 18, "big_budget": 1 << 20, "allow_rnr": True},
             "9adc99a96212b278976eab142c3ddc15df427a06b4ce7cdb7bcf2c066b000528"),
    "softhca": ({"wire": "softhca", "max_wrs": 150, "max_len": 4 << 20, "big_budget": 12 << 20, "ctas": 3,
                 "chunk_bytes": 20 * K + 16, "data_mem": "dev", "allow_rnr": True},
                "f3e3c63872000590ece2fea4554285258df61d66ebc3b8d4d0ba0ad31609c1b7"),
}


def program_digest(p: Program) -> str:
    """Everything a program is made of; a WR's ``fence`` only counts when it is set."""
    h = hashlib.sha256()
    h.update(repr((p.seed, sorted(p.cfg.items()), p.rnr)).encode())
    for name in sorted(p.bufs):
        b = p.bufs[name]
        h.update(repr((name, b.mem, b.init.dtype.str, b.init.size)).encode())
        h.update(b.init.tobytes())
    for name in sorted(p.mrs):
        h.update(repr(dataclasses.astuple(p.mrs[name])).encode())
    for q in p.qps:
        h.update(repr(q.peer).encode())
        for w in q.wrs:
            d = dataclasses.asdict(w)
            if not d.get("fence", False):
                d.pop("fence", None)
            h.update(repr(sorted(d.items())).encode())
        for r in q.recvs:
            h.update(repr(dataclasses.astuple(r)).encode())
    return h.hexdigest()


@pytest.mark.parametrize("name", sorted(DIGEST_CFGS))
def test_generator_without_fences_is_unchanged(name):
    cfg, want = DIGEST_CFGS[name]
    h = hashlib.sha256()
    for seed in range(12):
        h.update(program_digest(F.generate(seed, cfg)).encode())
    assert h.hexdigest() == want


FENCE_CFG = {"wire": "verbs", "max_wrs": 60, "max_len": 1 << 18, "big_budget": 1 << 20, "allow_rnr": True, "fences": True,
             "ctas": 3, "chunk_bytes": 20 * K + 16}


def _overlaps(a, b):
    return a[0] == b[0] and a[1] < b[2] and b[1] < a[2]


def _footprints(prog, qi, w):
    """(reads, writes) of one WR as (buffer, start, end) spans, from its MRs."""
    def span(mr_name, off, n):
        m = prog.mrs[mr_name]
        return (m.buf, m.off + off, m.off + off + n)
    reads, writes = [], []
    if w.op in ("WRITE", "WRITE_IMM") and w.inline is None and w.n:
        reads.append(span(w.lmr, w.loff, w.n)); writes.append(span(w.rmr, w.roff, w.n))
    elif w.op == "READ" and w.n:
        reads.append(span(w.rmr, w.roff, w.n)); writes.append(span(w.lmr, w.loff, w.n))
    elif w.op in ("SEND", "SEND_IMM") and w.inline is None and w.n:
        reads.append(span(w.lmr, w.loff, w.n))
    elif w.op in ("FA", "CS"):
        writes.append(span(w.lmr, w.loff, 8))
    return reads, writes


def test_fenced_programs_only_overlap_across_a_fence():
    """Every generated dependency (a later WR touching bytes an earlier one wrote, or writing bytes it read) has the
    fence on the later WR; the atomic words, ordered by retirement, are the only exception.  And the generator reaches
    every pair kind on both wire configs."""
    kinds = set()
    for wire in ("verbs", "softhca"):
        for seed in range(60):
            p = F.generate(seed, dict(FENCE_CFG, wire=wire))
            for qi, q in enumerate(p.qps):
                fp = [_footprints(p, qi, w) for w in q.wrs]
                for j, wj in enumerate(q.wrs):
                    rj, wrj = fp[j]
                    for i in range(j):
                        ri, wri = fp[i]
                        dep = any(_overlaps(a, b) for a in wri for b in rj + wrj) or any(_overlaps(a, b) for a in ri for b in wrj)
                        if dep and not F.fenced(wj):
                            raise AssertionError(f"seed {seed} qp {qi}: wr {j} depends on wr {i} without a fence")
                    if F.fenced(wj) and j:
                        prev = q.wrs[j - 1]
                        kinds.add((prev.op, wj.op))
    want = {("WRITE", "READ"), ("WRITE", "WRITE"), ("READ", "WRITE"), ("READ", "SEND")}
    assert want <= kinds and kinds & {("WRITE", "FA"), ("WRITE", "CS")}, kinds


def _prog(wrs, recvs=()):
    bufs = {"SRC": Buf("SRC", (M.np.arange(256) % 251 + 1).astype(M.np.uint8)), "DST": Buf("DST", M.np.zeros(256, M.np.uint8)),
            "ATOM": Buf("ATOM", M.np.zeros(16, M.np.uint8)), "FETCH": Buf("FETCH", M.np.full(64, 0xEE, M.np.uint8))}
    mrs = {"src": MR("src", "SRC", 0, 256, M.ACC_ALL, "local"), "dst": MR("dst", "DST", 0, 256, M.ACC_ALL, "remote"),
           "dstl": MR("dstl", "DST", 0, 256, M.ACC_ALL, "local"), "atom": MR("atom", "ATOM", 0, 16, M.ACC_ALL, "remote"),
           "fetch": MR("fetch", "FETCH", 0, 64, M.ACC_ALL, "local")}
    return Program(0, {"wire": "verbs", "ctas": 1, "chunk_bytes": 1 << 16}, bufs, mrs, [QpProg(0, list(wrs), list(recvs))])


def test_model_executes_a_fenced_read_after_the_write():
    o = M.run_model(_prog([FWR("WRITE", 32, "src", 0, "dst", 0), FWR("READ", 32, "dstl", 64, "dst", 0, fence=True)]))
    assert o.mem["DST"][64:96].tolist() == list(range(1, 33))


def test_fence_flag_words():
    assert api._ctrl_flags(True, True) == 0x88 and api._ctrl_flags(False, True) == 0x80 and api._ctrl_flags(True, False) == 0x08
    assert api._verbs_flags(True, False) == 1 and api._verbs_flags(False, True) == 2 and api._verbs_flags(True, True) == 3


@pytest.fixture(scope="module")
def verbs_lib():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    if lib.rn_verbs_available() < 2 or lib.rn_verbs_is_mock() != 1:
        pytest.fail("the mock rdma-core provider did not load: " + lib.rn_verbs_why().decode(errors="replace"))
    return lib


def test_mock_connectx_runs_directed_fenced_pairs(verbs_lib):
    """Each dependent pair once, by hand, through the verbs wire's fence flag."""
    p = _prog([FWR("WRITE", 40, "src", 0, "dst", 0, signaled=False), FWR("READ", 40, "dstl", 64, "dst", 0, fence=True),
               FWR("WRITE", 24, "src", 100, "dst", 8, fence=True),
               FWR("READ", 16, "dstl", 128, "src", 200, signaled=False), FWR("WRITE", 16, "dstl", 128, "dst", 160, fence=True),
               FWR("SEND", 16, "dstl", 128, fence=True),
               FWR("WRITE", 8, "src", 48, "atom", 0, signaled=False), FWR("FA", 8, "fetch", 0, "atom", 0, add=3, fence=True)],
              recvs=[Recv("dst", 192, 16)])
    wire = F.with_fences(M.VerbsWire(device=None))
    try:
        M.run_program(p, wire)
    finally:
        wire.close()


def test_mock_connectx_matches_the_model_on_fenced_programs(verbs_lib):
    for seed in (M.replay_seed(),) if M.replay_seed() is not None else range(M.soak_seeds(40)):
        F.check_seed(seed, FENCE_CFG, lambda: M.VerbsWire(device=None))
