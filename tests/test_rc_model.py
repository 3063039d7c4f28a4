"""The RC reference model (tests/rc_model.py) on its own, and against the mock ConnectX on host DRAM.

The first half runs hand-written programs whose bytes and completions were worked out by hand, so the model is checked
without any wire.  The second half runs random programs on two mock NICs and compares every byte, every completion and
the final QP state with the model.  ``RN_RC_SEED=<n>`` replays one seed; ``RN_RC_SOAK=<n>`` runs n seeds."""
import numpy as np
import pytest

import rc_model as M
from rc_model import MR, WR, Buf, Program, QpProg, Recv


def _prog(wrs, recvs=(), src=64, dst=64, extra_mrs=(), atom=(), host_atom=False):
    """One loopback QP.  SRC holds bytes 1..src, DST is zeros, ATOM holds the given u64 words, FETCH is 0xEE."""
    bufs = {"SRC": Buf("SRC", (np.arange(src) % 251 + 1).astype(np.uint8)), "DST": Buf("DST", np.zeros(dst, np.uint8)),
            "ATOM": Buf("ATOM", np.array(list(atom) or [0], dtype=np.uint64).view(np.uint8).copy(), "host" if host_atom else "dev"),
            "FETCH": Buf("FETCH", np.full(64, 0xEE, np.uint8))}
    mrs = {"src": MR("src", "SRC", 0, src, M.ACC_ALL, "local"), "dst": MR("dst", "DST", 8, dst - 16, M.ACC_ALL, "remote"),
           "atom": MR("atom", "ATOM", 0, bufs["ATOM"].init.size, M.ACC_ALL, "remote"),
           "fetch": MR("fetch", "FETCH", 0, 64, M.ACC_ALL, "local")}
    for m in extra_mrs:
        mrs[m.name] = m
    return Program(0, {"ctas": 1, "chunk_bytes": 1 << 16}, bufs, mrs, [QpProg(0, list(wrs), list(recvs))])


def _req(o):
    return [(c.wr, c.status) + ((c.byte_cnt,) if c.status == "OK" else ()) for c in o.qps[0].req]


def _resp(o):
    return [(c.recv, c.status) + ((c.kind, c.byte_cnt, c.imm) if c.status == "OK" else ()) for c in o.qps[0].resp]


def test_flush_after_a_mid_program_fault():
    p = _prog([WR("WRITE", 4, "src", 0, "dst", 0), WR("WRITE", 4, "src", 4, "dst", 8, bad_rkey=True),
               WR("WRITE", 4, "src", 8, "dst", 16), WR("READ", 4, "dst", 24, "src", 0)])
    o = M.run_model(p)
    assert _req(o) == [(0, "OK", 4), (1, "REMOTE_ACCESS_ERR"), (2, "WR_FLUSH_ERR"), (3, "WR_FLUSH_ERR")]
    want = np.zeros(64, np.uint8)
    want[8:12] = [1, 2, 3, 4]
    assert (o.mem["DST"] == want).all()
    q = o.qps[0]
    assert (q.state, q.n_wqe, q.n_err) == ("ERR", 4, 3)


def test_unsignaled_wrs_around_an_error():
    """An unsignaled success gives no CQE; an unsignaled error and the unsignaled flushes behind it each give one."""
    p = _prog([WR("WRITE", 2, "src", 0, "dst", 0, signaled=False), WR("WRITE", 2, "src", 0, "dst", 4, signaled=False, bad_lkey=True),
               WR("WRITE", 2, "src", 0, "dst", 8, signaled=False), WR("NOP")])
    o = M.run_model(p)
    assert _req(o) == [(1, "LOCAL_PROT_ERR"), (2, "WR_FLUSH_ERR"), (3, "WR_FLUSH_ERR")]
    assert o.mem["DST"][8:10].tolist() == [1, 2] and not o.mem["DST"][12:].any()


def test_atomic_sees_an_earlier_write_to_its_word():
    p = _prog([WR("WRITE", 8, "src", 0, "atom", 8), WR("FA", 8, "fetch", 0, "atom", 8, add=5),
               WR("CS", 8, "fetch", 8, "atom", 0, add=99, compare=7), WR("CS", 8, "fetch", 16, "atom", 0, add=42, compare=8)],
              atom=[7, 0])
    o = M.run_model(p)
    written = int(np.arange(1, 9, dtype=np.uint8).view(np.uint64)[0])
    assert o.mem["ATOM"].view(np.uint64).tolist() == [99, written + 5]
    assert o.mem["FETCH"][:24].view(np.uint64).tolist() == [written, 7, 99]     # CS hit returns 7, CS miss returns 99
    assert _req(o) == [(0, "OK", 8), (1, "OK", 8), (2, "OK", 8), (3, "OK", 8)]


def test_send_exact_fit_then_one_byte_over():
    p = _prog([WR("SEND", 10, "src", 0), WR("SEND_IMM", 11, "src", 0, imm=5), WR("SEND", 1, "src", 0)],
              recvs=[Recv("dst", 0, 10), Recv("dst", 16, 10), Recv("dst", 32, 10)])
    o = M.run_model(p)
    assert _req(o) == [(0, "OK", 10), (1, "REMOTE_INVAL_REQ_ERR"), (2, "WR_FLUSH_ERR")]
    assert _resp(o) == [(0, "OK", "SEND", 10, 0), (1, "REMOTE_INVAL_REQ_ERR")]       # the third receive is never taken
    assert o.mem["DST"][8:18].tolist() == list(range(1, 11)) and not o.mem["DST"][18:].any()


def test_zero_length_write_imm_checks_no_key_and_still_takes_a_receive():
    p = _prog([WR("WRITE_IMM", 0, "src", -100, "dst", 1 << 40, imm=0xABCD, bad_lkey=True, bad_rkey=True),
               WR("READ", 0, "dst", 1 << 40, "src", -3, bad_lkey=True, bad_rkey=True), WR("WRITE", 0, "src", 0, "dst", 0)],
              recvs=[Recv("dst", 0, 0)])
    o = M.run_model(p)
    assert _req(o) == [(0, "OK", 0), (1, "OK", 0), (2, "OK", 0)]
    assert _resp(o) == [(0, "OK", "WR_IMM", 0, 0xABCD)]
    assert not o.mem["DST"].any()


def test_a_send_that_fails_its_own_check_takes_no_receive():
    p = _prog([WR("SEND", 8, "src", 0, bad_lkey=True), WR("SEND", 8, "src", 0)], recvs=[Recv("dst", 0, 8)])
    o = M.run_model(p)
    assert _req(o) == [(0, "LOCAL_PROT_ERR"), (1, "WR_FLUSH_ERR")]
    assert _resp(o) == [] and not o.mem["DST"].any()


def test_receive_without_local_write_fails_at_the_requester():
    nolw = MR("nolw", "DST", 8, 32, M.NO_LOCAL_WRITE, "remote")
    p = _prog([WR("SEND", 8, "src", 0)], recvs=[Recv("nolw", 0, 16)], extra_mrs=[nolw])
    o = M.run_model(p)
    assert _req(o) == [(0, "REMOTE_ACCESS_ERR")] and _resp(o) == [(0, "REMOTE_ACCESS_ERR")]


def test_no_receive_is_an_rnr_error():
    o = M.run_model(_prog([WR("WRITE", 1, "src", 0, "dst", 0), WR("SEND_IMM", 4, "src", 0, imm=1)]))
    assert _req(o) == [(0, "OK", 1), (1, "RNR_RETRY_EXC_ERR")]


def test_one_syndrome_per_fault_class():
    ro = MR("ro", "DST", 8, 16, M.ACC_REMOTE_READ, "local")
    nrr = MR("nrr", "SRC", 0, 64, M.ACC_ALL & ~M.ACC_REMOTE_READ, "remote")
    cases = {
        "LOCAL_ACCESS_ERR": WR("READ", 4, "ro", 0, "src", 0),
        "LOCAL_PROT_ERR": WR("WRITE", 4, "src", 61, "dst", 0),              # one byte past the local MR
        "REMOTE_ACCESS_ERR": WR("READ", 4, "dst", 0, "nrr", 0),              # remote key without REMOTE_READ
        "LOCAL_LENGTH_ERR": WR("FA", 4, "fetch", 0, "atom", 0),
        "REMOTE_INVAL_REQ_ERR": WR("CS", 8, "fetch", 0, "atom", 4, compare=0),
    }
    for want, w in cases.items():
        o = M.run_model(_prog([w], extra_mrs=[ro, nrr]))
        assert _req(o) == [(0, want)], want
        assert not o.mem["DST"].any() and (o.mem["FETCH"] == 0xEE).all()
    o = M.run_model(_prog([WR("FA", 8, "fetch", 0, "atom", 0, add=1)], host_atom=True), host_native_atomics=False)
    assert _req(o) == [(0, "REMOTE_OP_ERR")]
    o = M.run_model(_prog([WR("FA", 8, "fetch", 0, "atom", 0, add=1)], host_atom=True), host_native_atomics=True)
    assert _req(o) == [(0, "OK", 8)]


def test_too_long_fails_before_any_key_and_takes_no_receive():
    """Longer than the maximum message length: LOCAL_LENGTH_ERR even with bad keys and an MR far too short, nothing moves,
    the receive stays for later, and the next WR is flushed.  The limit itself is a legal length."""
    for op in M.MSG_OPS:
        for n in M.too_long_lengths(M.MAX_MSG):
            w = WR(op, n, "dst" if op == "READ" else "src", 0, None if op.startswith("SEND") else ("src" if op == "READ" else "dst"),
                   0, bad_lkey=True, bad_rkey=True)
            o = M.run_model(_prog([w, WR("WRITE", 4, "src", 0, "dst", 0)], recvs=[Recv("dst", 0, 48)]))
            assert _req(o) == [(0, "LOCAL_LENGTH_ERR"), (1, "WR_FLUSH_ERR")], (op, n)
            assert _resp(o) == [] and not o.mem["DST"].any()
    o = M.run_model(_prog([WR("SEND", M.MAX_MSG, "src", 0)], recvs=[Recv("dst", 0, 48)]))
    assert _req(o) == [(0, "LOCAL_PROT_ERR")]        # at the limit the length passes and the key check fails


def test_mr_edges():
    """An access ending at the MR's last byte succeeds; one byte more is a remote access error; canaries stay."""
    ok = M.run_model(_prog([WR("WRITE", 16, "src", 0, "dst", 32)]))
    assert _req(ok) == [(0, "OK", 16)] and ok.mem["DST"][40:56].tolist() == list(range(1, 17))
    assert not ok.mem["DST"][:40].any() and not ok.mem["DST"][56:].any()
    past = M.run_model(_prog([WR("WRITE", 17, "src", 0, "dst", 32)]))
    assert _req(past) == [(0, "REMOTE_ACCESS_ERR")] and not past.mem["DST"].any()


def test_bulk_chunk_prediction():
    assert M._chunks(5 << 20, 1, 64 << 10) == [640 << 10] * 8            # grown to ~8 chunks per CTA
    assert M._chunks(5 << 20, 32, 64 << 10) == [64 << 10] * 80
    assert M._chunks(100, 32, 16 << 10) == [100]
    assert M._chunks((2 << 20) + 48, 32, 1 << 20) == [1 << 20, 1 << 20, 48]
    assert M.bulk_chunks((2 << 20) + 48, 0, 16, 32, 1 << 20) == 2        # the 48-byte tail goes generic
    assert M.bulk_chunks(1 << 20, 0, 8, 32, 1 << 20) == 0                 # misaligned destination: all generic
    assert M.bulk_chunks(4096, 0, 0, 1, 1 << 16) == 1 and M.bulk_chunks(4095, 0, 0, 1, 1 << 16) == 0
    assert M.bulk_chunks(4097, 0, 0, 1, 1 << 16) == 0                     # length not a multiple of 16


def _check_promises(wire, extra):
    """Write targets never overlap each other or a source, a fault program fails exactly once where it was built to;
    returns the fault classes and special cases the programs reached."""
    seen = set()
    for seed in range(150):
        p = M.generate(seed, {"wire": wire, "max_wrs": 60, "max_len": 1 << 18, "big_budget": 1 << 20, "allow_rnr": True,
                              "ctas": 3, "chunk_bytes": (20 << 10) + 16, **extra})
        o = M.run_model(p)
        for qi, (qp, q) in enumerate(zip(p.qps, o.qps)):
            faults = [i for i, w in enumerate(qp.wrs) if w.fault]
            errs = [c for c in q.req if c.status not in ("OK", "WR_FLUSH_ERR")]
            assert len(faults) <= 1 and len(errs) == len(faults) + p.rnr, (seed, qi)
            if faults:
                assert errs[0].wr == faults[0], (seed, qi, qp.wrs[faults[0]])
                seen.add(qp.wrs[faults[0]].fault)
            if p.rnr:
                assert q.req[-1].status == "RNR_RETRY_EXC_ERR"
            # no byte is written twice, except an atomic word after the one WRITE that seeded it
            spans = sorted((b, s, e, i) for i, b, s, e in q.writes if not b.endswith("ATOM"))
            for (b0, s0, e0, i0), (b1, s1, e1, i1) in zip(spans, spans[1:]):
                assert b0 != b1 or e0 <= s1, (seed, qi, i0, i1)
            assert not any(b.endswith("SRC") for _, b, _, _ in q.writes)
            for i, w in enumerate(qp.wrs):
                if w.op in M.RDMA_OPS and w.n == 0 and w.bad_rkey:
                    seen.add("zero_length_bad_keys")
                if w.rmr and "dstfit" in w.rmr and not w.fault:
                    seen.add("exact_fit")
                if w.fault == "too_long":
                    assert w.n > M.MAX_MSG and w.op in M.MSG_OPS, (seed, qi, i)
                    seen.add(("too_long", w.op))
    return seen


@pytest.mark.parametrize("wire", ["verbs", "softhca"])
def test_generated_programs_keep_their_promises(wire):
    """... and the generator reaches every fault class, exact fits, atomics on written words and zero-length RDMA."""
    seen = _check_promises(wire, {})
    want = set(M.FAULTS) - ({"atomic_len4"} if wire == "verbs" else set())
    assert want | {"zero_length_bad_keys", "exact_fit"} <= seen, sorted(want - seen)
    assert not any(isinstance(x, tuple) for x in seen)           # no over-long WR unless asked for


@pytest.mark.parametrize("wire", ["verbs", "softhca"])
def test_generated_programs_with_max_msg_reach_every_too_long_opcode(wire):
    seen = _check_promises(wire, {"max_msg": M.MAX_MSG})
    want = {("too_long", op) for op in M.MSG_OPS}
    assert want <= seen, sorted(want - seen)


# ---------------------------------------------------------------------------------------------------------------- the mock ConnectX
MOCK_CFG = {"wire": "verbs", "max_wrs": 60, "max_len": 1 << 18, "big_budget": 1 << 20, "allow_rnr": True}
MAX_MSG_EVERY = 3      # every third seed also builds over-long WRs (cfg["max_msg"])


@pytest.fixture(scope="module")
def verbs_lib():
    from rocnrdma_b200 import _native as N
    lib = N.load()
    if lib.rn_verbs_available() < 2 or lib.rn_verbs_is_mock() != 1:
        pytest.fail("the mock rdma-core provider did not load: " + lib.rn_verbs_why().decode(errors="replace"))
    return lib


def _seeds(n):
    s = M.replay_seed()
    return [s] if s is not None else range(M.soak_seeds(n))


def test_mock_connectx_matches_the_model_on_host_dram(verbs_lib):
    checked = 0
    for seed in _seeds(120):
        cfg = dict(MOCK_CFG, max_msg=M.MAX_MSG) if seed % MAX_MSG_EVERY == MAX_MSG_EVERY - 1 else MOCK_CFG
        M.check_seed(seed, cfg, lambda: M.VerbsWire(device=None))
        checked += 1
    assert checked >= 1


def test_mock_send_with_a_bad_lkey_takes_no_receive(verbs_lib):
    """The case the random programs found first: the requester's own failure must not reach the responder."""
    p = _prog([WR("SEND", 8, "src", 0, bad_lkey=True), WR("SEND", 8, "src", 0)], recvs=[Recv("dst", 0, 8)])
    p.cfg = {"wire": "verbs"}
    wire = M.VerbsWire(device=None)
    try:
        M.run_program(p, wire)
    finally:
        wire.close()


def test_mock_zero_length_rdma_checks_no_key(verbs_lib):
    p = _prog([WR("WRITE", 0, "src", -100, "dst", 1 << 40, bad_lkey=True, bad_rkey=True),
               WR("WRITE_IMM", 0, "src", 0, "dst", 1 << 30, imm=3, bad_rkey=True),
               WR("READ", 0, "dst", 1 << 40, "src", -3, bad_lkey=True, bad_rkey=True)], recvs=[Recv("dst", 0, 0)])
    p.cfg = {"wire": "verbs"}
    wire = M.VerbsWire(device=None)
    try:
        M.run_program(p, wire)
    finally:
        wire.close()
