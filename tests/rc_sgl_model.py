"""Scatter-gather work requests on top of the RC reference model (tests/rc_model.py): a WR type with a two-entry list, its
execution under the contract of DESIGN.md section 3.1, a program generator that splices such WRs into rc_model's random
programs, and wires that post them as lists.  rc_model.py itself is unchanged.

The contract, as the model executes it:

* The message is entry 0 then entry 1; ``n`` is the total.  A gather WRITE / WRITE_IMM writes ``[roff, roff + n)`` of
  the remote MR, a scatter READ fetches that range and puts the first ``n - n1`` bytes in entry 0 and the rest in
  entry 1, a gather SEND delivers the concatenation into the receive's buffer.  Both CQEs carry the total.
* Checks in order: the total against the maximum message length (``LOCAL_LENGTH_ERR``, before any key); each posted
  entry's local key over its own range, in list order, with the access its role needs (none for a WRITE or SEND source,
  local write for a READ destination); the remote key over the whole length; for a SEND, a receive shorter than the
  total fails with ``REMOTE_INVAL_REQ_ERR``.  A WR that fails a requester-side check consumes no receive.
* Posters drop zero-length entries (with none left, entry 0 is posted with 0 bytes), so a dropped entry's key is never
  looked at.  A ``raw`` WR is a hand-built two-segment WQE that keeps its zero-length segment: that segment's key is
  checked over an empty range.  A zero-total WRITE or READ checks no key.

``generate(seed, cfg)`` is ``rc_model.generate`` when ``cfg["sgl"]`` is not set.  With it, each QP gets 2-6 gather WRs
(every opcode that takes a list) on bytes of their own, appended to the QP's DST buffer; on loopback programs, about
one in three of them carries one fault of its own: a bad key or a read-only MR on entry 1, a gather SEND longer than
its receive, or (with ``cfg["max_msg"]``) two entries that each fit but sum past the limit.  The new WRs draw from a
random stream of their own and go in front of random WRs, never after a QP's last WR.
"""
import contextlib
import ctypes as C
import types
from dataclasses import dataclass
from typing import Optional
from unittest import mock

import numpy as np

import rc_model as M
from rc_model import MR, WR, Recv, ReqCqe, RespCqe

_run_model_rc = M.run_model        # rc_model's own model (run_program below swaps M.run_model for this module's)
SGL_OPS = ("WRITE", "WRITE_IMM", "READ", "SEND", "SEND_IMM")
SGL_FAULTS = ("bad_lkey1", "no_local_write1", "send_too_long", "send_bad_lkey1", "too_long")


@dataclass
class GWR(WR):
    sgl: bool = False              # posted as a list: entry 0 = (lmr, loff, n - n1), entry 1 = (lmr1, loff1, n1)
    lmr1: Optional[str] = None
    loff1: int = 0
    n1: int = 0
    bad_lkey1: bool = False
    raw: bool = False              # a hand-built two-segment WQE: a zero-length segment stays in it


def is_sgl(w) -> bool:
    return bool(getattr(w, "sgl", False))


def entries(w):
    """The entries the WQE carries, as (mr, off, n, bad key): zero-length ones dropped unless ``raw``."""
    es = [(w.lmr, w.loff, w.n - w.n1, w.bad_lkey), (w.lmr1, w.loff1, w.n1, w.bad_lkey1)]
    if w.raw:
        return es
    kept = [e for e in es if e[2]]
    return kept or [(w.lmr, w.loff, 0, w.bad_lkey)]


def sg_bulk_chunks(spans, remote, read, ctas, chunk_bytes):
    """Chunks of a list WQE that go through the TMA bulk path: the granule comes from the total, chunks never straddle an
    entry, entry k's remote side starts after the entries before it.  ``spans`` = [(local position, n)]."""
    total = sum(n for _, n in spans)
    want = -(-total // (8 * ctas))
    g = max(chunk_bytes, -(-want // M.KSUB) * M.KSUB)
    cnt, roff = 0, 0
    for lp, n in spans:
        for off in range(0, n, g):
            c = min(g, n - off)
            s, d = (remote + roff + off, lp + off) if read else (lp + off, remote + roff + off)
            cnt += c >= M.BULK_MIN and s % 16 == 0 and d % 16 == 0 and c % 16 == 0
        roff += n
    return cnt


# ---------------------------------------------------------------------------------------------------------------- model
def _exec_sgl(prog, qp, w, mem, o, i, rq, max_msg):
    """One list WR on a QP that has not failed.  Returns (syndrome or None, receive index taken or None)."""
    cfg = prog.cfg

    def at(mr_name, off):
        m = prog.mrs[mr_name]
        return m.buf, m.off + off

    if w.n > max_msg:
        return "LOCAL_LENGTH_ERR", None
    taken = None
    if w.op in M.RDMA_OPS and w.n == 0:
        if w.op == "WRITE_IMM":
            if rq >= len(qp.recvs):
                return "RNR_RETRY_EXC_ERR", None
            taken = rq
        return None, taken
    need = M.ACC_LOCAL_WRITE if w.op == "READ" else 0
    es = entries(w)
    for mr_name, off, n, bad in es:
        syn = M._key_check(prog.mrs[mr_name], bad, off, n, need, False)
        if syn:
            return syn, None
    if w.op != "READ" and w.op not in ("SEND", "SEND_IMM"):
        syn = M._key_check(prog.mrs[w.rmr], w.bad_rkey, w.roff, w.n, M.ACC_REMOTE_WRITE, True)
    elif w.op == "READ":
        syn = M._key_check(prog.mrs[w.rmr], w.bad_rkey, w.roff, w.n, M.ACC_REMOTE_READ, True)
    else:
        syn = None
    if syn:
        return syn, None
    if w.op in M.RECV_OPS:
        if rq >= len(qp.recvs):
            return "RNR_RETRY_EXC_ERR", None
        taken = rq
        if w.op != "WRITE_IMM":
            r = qp.recvs[rq]
            if r.n < w.n:
                return "REMOTE_INVAL_REQ_ERR", taken
            syn = M._key_check(prog.mrs[r.mr], False, r.off, w.n, M.ACC_LOCAL_WRITE, True)
            if syn:
                return syn, taken
    if w.op in ("SEND", "SEND_IMM"):
        rb, rp = at(qp.recvs[taken].mr, qp.recvs[taken].off)
    else:
        rb, rp = at(w.rmr, w.roff)
    spans, pos = [], 0
    for mr_name, off, n, _ in es:
        lb, lp = at(mr_name, off)
        if w.op == "READ":
            mem[lb][lp:lp + n] = mem[rb][rp + pos:rp + pos + n]
            o.writes.append((i, lb, lp, lp + n))
        else:
            mem[rb][rp + pos:rp + pos + n] = mem[lb][lp:lp + n]
        spans.append((lp, n))
        pos += n
    if w.op != "READ":
        o.writes.append((i, rb, rp, rp + w.n))
    o.bulk_chunks += sg_bulk_chunks([s for s in spans if s[1]], rp, w.op == "READ", cfg.get("ctas", 1),
                                    cfg.get("chunk_bytes", 1 << 19))
    return None, taken


def run_model(prog: M.Program, host_native_atomics: bool = True, resolve_cas: bool = False) -> M.Outcome:
    """rc_model.run_model, extended by list WRs: every run of ordinary WRs is executed by rc_model.run_model itself (on
    the memory as the WRs before left it), every list WR by the rules above."""
    max_msg = prog.cfg.get("max_msg") or M.MAX_MSG
    mem = {k: b.init.copy() for k, b in prog.bufs.items()}
    out = M.Outcome(mem, [M.QpOutcome() for _ in prog.qps])
    for qi, qp in enumerate(prog.qps):
        o = out.qps[qi]
        err, rq, i = False, 0, 0
        while i < len(qp.wrs):
            if err:
                o.n_wqe += 1
                o.n_err += 1
                o.req.append(ReqCqe(i, "WR_FLUSH_ERR"))
                i += 1
                continue
            w = qp.wrs[i]
            if not is_sgl(w):
                j = i
                while j < len(qp.wrs) and not is_sgl(qp.wrs[j]):
                    j += 1
                # a QP's WRs touch only its own buffers (q<i>.*): the run is executed on those alone
                own = {k: v for k, v in mem.items() if k.startswith(f"q{qi}.") or not k.startswith("q")}
                sub = M.Program(prog.seed, prog.cfg, {k: M.Buf(k, v, prog.bufs[k].mem) for k, v in own.items()}, prog.mrs,
                                [M.QpProg(qp.peer, qp.wrs[i:j], qp.recvs[rq:])], prog.rnr)
                r = _run_model_rc(sub, host_native_atomics, resolve_cas)
                so = r.qps[0]
                mem.update(r.mem)
                o.req += [ReqCqe(c.wr + i, c.status, c.opcode, c.byte_cnt) for c in so.req]
                o.resp += [RespCqe(c.recv + rq, c.status, c.kind, c.byte_cnt, c.imm) for c in so.resp]
                o.writes += [(k + i, b, s, e) for k, b, s, e in so.writes]
                o.n_wqe += so.n_wqe
                o.n_err += so.n_err
                o.bulk_chunks += so.bulk_chunks
                rq += len(so.resp)
                if so.state == "ERR":
                    err, o.state = True, "ERR"
                i = j
                continue
            o.n_wqe += 1
            syn, taken = _exec_sgl(prog, qp, w, mem, o, i, rq, max_msg)
            if taken is not None:
                rq += 1
                kind = {"SEND": "SEND", "SEND_IMM": "SEND_IMM", "WRITE_IMM": "WR_IMM"}[w.op]
                o.resp.append(RespCqe(taken, syn or "OK", kind, w.n, w.imm))
            if syn is not None:
                err, o.state = True, "ERR"
                o.n_err += 1
                o.req.append(ReqCqe(i, syn))
            elif w.signaled:
                o.req.append(ReqCqe(i, "OK", w.op, w.n))
            i += 1
    return out


# ---------------------------------------------------------------------------------------------------------------- generator
class _Tail:
    """Bump allocator over bytes appended to a buffer: 16-byte frames plus a gap, so regions never overlap."""

    def __init__(self, start):
        self.top = start + 64

    def take(self, n, mis=0, gap=48):
        start = (self.top + 15) // 16 * 16 + mis
        self.top = start + n + gap
        return start


def _sgl_for(seed, qi, cfg, prog):
    p = f"q{qi}."
    rng = np.random.default_rng([seed, qi, 0x5617])
    g = M.granule(cfg)
    src_n = prog.bufs[p + "SRC"].init.size
    cap = max(1, min(cfg["max_len"], 3 * g + 48, (src_n - 4096) // 2))
    lens = [x for x in (0, 1, 15, 16, 17, 64, 4095, 4096, 4097, 16384, 16400, g - 16, g, g + 48, 3 * g + 48) if x <= cap]
    dst = _Tail(prog.bufs[p + "DST"].init.size)
    mrs = {}
    faulty = not cfg.get("pairs") and rng.random() < 0.35
    kinds = [f for f in SGL_FAULTS if f != "too_long" or cfg.get("max_msg")]
    fault_at = -1

    def mr(kind, off, n, access, side):
        name = f"{p}g{len(mrs)}.{kind}"
        mrs[name] = MR(name, p + "DST", off, n, access, side)
        return name

    def src_off(n):             # read-only random source: any 16-byte frame that holds n bytes, any residue
        return 16 * int(rng.integers(0, max(1, (src_n - n - 32) // 16))) + int(rng.choice(M.MIS))

    new = []                    # (WR, its receive or None)
    count = int(rng.integers(2, 7))
    if faulty:
        fault_at = int(rng.integers(0, count))
    for k in range(count):
        fault = str(rng.choice(kinds)) if k == fault_at else None
        op = str(rng.choice(SGL_OPS))
        if fault in ("send_too_long", "send_bad_lkey1"):
            op = str(rng.choice(["SEND", "SEND_IMM"]))
        elif fault == "no_local_write1":
            op = "READ"
        n0, n1 = int(rng.choice(lens)), int(rng.choice(lens))
        if fault or rng.random() < 0.9:
            n0, n1 = max(n0, 1) if fault else n0, max(n1, 1)     # mostly two entries; a fault needs entry 1
        raw = fault is None and n0 == 0 and n1 > 0 and rng.random() < 0.5
        w = GWR(op, n0 + n1, sgl=True, n1=n1, raw=raw, fault=fault, signaled=bool(rng.integers(0, 4)))
        if op.endswith("IMM"):
            w.imm = int(rng.integers(0, 2**32))
        if fault == "too_long":
            w.n1 = (1 << 29) + 16
            w.n = (1 << 29) + 8 + w.n1
        m0, m1 = int(rng.choice(M.MIS)), int(rng.choice(M.MIS))
        if op == "READ":
            w.lmr, w.loff = mr("s0", dst.take(max(n0, 1), m0), max(n0, 1), M.ACC_ALL, "local"), 0
            acc1 = M.NO_LOCAL_WRITE if fault == "no_local_write1" else M.ACC_ALL
            w.lmr1, w.loff1 = mr("s1", dst.take(max(n1, 1), m1), max(n1, 1), acc1, "local"), 0
            w.rmr, w.roff = p + "src_r", src_off(w.n if fault != "too_long" else 64)
        else:
            w.lmr, w.loff = p + "src_l", src_off(n0)
            w.lmr1, w.loff1 = p + "src_l", src_off(n1)
            if op.startswith("WRITE"):
                span = w.n if fault != "too_long" else 64
                w.rmr, w.roff = mr("g", dst.take(span, int(rng.choice(M.MIS))), span, M.ACC_ALL, "remote"), 0
        w.bad_lkey1 = fault in ("bad_lkey1", "send_bad_lkey1")
        recv = None
        if op in M.RECV_OPS:
            if op == "WRITE_IMM" or fault == "too_long":
                recv = Recv(mr("rimm", dst.take(16), 16, M.ACC_ALL, "remote"), 0, 16)
            else:
                rn_ = w.n - 1 if fault == "send_too_long" else (w.n if rng.random() < 0.4 else w.n + int(rng.integers(1, 64)))
                recv = Recv(mr("rcv", dst.take(max(rn_, 1), int(rng.choice(M.MIS))), max(rn_, 1), M.ACC_ALL, "remote"), 0, rn_)
        new.append((w, recv))
    last = len(prog.qps[qi].wrs) - 1
    at = sorted(int(x) for x in rng.integers(0, max(last, 0) + 1, len(new)))
    return new, at, mrs, dst.top + 64


def _splice(prog, qi, new, at):
    """Insert new WR j in front of original WR at[j]; receives keep the order of the WRs that consume them."""
    qp = prog.qps[qi]
    rnr_last = prog.rnr and qp.wrs and qp.wrs[-1].op in M.RECV_OPS
    recv_of, k = [], 0
    for i, w in enumerate(qp.wrs):       # which original WRs own a receive, in order (as rc_model.generate adds them)
        own = w.op in M.RECV_OPS and not (rnr_last and i == len(qp.wrs) - 1)
        recv_of.append(qp.recvs[k] if own else None)
        k += own
    assert k == len(qp.recvs)
    out_w, out_r, j = [], [], 0
    for i, w in enumerate(qp.wrs):
        while j < len(at) and at[j] == i:
            x, r = new[j]
            out_w.append(x)
            if r is not None:
                out_r.append(r)
            j += 1
        out_w.append(w)
        if recv_of[i] is not None:
            out_r.append(recv_of[i])
    qp.wrs, qp.recvs = out_w, out_r


def generate(seed: int, cfg: dict) -> M.Program:
    prog = M.generate(seed, cfg)
    if not cfg.get("sgl"):
        return prog
    for qi in range(len(prog.qps)):
        new, at, mrs, dst_n = _sgl_for(seed, qi, prog.cfg, prog)
        b = prog.bufs[f"q{qi}.DST"]
        tail = np.random.default_rng([seed, qi, 0xD58]).integers(0, 256, dst_n - b.init.size, dtype=np.uint8)
        b.init = np.concatenate([b.init, tail])
        prog.mrs.update(mrs)
        _splice(prog, qi, new, at)
    for qp in prog.qps:
        for w in qp.wrs:
            if w.op == "CS":
                w.compare = None                          # resolve against the memory the gathers leave
    run_model(prog, host_native_atomics=prog.cfg.get("host_native_atomics", True), resolve_cas=True)
    for qp in prog.qps:
        for w in qp.wrs:
            if w.op == "CS" and w.compare is None:       # never executed (flushed): any value
                w.compare = 0
    return prog


# ---------------------------------------------------------------------------------------------------------------- wires
def raw_wqe(opcode, sges, raddr, rkey, flags, imm) -> bytes:
    """A two-segment WQE as given, zero-length segments included (index and QP number are filled in when it is posted)."""
    import rocnrdma_b200.wire as W
    segs = b"".join(W.data_seg(a, k, n) for a, k, n in sges)
    if opcode in (W.OP_SEND, W.OP_SEND_IMM):
        b = W.ctrl_seg(opcode, 0, 0, 1 + len(sges), flags, imm) + segs
    else:
        b = W.ctrl_seg(opcode, 0, 0, 2 + len(sges), flags, imm) + W.raddr_seg(raddr, rkey) + segs
    return b + bytes(W.WQEBB - len(b))


class _SglQp:
    """A queue pair that posts the list WRs of one program QP as lists.  rc_model.run_program makes exactly one post
    call per WR, in program order, so the n-th call belongs to WR n; a list WR's call is replaced by the list post."""
    _POSTS = ("post_raw", "post_write", "post_read", "post_send", "post_write_inline", "post_send_inline",
              "post_fetch_add", "post_cmp_swap")

    def __init__(self, qp, wrs, mrs):
        self._qp, self._wrs, self._mrs, self._next = qp, wrs, mrs, 0

    def __getattr__(self, name):
        attr = getattr(self._qp, name)
        if name not in self._POSTS:
            return attr

        def post(*a, **kw):
            w = self._wrs[self._next]
            self._next += 1
            return self._post_sgl(w) if is_sgl(w) else attr(*a, **kw)
        return post

    def _post_sgl(self, w):
        import rocnrdma_b200.wire as W
        q = self._qp

        def ent(mr_name, off, n, bad):
            m = self._mrs[mr_name]
            return (types.SimpleNamespace(addr=m.addr, lkey=m.lkey ^ 0x5A) if bad else m), off, n
        sges = [ent(w.lmr, w.loff, w.n - w.n1, w.bad_lkey), ent(w.lmr1, w.loff1, w.n1, w.bad_lkey1)]
        r = self._mrs.get(w.rmr)
        imm = w.imm if w.op.endswith("IMM") else None
        op = {"WRITE": W.OP_RDMA_WRITE, "WRITE_IMM": W.OP_RDMA_WRITE_IMM, "READ": W.OP_RDMA_READ, "SEND": W.OP_SEND,
              "SEND_IMM": W.OP_SEND_IMM}[w.op]
        if w.raw:
            b = raw_wqe(op, [(m.addr + off, m.lkey, n) for m, off, n in sges], (r.addr + w.roff) if r else 0,
                        r.rkey if r else 0, W.CTRL_CQ_UPDATE if w.signaled else 0, w.imm)
            buf, tok = (C.c_uint8 * 64)(*b), C.c_uint64()
            lib = q.ctx._lib
            if getattr(q, "_vq", None) is not None:
                rc = lib.rn_verbs_mock_post_wqe(q._vq, buf, C.byref(tok))
            else:
                rc = lib.rn_post_wqe_bytes(q._q, buf, C.byref(tok))
            assert rc == 0, rc
            return tok.value
        if w.op.startswith("WRITE"):
            return q.post_write_sg(sges, r, dst_off=w.roff, signaled=w.signaled, imm=imm)
        if w.op == "READ":
            return q.post_read_sg(sges, r, remote_off=w.roff, signaled=w.signaled)
        return q.post_send_sg(sges, signaled=w.signaled, imm=imm)


def with_sgl(wire):
    """Make ``wire`` (an rc_model wire) post every list WR as a list."""
    setup = wire.setup

    def sgl_setup(prog):
        W = setup(prog)
        wire.qps = [_SglQp(q, prog.qps[i].wrs, wire.mrs) for i, q in enumerate(wire.qps)]
        return W
    wire.setup = sgl_setup
    return wire


@contextlib.contextmanager
def _with_model():
    """rc_model.run_program compares a wire with rc_model.run_model: for list programs, with this module's model."""
    with mock.patch.object(M, "run_model", run_model):
        yield


def run_program(prog, wire, timeout_s=30.0):
    with _with_model():
        return M.run_program(prog, with_sgl(wire), timeout_s)


def check_seed(seed, cfg, make_wire, timeout_s=30.0):
    """rc_model.check_seed for list programs: generate, run on a fresh wire that posts the lists, compare."""
    prog = generate(seed, cfg)
    wire = make_wire()
    try:
        return prog, run_program(prog, wire, timeout_s)
    finally:
        wire.close()
