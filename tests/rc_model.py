"""A reference model of RC queue-pair semantics, a generator of random work-request programs, and a runner that executes a
program on either wire (the software HCA's engine, or the mock ConnectX) and compares everything with the model.

The model is plain Python and numpy and is written from the contract in DESIGN.md section 3.1, not from either wire:

* WRs of one QP complete in posting order.  A successful signaled WR gives one requester CQE (byte_cnt = its length, 8
  for an atomic); a successful unsignaled WR gives none; an error or a flush always gives one.
* The first failing WR completes with its error; every later WR of the QP is flushed (WR_FLUSH_ERR), writes nothing and
  consumes no receive; the QP ends in ERR.
* A successful WRITE / READ / SEND moves exactly its bytes and nothing else changes, canary bytes around every MR
  included.  SEND and WRITE_IMM consume receives in order; a WR that fails a requester-side check consumes none.
* Atomics execute in WR order and see every byte written by earlier WRITEs of the QP.
* Zero-length WRITE, WRITE_IMM and READ check no key and move nothing (WRITE_IMM still consumes a receive).
* A WRITE, WRITE_IMM, READ, SEND or SEND_IMM longer than the maximum message length (2^30 bytes, inclusive) fails with
  LOCAL_LENGTH_ERR before any key is looked at: it moves nothing and consumes no receive.  ``cfg["max_msg"]`` (that
  length) makes the generator build such WRs (fault ``too_long``); without it the programs are what they always were.

Programs address memory as (MR name, offset from the MR's start), so the runner only has to turn MR names into keys and
addresses; the model itself never sees a pointer.  Every buffer base is 16-byte aligned, so an offset's residue mod 16 is
the address's, which is what the engine's bulk condition looks at.
"""
import dataclasses
import gc
import os
import time
import types
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

KSUB, BULK_MIN = 16384, 4096
ACC_LOCAL_WRITE, ACC_REMOTE_WRITE, ACC_REMOTE_READ, ACC_REMOTE_ATOMIC = 1, 2, 4, 8
ACC_ALL = 15
# IB requires LOCAL_WRITE wherever REMOTE_WRITE or REMOTE_ATOMIC is granted (the verbs backend adds it), so an MR
# without LOCAL_WRITE is a read-only one
NO_LOCAL_WRITE = ACC_REMOTE_READ
RDMA_OPS = ("WRITE", "WRITE_IMM", "READ")
RECV_OPS = ("SEND", "SEND_IMM", "WRITE_IMM")
MSG_OPS = ("WRITE", "WRITE_IMM", "READ", "SEND", "SEND_IMM")
MAX_MSG = 1 << 30


def too_long_lengths(max_msg):
    """Byte counts past the maximum message length: just past it, and where a 31-bit byte count would wrap."""
    return [max_msg + 1, max_msg + 16, 2**31 - 1, 2**31, 2**31 + 64, 2**32 - 16]


def _chunks(nbytes, ctas, chunk_bytes):
    """The chunk lengths the engine cuts a WQE into (write_resolved's granule policy): at least the QP's chunk_bytes,
    grown in 16 KiB steps so that a large message makes about 8 chunks per engine CTA."""
    want = -(-nbytes // (8 * ctas))
    g = max(chunk_bytes, -(-want // KSUB) * KSUB)
    return [min(g, nbytes - off) for off in range(0, nbytes, g)]


def bulk_chunks(nbytes, src, dst, ctas, chunk_bytes):
    """How many chunks of one WQE the engine moves through the TMA bulk path: length >= 4096 and source, destination
    and length all 16-byte aligned (the rest go through the generic copy)."""
    n, off = 0, 0
    for c in _chunks(nbytes, ctas, chunk_bytes):
        if c >= BULK_MIN and (src + off) % 16 == 0 and (dst + off) % 16 == 0 and c % 16 == 0:
            n += 1
        off += c
    return n


# ---------------------------------------------------------------------------------------------------------------- program
@dataclass
class Buf:
    name: str
    init: np.ndarray          # uint8, the initial bytes
    mem: str = "dev"          # "dev" or "host" (pinned host memory on a GPU run)


@dataclass
class MR:
    name: str
    buf: str
    off: int                  # start within the buffer
    n: int
    access: int
    side: str                 # "local" (requester's HCA) or "remote" (responder's HCA)


@dataclass
class WR:
    op: str                   # WRITE, WRITE_IMM, READ, SEND, SEND_IMM, FA, CS, NOP
    n: int = 0
    lmr: Optional[str] = None
    loff: int = 0
    rmr: Optional[str] = None
    roff: int = 0
    signaled: bool = True
    imm: int = 0
    inline: Optional[bytes] = None
    add: int = 0              # FA addend / CS swap value
    compare: Optional[int] = None   # CS: None until the generator resolves it against the model
    cas_hit: bool = False
    bad_lkey: bool = False
    bad_rkey: bool = False
    fault: Optional[str] = None     # what the generator meant to break (reporting only)


@dataclass
class Recv:
    mr: str
    off: int
    n: int


@dataclass
class QpProg:
    peer: int                 # index of the QP that answers (itself for loopback)
    wrs: List[WR] = field(default_factory=list)
    recvs: List[Recv] = field(default_factory=list)   # posted on the peer's receive queue, in order


@dataclass
class Program:
    seed: int
    cfg: dict
    bufs: Dict[str, Buf]
    mrs: Dict[str, MR]
    qps: List[QpProg]
    rnr: bool = False


# ---------------------------------------------------------------------------------------------------------------- model
@dataclass
class ReqCqe:
    wr: int
    status: str
    opcode: str = ""
    byte_cnt: int = 0


@dataclass
class RespCqe:
    recv: int
    status: str
    kind: str = ""            # SEND, SEND_IMM, WR_IMM
    byte_cnt: int = 0
    imm: int = 0


@dataclass
class QpOutcome:
    req: List[ReqCqe] = field(default_factory=list)
    resp: List[RespCqe] = field(default_factory=list)   # completions of this program's receives (on the peer's RQ)
    state: str = "RTS"
    n_wqe: int = 0
    n_err: int = 0
    bulk_chunks: int = 0
    writes: list = field(default_factory=list)          # (wr index, buffer, lo, hi) for failure reports


@dataclass
class Outcome:
    mem: Dict[str, np.ndarray]
    qps: List[QpOutcome]


def _key_check(mr: MR, bad: bool, off: int, n: int, need: int, remote: bool) -> Optional[str]:
    prot = "REMOTE_ACCESS_ERR" if remote else "LOCAL_PROT_ERR"
    if bad or off < 0 or off + n > mr.n:
        return prot
    if (mr.access & need) != need:
        return "REMOTE_ACCESS_ERR" if remote else "LOCAL_ACCESS_ERR"
    return None


def run_model(prog: Program, host_native_atomics: bool = True, resolve_cas: bool = False) -> Outcome:
    """Execute every QP's program (QPs touch disjoint memory, so one after the other is as good as interleaved).
    With ``resolve_cas`` a CS whose compare is still None gets one that hits (``cas_hit``) or misses the word's current
    value: that is how the generator makes half of the CAS succeed."""
    cfg = prog.cfg
    max_msg = cfg.get("max_msg") or MAX_MSG
    mem = {k: b.init.copy() for k, b in prog.bufs.items()}
    out = Outcome(mem, [QpOutcome() for _ in prog.qps])

    def at(mr_name, off, n):
        mr = prog.mrs[mr_name]
        return mr.buf, mr.off + off

    for qi, qp in enumerate(prog.qps):
        o = out.qps[qi]
        err = False
        rq = 0                                   # next receive of this program's receive list
        for i, w in enumerate(qp.wrs):
            o.n_wqe += 1
            if err:
                o.n_err += 1
                o.req.append(ReqCqe(i, "WR_FLUSH_ERR"))
                continue
            syn, nbytes = None, w.n
            recv_taken = None
            if w.op in MSG_OPS and w.n > max_msg:
                syn = "LOCAL_LENGTH_ERR"                # before any key, and before a receive is matched
            elif w.op == "NOP":
                nbytes = 0
            elif w.op in RDMA_OPS and w.n == 0:
                # zero-length RDMA: no key is looked at, nothing moves; WRITE_IMM still needs and takes a receive
                if w.op == "WRITE_IMM":
                    if rq >= len(qp.recvs):
                        syn = "RNR_RETRY_EXC_ERR"
                    else:
                        recv_taken = rq
                        rq += 1
            elif w.op in ("WRITE", "WRITE_IMM"):
                if w.inline is None:
                    syn = _key_check(prog.mrs[w.lmr], w.bad_lkey, w.loff, w.n, 0, False)
                if syn is None:
                    syn = _key_check(prog.mrs[w.rmr], w.bad_rkey, w.roff, w.n, ACC_REMOTE_WRITE, True)
                if syn is None and w.op == "WRITE_IMM":
                    if rq >= len(qp.recvs):
                        syn = "RNR_RETRY_EXC_ERR"
                    else:
                        recv_taken = rq
                        rq += 1
                if syn is None:
                    db, dp = at(w.rmr, w.roff, w.n)
                    if w.inline is not None:
                        mem[db][dp:dp + w.n] = np.frombuffer(w.inline, dtype=np.uint8)
                    else:
                        sb, sp = at(w.lmr, w.loff, w.n)
                        mem[db][dp:dp + w.n] = mem[sb][sp:sp + w.n]
                        o.bulk_chunks += bulk_chunks(w.n, sp, dp, cfg.get("ctas", 1), cfg.get("chunk_bytes", 1 << 19))
                    o.writes.append((i, db, dp, dp + w.n))
            elif w.op == "READ":
                syn = _key_check(prog.mrs[w.lmr], w.bad_lkey, w.loff, w.n, ACC_LOCAL_WRITE, False)
                if syn is None:
                    syn = _key_check(prog.mrs[w.rmr], w.bad_rkey, w.roff, w.n, ACC_REMOTE_READ, True)
                if syn is None:
                    db, dp = at(w.lmr, w.loff, w.n)
                    sb, sp = at(w.rmr, w.roff, w.n)
                    mem[db][dp:dp + w.n] = mem[sb][sp:sp + w.n]
                    o.bulk_chunks += bulk_chunks(w.n, sp, dp, cfg.get("ctas", 1), cfg.get("chunk_bytes", 1 << 19))
                    o.writes.append((i, db, dp, dp + w.n))
            elif w.op in ("SEND", "SEND_IMM"):
                if w.inline is None:
                    syn = _key_check(prog.mrs[w.lmr], w.bad_lkey, w.loff, w.n, 0, False)
                if syn is None:
                    if rq >= len(qp.recvs):
                        syn = "RNR_RETRY_EXC_ERR"
                    else:
                        r = qp.recvs[rq]
                        recv_taken = rq
                        rq += 1
                        if r.n < w.n:
                            syn = "REMOTE_INVAL_REQ_ERR"
                        else:
                            syn = _key_check(prog.mrs[r.mr], False, r.off, w.n, ACC_LOCAL_WRITE, True)
                if syn is None:
                    db, dp = at(r.mr, r.off, w.n)
                    if w.inline is not None:
                        mem[db][dp:dp + w.n] = np.frombuffer(w.inline, dtype=np.uint8)
                    else:
                        sb, sp = at(w.lmr, w.loff, w.n)
                        mem[db][dp:dp + w.n] = mem[sb][sp:sp + w.n]
                        o.bulk_chunks += bulk_chunks(w.n, sp, dp, cfg.get("ctas", 1), cfg.get("chunk_bytes", 1 << 19))
                    o.writes.append((i, db, dp, dp + w.n))
            elif w.op in ("FA", "CS"):
                if w.n != 8:
                    syn = "LOCAL_LENGTH_ERR"
                else:
                    syn = _key_check(prog.mrs[w.lmr], w.bad_lkey, w.loff, 8, ACC_LOCAL_WRITE, False)
                    if syn is None and w.roff % 8:
                        syn = "REMOTE_INVAL_REQ_ERR"
                    if syn is None:
                        syn = _key_check(prog.mrs[w.rmr], w.bad_rkey, w.roff, 8, ACC_REMOTE_ATOMIC, True)
                    if syn is None and prog.bufs[prog.mrs[w.rmr].buf].mem == "host" and not host_native_atomics:
                        syn = "REMOTE_OP_ERR"
                if syn is None:
                    tb, tp = at(w.rmr, w.roff, 8)
                    old = int(mem[tb][tp:tp + 8].view(np.uint64)[0])
                    if w.op == "CS" and w.compare is None and resolve_cas:
                        w.compare = old if w.cas_hit else old ^ (1 + (w.add & 0xFFFF))
                    new = (old + w.add) & (2**64 - 1) if w.op == "FA" else (w.add if old == w.compare else old)
                    mem[tb][tp:tp + 8] = np.array([new], dtype=np.uint64).view(np.uint8)
                    fb, fp = at(w.lmr, w.loff, 8)
                    mem[fb][fp:fp + 8] = np.array([old], dtype=np.uint64).view(np.uint8)
                    o.writes.append((i, tb, tp, tp + 8))
                    o.writes.append((i, fb, fp, fp + 8))
                    nbytes = 8
            else:
                raise ValueError(w.op)
            if recv_taken is not None:
                kind = {"SEND": "SEND", "SEND_IMM": "SEND_IMM", "WRITE_IMM": "WR_IMM"}[w.op]
                o.resp.append(RespCqe(recv_taken, syn or "OK", kind, w.n, w.imm))
            if syn is not None:
                err = True
                o.n_err += 1
                o.state = "ERR"
                o.req.append(ReqCqe(i, syn))
            elif w.signaled:
                o.req.append(ReqCqe(i, "OK", w.op, nbytes))
    return out


# ---------------------------------------------------------------------------------------------------------------- generator
def granule(cfg):
    return cfg.get("chunk_bytes", 1 << 19)


def _edge_lengths(cfg):
    g = granule(cfg)
    e = [0, 1, 15, 16, 17, 63, 64, 65, 4095, 4096, 4097, 16383, 16384, 16385, g - 16, g, g + 1, g + 16, 2 * g + 48]
    return [x for x in e if x <= cfg["max_len"]]


class _Alloc:
    """Bump allocator over one buffer: every region gets its own 16-byte frame plus a gap, so regions never overlap and
    bytes between them are canaries.  ``mis`` is the start's residue mod 16."""

    def __init__(self):
        self.top = 64

    def take(self, n, mis=0, gap=48):
        start = (self.top + 15) // 16 * 16 + mis
        self.top = start + n + gap
        return start


FAULTS = ["bad_lkey", "bad_rkey", "local_past_end", "remote_past_end", "no_remote_write", "no_remote_read",
          "no_remote_atomic", "no_local_write", "atomic_misaligned", "atomic_len4", "send_too_long", "recv_no_local_write"]
MIS = (0, 1, 8, 15)


def generate(seed: int, cfg: dict) -> Program:
    """A random program for ``cfg``: n_qps QPs (loopback, or connected pairs when ``pairs``), up to ``max_wrs`` WRs each,
    lengths biased to the engine's edges, and about one program in three with exactly one faulting WR."""
    rng = np.random.default_rng(seed)
    cfg = dict(cfg)
    verbs = cfg.get("wire") == "verbs"
    n_qps = cfg.get("n_qps") or int(rng.integers(1, 5))
    pairs = cfg.get("pairs", bool(rng.integers(0, 2))) and n_qps >= 2
    cfg["n_qps"], cfg["pairs"] = n_qps, pairs
    if "shared_cq" not in cfg:
        cfg["shared_cq"] = bool(rng.integers(0, 4) == 0)
    edges = _edge_lengths(cfg)
    bufs, mrs, qps = {}, {}, []
    # Faults and RNR only on loopback QPs: a failed QP stops answering its peer, and when the peer notices depends on
    # timing the model does not know (DESIGN.md section 6).
    rnr_prog = not pairs and cfg.get("allow_rnr", False) and rng.random() < 0.3
    fault_prog = not pairs and not rnr_prog and rng.random() < 0.5
    data_mem = cfg.get("data_mem", "dev")

    def pick_len(cap):
        r = rng.random()
        if r < 0.6:
            n = int(rng.choice(edges))
        elif r < 0.9:
            n = int(np.exp(rng.uniform(0, np.log(min(cap, 1 << 16)))))
        else:
            n = int(rng.integers(1, cap + 1))
        return min(n, cap)

    for qi in range(n_qps):
        peer = (qi ^ 1) if pairs and (qi ^ 1) < n_qps else qi
        p = f"q{qi}."
        n_wr = int(rng.integers(max(2, cfg["max_wrs"] // 3), cfg["max_wrs"] + 1))
        big_left = cfg.get("big_budget", 16 << 20)
        src_n = min(cfg["max_len"], big_left) + 4096
        dst = _Alloc()
        atom_words = 16
        fetch = _Alloc()
        written_words, atomic_words = set(), set()
        wrs, recvs = [], []
        extra_mrs = []            # (name, buf, off, n, access, side)
        fault_at = int(rng.integers(0, n_wr)) if fault_prog else -1
        fault_kind = None
        if fault_prog:
            kinds = [f for f in FAULTS if not (verbs and f == "atomic_len4")] + ["too_long"] * (len(FAULTS) if cfg.get("max_msg") else 0)
            fault_kind = kinds[int(rng.integers(0, len(kinds)))]
        exact_fits = 0 if fault_prog else int(rng.integers(1, 4))
        exact_at = set(int(x) for x in rng.choice(n_wr, size=min(exact_fits, n_wr), replace=False)) if exact_fits else set()
        unsig_left = 0
        ops = ["WRITE"] * 25 + ["WRITE_IMM"] * 7 + ["READ"] * 15 + ["SEND"] * 9 + ["SEND_IMM"] * 5 + ["IWRITE"] * 6 + \
              ["IWRITE_IMM"] * 3 + ["ISEND"] * 4 + ["FA"] * 7 + ["CS"] * 7 + ([] if verbs else ["NOP"] * 3)

        def src_off(n):
            # Read-only random source: any offset with the chosen residue mod 16 (sources may overlap each other)
            hi = max(0, (src_n - n - 16) // 16)
            return int(rng.integers(0, hi + 1)) * 16 + int(rng.choice(MIS))

        def new_mr(kind, buf, off, n, access, side):
            name = f"{p}x{len(extra_mrs)}.{kind}"
            extra_mrs.append((name, buf, off, n, access, side))
            return name

        for i in range(n_wr):
            fault = fault_kind if i == fault_at else None
            exact = i in exact_at
            op = str(rng.choice(ops))
            # a fault or an exact fit picks an opcode it applies to
            if fault in ("bad_lkey", "local_past_end"):
                op = str(rng.choice(["WRITE", "READ", "SEND", "SEND_IMM", "FA"]))
            elif fault in ("bad_rkey", "remote_past_end"):
                op = str(rng.choice(["WRITE", "WRITE_IMM", "READ", "CS"]))
            elif fault == "no_remote_write":
                op = str(rng.choice(["WRITE", "WRITE_IMM", "IWRITE"]))
            elif fault == "no_remote_read":
                op = "READ"
            elif fault in ("no_remote_atomic", "atomic_misaligned", "atomic_len4"):
                op = str(rng.choice(["FA", "CS"]))
            elif fault == "no_local_write":
                op = str(rng.choice(["READ", "FA"]))
            elif fault in ("send_too_long", "recv_no_local_write"):
                op = str(rng.choice(["SEND", "SEND_IMM", "ISEND"]))
            elif fault == "too_long":
                op = str(rng.choice(MSG_OPS))
            elif exact:
                op = str(rng.choice(["WRITE", "READ", "SEND"]))
            if rnr_prog and i == n_wr - 1:
                op = "SEND"
            if unsig_left == 0 and rng.random() < 0.09:
                unsig_left = int(rng.integers(1, 7))
            signaled = unsig_left == 0 or i == n_wr - 1
            unsig_left = max(0, unsig_left - 1)
            w = WR(op=op, signaled=signaled, fault=fault)
            inline = op.startswith("I")
            base = op[1:] if inline else op
            w.op = base
            if base in ("WRITE_IMM", "SEND_IMM"):
                w.imm = int(rng.integers(0, 2**32))
            if base == "NOP":
                pass
            elif inline:
                n = int(rng.integers(1, 29))
                if fault in ("send_too_long", "recv_no_local_write"):
                    n = max(n, 2)
                w.n, w.inline = n, rng.integers(0, 256, n, dtype=np.uint8).tobytes()
                if base.startswith("WRITE"):
                    w.rmr, w.roff = p + "dst_r", dst.take(n, int(rng.choice(MIS))) - 64
                    if fault == "no_remote_write":
                        w.rmr = new_mr("dst_norw", p + "DST", 64 + w.roff, n, ACC_ALL & ~ACC_REMOTE_WRITE, "remote")
                        w.roff = 0
            elif base in ("FA", "CS"):
                w.n = 4 if fault == "atomic_len4" else 8
                w.add = int(rng.integers(0, 2**63)) * 2 + int(rng.integers(0, 2))
                w.cas_hit = bool(rng.integers(0, 2))
                w.lmr, w.loff = p + "fetch", fetch.take(8, int(rng.choice((0, 0, 0, 1))), gap=8) - 64
                word = int(rng.integers(0, atom_words))
                w.rmr, w.roff = p + "atom", 8 * word
                atomic_words.add(word)
                if fault == "atomic_misaligned":
                    w.roff += 4
                elif fault == "no_remote_atomic":
                    w.rmr = p + "atom_noatomic"
                elif fault == "no_local_write":
                    w.lmr = new_mr("fetch_nolw", p + "FETCH", 64 + w.loff, 8, NO_LOCAL_WRITE, "local")
                    w.loff = 0
                elif fault == "bad_lkey":
                    w.bad_lkey = True
                elif fault == "bad_rkey":
                    w.bad_rkey = True
                elif fault == "local_past_end":
                    w.lmr = new_mr("fetch7", p + "FETCH", 64 + w.loff, 7, ACC_ALL, "local")
                    w.loff = 0
                elif fault == "remote_past_end":
                    w.rmr = new_mr("atom7", p + "ATOM", 8 * word, 7, ACC_ALL, "remote")
                    w.roff = 0
            elif fault == "too_long":
                # far longer than its MRs, which the length-first rule makes harmless: nothing may be looked at or moved
                w.n = int(rng.choice(too_long_lengths(cfg["max_msg"])))
                if base == "READ":
                    w.lmr, w.loff = p + "dst_l", dst.take(64) - 64
                    w.rmr, w.roff = p + "src_r", src_off(64)
                else:
                    w.lmr, w.loff = p + "src_l", src_off(64)
                    if base.startswith("WRITE"):
                        w.rmr, w.roff = p + "dst_r", dst.take(64) - 64
            else:
                n = pick_len(min(cfg["max_len"], max(1, big_left)))
                if exact or fault:
                    n = max(n, 1)           # zero-length RDMA checks no key: a fault needs bytes
                if fault in ("local_past_end", "remote_past_end"):
                    n = max(n, 2)           # the MR is one byte shorter than the access, and not empty
                if n > 4 * granule(cfg):
                    big_left -= n
                w.n = n
                smis, dmis = int(rng.choice(MIS)), int(rng.choice(MIS))
                if rng.random() < 0.3:
                    dmis = smis
                # the one intended cross-WR dependency: an 8-byte WRITE to an atomic word, before any atomic on it
                free_words = [k for k in range(atom_words) if k not in written_words and k not in atomic_words]
                if base == "WRITE" and fault is None and not exact and free_words and rng.random() < 0.12:
                    word = int(rng.choice(free_words))
                    written_words.add(word)
                    w.n = 8
                    w.lmr, w.loff = p + "src_l", src_off(8)
                    w.rmr, w.roff = p + "atom", 8 * word
                    wrs.append(w)
                    continue
                if base in ("WRITE", "WRITE_IMM"):
                    w.lmr, w.loff = p + "src_l", src_off(n)
                    w.rmr, w.roff = p + "dst_r", dst.take(n, dmis) - 64
                    if exact or fault == "remote_past_end":
                        w.rmr = new_mr("dstfit", p + "DST", 64 + w.roff, n - (fault is not None), ACC_REMOTE_WRITE, "remote")
                        w.roff = 0
                    elif fault == "local_past_end":
                        w.lmr = new_mr("srcfit", p + "SRC", w.loff, n - 1, ACC_ALL, "local")
                        w.loff = 0
                    elif fault == "no_remote_write":
                        w.rmr = new_mr("dst_norw", p + "DST", 64 + w.roff, n, ACC_ALL & ~ACC_REMOTE_WRITE, "remote")
                        w.roff = 0
                    if n == 0 and fault is None and rng.random() < 0.5:
                        w.bad_lkey = w.bad_rkey = True      # zero-length: keys are not looked at
                        w.loff, w.roff = -(1 << 20), 1 << 40
                elif base == "READ":
                    w.lmr, w.loff = p + "dst_l", dst.take(n, dmis) - 64
                    w.rmr, w.roff = p + "src_r", src_off(n)
                    if exact or fault == "local_past_end":
                        w.lmr = new_mr("dstfit", p + "DST", 64 + w.loff, n - (fault is not None), ACC_LOCAL_WRITE, "local")
                        w.loff = 0
                    elif fault == "remote_past_end":
                        w.rmr = new_mr("srcfit", p + "SRC", w.roff, n - 1, ACC_REMOTE_READ, "remote")
                        w.roff = 0
                    elif fault == "no_remote_read":
                        w.rmr = new_mr("src_norr", p + "SRC", 0, src_n, ACC_ALL & ~ACC_REMOTE_READ, "remote")
                    elif fault == "no_local_write":
                        w.lmr = new_mr("dst_nolw", p + "DST", 64 + w.loff, n, NO_LOCAL_WRITE, "local")
                        w.loff = 0
                    if n == 0 and fault is None and rng.random() < 0.5:
                        w.bad_lkey = w.bad_rkey = True
                        w.loff, w.roff = 1 << 40, -(1 << 20)
                else:   # SEND, SEND_IMM
                    w.lmr, w.loff = p + "src_l", src_off(n)
                    if fault == "local_past_end":
                        w.lmr = new_mr("srcfit", p + "SRC", w.loff, n - 1, ACC_ALL, "local")
                        w.loff = 0
                if fault == "bad_lkey":
                    w.bad_lkey = True
                elif fault == "bad_rkey":
                    w.bad_rkey = True
            # its receive, on the responder's queue
            if base in RECV_OPS and not (rnr_prog and i == n_wr - 1):
                if base == "WRITE_IMM" or fault == "too_long":
                    recvs.append(Recv(p + "rcv", dst.take(16) - 64, 16))
                else:
                    if fault == "send_too_long":
                        rn_ = w.n - 1
                    elif exact or rng.random() < 0.3:
                        rn_ = w.n
                    else:
                        rn_ = w.n + int(rng.integers(1, 64))
                    roff = dst.take(max(rn_, 1), int(rng.choice(MIS)))
                    mr = p + "rcv"
                    if fault == "recv_no_local_write":
                        mr = new_mr("rcv_nolw", p + "DST", roff, max(rn_, 1), NO_LOCAL_WRITE, "remote")
                        roff = 64
                    recvs.append(Recv(mr, roff - 64, rn_))
            wrs.append(w)
        dst_n = dst.top + 64
        rnd = np.random.default_rng(seed * 7919 + qi)
        bufs[p + "SRC"] = Buf(p + "SRC", rnd.integers(0, 256, src_n, dtype=np.uint8), data_mem)
        bufs[p + "DST"] = Buf(p + "DST", rnd.integers(0, 256, dst_n, dtype=np.uint8), data_mem)
        bufs[p + "ATOM"] = Buf(p + "ATOM", rnd.integers(0, 256, 8 * atom_words + 64, dtype=np.uint8), cfg.get("atom_mem", "dev"))
        bufs[p + "FETCH"] = Buf(p + "FETCH", rnd.integers(0, 256, fetch.top + 128, dtype=np.uint8), data_mem)
        # the working MRs: sub-ranges of their buffers (canaries on both sides), each missing an access bit it never needs
        drop = lambda need: ACC_ALL & ~int(rng.choice([b for b in (2, 4, 8) if not b & need] + [0]))
        mrs[p + "src_l"] = MR(p + "src_l", p + "SRC", 0, src_n, drop(ACC_REMOTE_READ), "local")
        mrs[p + "src_r"] = MR(p + "src_r", p + "SRC", 0, src_n, drop(ACC_REMOTE_READ), "remote")
        mrs[p + "dst_r"] = MR(p + "dst_r", p + "DST", 64, dst_n - 128, drop(ACC_REMOTE_WRITE), "remote")
        mrs[p + "dst_l"] = MR(p + "dst_l", p + "DST", 64, dst_n - 128, drop(ACC_LOCAL_WRITE), "local")
        mrs[p + "rcv"] = MR(p + "rcv", p + "DST", 64, dst_n - 128, drop(ACC_LOCAL_WRITE), "remote")
        mrs[p + "atom"] = MR(p + "atom", p + "ATOM", 0, 8 * atom_words, ACC_ALL, "remote")
        mrs[p + "atom_noatomic"] = MR(p + "atom_noatomic", p + "ATOM", 0, 8 * atom_words, ACC_ALL & ~ACC_REMOTE_ATOMIC, "remote")
        mrs[p + "fetch"] = MR(p + "fetch", p + "FETCH", 64, fetch.top, drop(ACC_LOCAL_WRITE), "local")
        for name, buf, off, n, acc, side in extra_mrs:
            mrs[name] = MR(name, buf, off, n, acc, side)
        qps.append(QpProg(peer, wrs, recvs))
    prog = Program(seed, cfg, bufs, mrs, qps, rnr=rnr_prog)
    run_model(prog, host_native_atomics=cfg.get("host_native_atomics", True), resolve_cas=True)
    for qp in prog.qps:
        for w in qp.wrs:
            if w.op == "CS" and w.compare is None:       # never executed (flushed or failed): any value
                w.compare = 0
    return prog


def describe_wr(prog: Program, qi: int, i: int) -> str:
    w = prog.qps[qi].wrs[i]
    d = {k: v for k, v in dataclasses.asdict(w).items() if v not in (None, False, 0, b"") or k == "n"}
    if w.inline is not None:
        d["inline"] = f"<{len(w.inline)} bytes>"
    return f"qp {qi} wr {i}: {d}"


# ---------------------------------------------------------------------------------------------------------------- runner
class Mismatch(AssertionError):
    pass


def replay_hint(prog: Program, env="RN_RC_SEED"):
    return f"replay: {env}={prog.seed} (config {prog.cfg}, rnr={prog.rnr})"


def run_program(prog: Program, wire, timeout_s: float = 30.0):
    """Execute ``prog`` through ``wire`` (an object with the methods of :class:`WireBase`) and compare everything with
    the model.  Raises :class:`Mismatch` naming the seed, the config and the first WR whose outcome differs."""
    import rocnrdma_b200.wire as W
    cfg = prog.cfg
    model = run_model(prog, host_native_atomics=wire.host_native_atomics)
    opcode = {"WRITE": W.OP_RDMA_WRITE, "WRITE_IMM": W.OP_RDMA_WRITE_IMM, "READ": W.OP_RDMA_READ, "SEND": W.OP_SEND,
              "SEND_IMM": W.OP_SEND_IMM, "FA": W.OP_ATOMIC_FA, "CS": W.OP_ATOMIC_CS, "NOP": W.OP_NOP}
    ctx_of = wire.setup(prog)           # allocates + fills buffers, registers MRs, creates and connects QPs
    qps = wire.qps
    mr = wire.mrs
    recv_tok = [dict() for _ in qps]    # per QP that owns the receive queue: token -> receive index
    for qi, qp in enumerate(prog.qps):
        for ri, r in enumerate(qp.recvs):
            tok = wire.post_recv(qps[qp.peer], mr[r.mr], r.off, r.n)
            recv_tok[qp.peer][tok & 0xFFFF] = (qi, ri)
    send_tok = [dict() for _ in qps]

    def post(qi, i, w: WR):
        q, l, r = qps[qi], mr.get(w.lmr), mr.get(w.rmr)
        if w.op == "NOP":
            return q.post_raw(W.OP_NOP, signaled=w.signaled)
        if w.inline is not None:
            imm = w.imm if w.op.endswith("IMM") else None
            if w.op.startswith("WRITE"):
                return q.post_write_inline(r, w.inline, dst_off=w.roff, signaled=w.signaled, imm=imm)
            return q.post_send_inline(w.inline, signaled=w.signaled, imm=imm)
        lkey = (l.lkey ^ 0x5A) if w.bad_lkey else (l.lkey if l else 0)
        rkey = (r.rkey ^ 0x5A) if w.bad_rkey else (r.rkey if r else 0)
        laddr = (l.addr + w.loff) & (2**64 - 1) if l else 0
        raddr = (r.addr + w.roff) & (2**64 - 1) if r else 0
        if w.op in ("FA", "CS"):
            if w.n != 8:
                return q.post_raw(opcode[w.op], laddr, lkey, raddr, rkey, w.n, signaled=w.signaled)
            if w.bad_lkey or w.bad_rkey:
                l = types.SimpleNamespace(addr=l.addr, lkey=lkey)
                r = types.SimpleNamespace(addr=r.addr, rkey=rkey)
            if w.op == "FA":
                return q.post_fetch_add(l, r, w.add, local_off=w.loff, remote_off=w.roff, signaled=w.signaled)
            return q.post_cmp_swap(l, r, w.compare, w.add, local_off=w.loff, remote_off=w.roff, signaled=w.signaled)
        if w.fault or w.bad_lkey or w.bad_rkey:
            return q.post_raw(opcode[w.op], laddr, lkey, raddr, rkey, w.n, signaled=w.signaled, imm=w.imm)
        imm = w.imm if w.op.endswith("IMM") else None
        if w.op.startswith("WRITE"):
            return q.post_write(l, r, w.n, src_off=w.loff, dst_off=w.roff, signaled=w.signaled, imm=imm)
        if w.op == "READ":
            return q.post_read(l, r, w.n, local_off=w.loff, remote_off=w.roff, signaled=w.signaled)
        return q.post_send(l, w.n, src_off=w.loff, signaled=w.signaled, imm=imm)

    def post_all():
        # interleave the QPs' programs, as concurrent posters would
        pos = [0] * len(prog.qps)
        rng = np.random.default_rng(prog.seed)
        while any(pos[k] < len(prog.qps[k].wrs) for k in range(len(pos))):
            for qi, qp in enumerate(prog.qps):
                for _ in range(int(rng.integers(1, 9))):
                    if pos[qi] < len(qp.wrs):
                        send_tok[qi][post(qi, pos[qi], qp.wrs[pos[qi]]) & 0xFFFF] = pos[qi]
                        pos[qi] += 1

    # how many CQEs each CQ must deliver
    expect = {}
    for qi, o in enumerate(model.qps):
        expect[id(qps[qi].scq)] = expect.get(id(qps[qi].scq), 0) + len(o.req)
        rcq = qps[prog.qps[qi].peer].rcq
        expect[id(rcq)] = expect.get(id(rcq), 0) + len(o.resp)
    cqs, cq_owner = {}, {}                # every CQ belongs to one QP (a shared CQ to both halves of one QP)
    for k, q in enumerate(qps):
        for cq in (q.scq, q.rcq):
            cqs[id(cq)], cq_owner[id(cq)] = cq, k
    got = {k: [] for k in cqs}
    try:
        wire.run(post_all, lambda: _collect(cqs, expect, got, timeout_s))
    except TimeoutError as e:
        raise Mismatch(f"{e}; {replay_hint(prog)}")
    final = wire.finish(prog)            # dict: buffer name -> np.ndarray, qp counters
    # ---- demultiplex the CQEs
    req = [[] for _ in qps]
    resp = [[] for _ in prog.qps]
    req_ops = {W.CQE_REQ, W.CQE_REQ_ERR}
    kinds = {W.CQE_RESP_SEND: "SEND", W.CQE_RESP_SEND_IMM: "SEND_IMM", W.CQE_RESP_WR_IMM: "WR_IMM"}
    for k, wcs in got.items():
        for wc in wcs:
            qi = cq_owner[k]
            if wc.qpn != qps[qi].qpn:
                raise Mismatch(f"completion {wc} on a CQ of qp {qi} (qpn {qps[qi].qpn}); {replay_hint(prog)}")
            if wc.opcode in req_ops:
                pos = send_tok[qi].get(wc.wqe_counter & 0xFFFF)
                req[qi].append(ReqCqe(pos, wc.status, "", wc.byte_cnt))
            else:
                owner, ri = recv_tok[qi].get(wc.wqe_counter & 0xFFFF, (None, None))
                if owner is None:
                    raise Mismatch(f"unknown receive completion {wc} on qp {qi}; {replay_hint(prog)}")
                resp[owner].append(RespCqe(ri, wc.status, kinds.get(wc.opcode, "ERR"), wc.byte_cnt, wc.imm))
    # ---- compare, per QP, first difference first
    errors = []
    for qi, o in enumerate(model.qps):
        a = req[qi]
        for k in range(max(len(a), len(o.req))):
            m = o.req[k] if k < len(o.req) else None
            g = a[k] if k < len(a) else None
            if m is None or g is None or m.wr != g.wr or m.status != g.status or (m.status == "OK" and m.byte_cnt != g.byte_cnt):
                wr_i = (m or g).wr
                errors.append(f"requester CQE #{k} of qp {qi}: model {m}, got {g}; " +
                              (describe_wr(prog, qi, wr_i) if wr_i is not None else ""))
                break
        a = resp[qi]
        for k in range(max(len(a), len(o.resp))):
            m = o.resp[k] if k < len(o.resp) else None
            g = a[k] if k < len(a) else None
            same = m is not None and g is not None and m.recv == g.recv and m.status == g.status
            if same and m.status == "OK":
                same = m.kind == g.kind and m.byte_cnt == g.byte_cnt and (m.kind == "SEND" or m.imm == g.imm)
            if not same:
                errors.append(f"responder CQE #{k} for qp {qi}'s receives: model {m}, got {g}")
                break
        c = final["counters"][qi]
        if (c["state"], c["n_wqe"], c["n_err"]) != (o.state, o.n_wqe, o.n_err):
            errors.append(f"qp {qi}: state/n_wqe/n_err model {(o.state, o.n_wqe, o.n_err)}, got "
                          f"{(c['state'], c['n_wqe'], c['n_err'])}")
    for name, want in model.mem.items():
        have = final["mem"][name]
        if not np.array_equal(want, have):
            bad = np.flatnonzero(want != have)
            lo, hi = int(bad[0]), int(bad[-1])
            who = [f"qp {qi} wr {i}" for qi, o in enumerate(model.qps) for i, b, s, e in o.writes if b == name and s <= lo + 16 and e >= lo - 16]
            errors.append(f"buffer {name}: {bad.size} bytes differ in [{lo}, {hi}] (model writers near the first: {who[:4]})")
    if "bulk_chunks" in final and final["bulk_chunks"] != sum(o.bulk_chunks for o in model.qps):
        errors.append(f"bulk chunks: model {sum(o.bulk_chunks for o in model.qps)}, engine {final['bulk_chunks']}")
    if errors:
        raise Mismatch("\n".join(errors[:8]) + f"\n{replay_hint(prog)}")
    return model


def _collect(cqs, expect, got, timeout_s):
    t0 = time.monotonic()
    while True:
        short = False
        for k, cq in cqs.items():
            if len(got[k]) < expect.get(k, 0):
                got[k] += cq.poll(min(32, expect[k] - len(got[k])))
                short = short or len(got[k]) < expect[k]
        if not short:
            break
        if time.monotonic() - t0 > timeout_s:
            raise TimeoutError("CQ wait: " + ", ".join(f"{len(got[k])}/{expect.get(k, 0)}" for k in cqs))
    time.sleep(0.02)
    for k, cq in cqs.items():                 # nothing more may arrive
        got[k] += cq.poll(32)


def soak_seeds(default: int) -> int:
    """How many seeds a test runs: ``RN_RC_SOAK`` raises it for a soak (off by default)."""
    return int(os.environ.get("RN_RC_SOAK", default))


def replay_seed() -> Optional[int]:
    s = os.environ.get("RN_RC_SEED")
    return int(s) if s else None


# ---------------------------------------------------------------------------------------------------------------- wires
class _WireBase:
    """What :func:`run_program` needs from a wire: ``setup`` (buffers, MRs, QPs), ``post_recv`` returning the token the
    receive's completion carries, ``run`` (post, then collect), ``finish`` (final bytes and counters)."""
    host_native_atomics = True

    def _qp_ctx(self, prog, qi):
        return 0

    def setup(self, prog: Program):
        import rocnrdma_b200.wire as W
        self.prog, self.bufs, self.mrs, self.qps = prog, {}, {}, []
        for name, b in prog.bufs.items():
            self.bufs[name] = self.alloc(b)
        owner_side = {}
        for qi, qp in enumerate(prog.qps):
            for name in prog.mrs:
                if name.startswith(f"q{qi}."):
                    owner_side[name] = (qi, qp.peer)
        for name, m in prog.mrs.items():
            qi, peer = owner_side.get(name, (0, prog.qps[0].peer))
            ctx = self.ctxs[self._qp_ctx(prog, qi if m.side == "local" else peer)]
            self.mrs[name] = ctx.reg_mr(self.bufs[m.buf], nbytes=m.n, access=m.access, offset=m.off)
        cqs = {}
        for qi, qp in enumerate(prog.qps):
            ctx = self.ctxs[self._qp_ctx(prog, qi)]
            scq = ctx.create_cq(512, self.cq_mem)
            rcq = scq if prog.cfg.get("shared_cq") else ctx.create_cq(512, self.cq_mem)
            self.qps.append(ctx.create_qp(scq, rcq, 256, 256, self.sq_mem, **self.qp_kw))
            cqs[qi] = (scq, rcq)
        for qi, qp in enumerate(prog.qps):
            if qp.peer == qi:
                self.qps[qi].connect()
            elif qp.peer > qi:
                self.qps[qi].connect(self.qps[qp.peer])
        self.n_recv = [0] * len(self.qps)
        return W

    def close(self):
        """Release everything the program allocated, now.  A context and its MRs reference each other, so without this
        the buffers would live until the cycle collector runs, holding caching-allocator segments that later tests
        expect ``empty_cache`` to return to the driver."""
        for mr in getattr(self, "mrs", {}).values():
            mr.dereg()
        for c in self.ctxs:
            c.close()
            c._mrs.clear()
        self.ctxs, self.mrs, self.bufs, self.qps = [], {}, {}, []
        gc.collect()
        if getattr(self, "device", None) is not None:
            import torch
            torch.cuda.synchronize(self.device)
            torch.cuda.empty_cache()


class VerbsWire(_WireBase):
    """The mock ConnectX through the verbs backend: two mock NICs (connected pairs span them), host-posted QPs.  Data
    buffers are host DRAM (``device=None``) or HBM of GPU ``device`` (the NIC's DMA is then cuMemcpyAsync)."""
    qp_kw = {}

    def __init__(self, device=None):
        import rocnrdma_b200 as rn
        import rocnrdma_b200.wire as W
        self.device = device
        self.cq_mem = self.sq_mem = W.MEM_HOST_PINNED
        self.ctxs = [rn.Context(device=device, wire="verbs", nic=0), rn.Context(device=device, wire="verbs", nic=1)]
        self._lib = self.ctxs[0]._lib

    def _qp_ctx(self, prog, qi):
        return qi % 2 if prog.cfg.get("pairs") else 0

    def alloc(self, b: Buf):
        if self.device is None:
            a = b.init.copy()
            assert a.ctypes.data % 16 == 0
            return a
        import torch
        t = torch.from_numpy(b.init.copy()).to(f"cuda:{self.device}")
        assert t.data_ptr() % 16 == 0
        return t

    def post_recv(self, qp, mr, off, n):
        import ctypes as C
        wr = C.c_uint64()
        rc = self._lib.rn_verbs_post_recv(qp._vq, mr.addr + off, mr.lkey, n, C.byref(wr))
        assert rc == 0, self._lib.rn_verbs_why()
        return wr.value

    def run(self, post_all, collect):
        if self.prog.rnr:
            self._lib.rn_verbs_mock_set_rnr_timeout_ms(50)
        try:
            post_all()
            collect()
        finally:
            self._lib.rn_verbs_mock_set_rnr_timeout_ms(500)

    def finish(self, prog):
        if self.device is not None:
            import torch
            torch.cuda.synchronize(self.device)
        mem = {k: (v.copy() if self.device is None else v.cpu().numpy()) for k, v in self.bufs.items()}
        return {"mem": mem, "counters": [q.counters() for q in self.qps]}


class SoftHcaWire(_WireBase):
    """The software HCA: one context on GPU ``device``, host-posted QPs, the engine on ``ctas`` SMs.  ``oneshot``: every
    WR is posted first and ``engine_run_oneshot`` drains them (claims are batches parsed by one warp); otherwise the
    engine is resident while the host posts (claims are mostly single)."""

    def __init__(self, device=0, ctas=32, chunk_bytes=512 << 10, queue_mem="host", oneshot=False):
        import rocnrdma_b200 as rn
        import rocnrdma_b200.wire as W
        self.device, self.ctas, self.oneshot = device, ctas, oneshot
        self.cq_mem = self.sq_mem = W.MEM_HOST_PINNED if queue_mem == "host" else W.MEM_DEVICE
        self.qp_kw = {"chunk_bytes": chunk_bytes}
        self.ctxs = [rn.Context(device=device)]
        self.host_native_atomics = self.ctxs[0].host_native_atomics

    def alloc(self, b: Buf):
        import torch
        t = torch.from_numpy(b.init.copy())
        t = t.pin_memory() if b.mem == "host" else t.to(f"cuda:{self.device}")
        assert t.data_ptr() % 16 == 0
        return t

    def post_recv(self, qp, mr, off, n):
        qp.post_recv(mr, n, off=off)
        k = self.qps.index(qp)
        self.n_recv[k] += 1
        return self.n_recv[k] - 1

    def run(self, post_all, collect):
        import torch
        ctx = self.ctxs[0]
        torch.cuda.synchronize(self.device)
        if self.oneshot:
            post_all()
            ctx.engine_run_oneshot(ctas=self.ctas)
            collect()
            return
        ctx.engine_start(ctas=self.ctas, idle_timeout_ms=5000, rnr_timeout_ms=50 if self.prog.rnr else 500)
        try:
            post_all()
            collect()
        finally:
            ctx.engine_stop()

    def finish(self, prog):
        import torch
        torch.cuda.synchronize(self.device)
        st = self.ctxs[0].engine_stats()
        assert st["fatal"] == 0 and st["running_ctas"] == 0, st
        mem = {k: v.cpu().numpy() for k, v in self.bufs.items()}
        return {"mem": mem, "counters": [q.counters() for q in self.qps], "bulk_chunks": st["n_bulk_chunks"]}


def check_seed(seed, cfg, make_wire, timeout_s=30.0):
    """Generate the program for (seed, cfg), run it on a fresh wire, compare with the model."""
    prog = generate(seed, cfg)
    wire = make_wire()
    try:
        return prog, run_program(prog, wire, timeout_s)
    finally:
        wire.close()
