"""Fenced work requests on top of the RC reference model (tests/rc_model.py): a WR type with the fence flag, a program
generator that splices dependent pairs whose later WR is fenced into rc_model's random programs, and wires that post
each WR with its flag.

The contract (DESIGN.md section 3.1): a fenced WR sees every effect of the earlier WRs of its QP.  The model executes
every QP in order, so it needs nothing more.  What changes is which programs are legal: without the fence, WRs whose
bytes overlap are unordered on the software HCA, so only a fenced WR may touch bytes an earlier WR wrote, or write
bytes an earlier WR read.

``generate(seed, cfg)`` is ``rc_model.generate`` when ``cfg["fences"]`` is not set.  With it, each QP's program gets
2-5 of these pairs, each on bytes of its own (appended to the QP's DST buffer, after everything rc_model placed there):

* write_read: WRITE a region, then a fenced READ of it back into a fresh one;
* write_write: WRITE a region, then a fenced WRITE of other bytes over part of it;
* read_write / read_send: READ into a fresh region, then a fenced WRITE / SEND sourced from it;
* write_atomic: WRITE 8 bytes to an atomic word nothing else touches, then a fenced FETCH_AND_ADD / COMPARE_AND_SWAP on it.

Lengths run from one byte to several engine chunks, aligned and not, so both the TMA and the generic copy are ordered.
The pairs draw from a random stream of their own and are placed in front of random WRs, never after a QP's last WR (an
RNR program still ends with its RNR).
"""
from dataclasses import dataclass

import numpy as np

import rc_model as M
from rc_model import MR, WR, Recv

PAIRS = ("write_read", "write_write", "read_write", "read_send", "write_atomic")


@dataclass
class FWR(WR):
    fence: bool = False       # IBV_SEND_FENCE: starts after every earlier WR of the QP finished


def fenced(w) -> bool:
    return bool(getattr(w, "fence", False))


class _Tail:
    """Bump allocator over bytes appended to a buffer: 16-byte frames plus a gap, so regions never overlap."""

    def __init__(self, start):
        self.top = start + 64

    def take(self, n, mis=0, gap=48):
        start = (self.top + 15) // 16 * 16 + mis
        self.top = start + n + gap
        return start


def _pairs_for(seed, qi, cfg, prog):
    p = f"q{qi}."
    qp = prog.qps[qi]
    rng = np.random.default_rng([seed, qi, 0xFE4CE])
    g = M.granule(cfg)
    src_n = prog.bufs[p + "SRC"].init.size
    cap = max(1, min(cfg["max_len"], 3 * g + 48, src_n - 4096))
    lens = [x for x in (1, 17, 64, 4096, 4097, 16384, 16400, g - 16, g, g + 48, 3 * g + 48) if 1 <= x <= cap]
    atom = prog.bufs[p + "ATOM"].init.size
    used = set()                # atomic words any WR of the QP touches
    for w in qp.wrs:
        if w.rmr and prog.mrs[w.rmr].buf == p + "ATOM":
            m = prog.mrs[w.rmr]
            used.update(range((m.off + w.roff) // 8, (m.off + w.roff + max(w.n, 1) - 1) // 8 + 1))
    free = [k for k in range((atom - 64) // 8) if k not in used]
    dst = _Tail(prog.bufs[p + "DST"].init.size)
    mrs = {}

    def mr(kind, off, n, side):
        name = f"{p}f{len(mrs)}.{kind}"
        mrs[name] = MR(name, p + "DST", off, n, M.ACC_ALL, side)
        return name

    def src_off(n):            # n <= src_n - 4096, so any of the first 128 frames holds it
        return 16 * int(rng.integers(0, 128)) + int(rng.choice(M.MIS))

    new = []                    # (WR, its receive or None), two per pair
    for _ in range(int(rng.integers(2, 6))):
        kind = PAIRS[int(rng.integers(0, len(PAIRS)))]
        n = int(rng.choice(lens))
        mis = int(rng.choice(M.MIS))
        if kind == "write_atomic":
            if not free:
                continue
            word = free.pop(int(rng.integers(0, len(free))))
            a = FWR("WRITE", 8, p + "src_l", 16 * int(rng.integers(0, 64)), p + "atom", 8 * word)
            b = FWR(str(rng.choice(["FA", "CS"])), 8, mr("ffetch", dst.take(8), 8, "local"), 0, p + "atom", 8 * word,
                    fence=True, add=int(rng.integers(0, 2**63)) * 2 + 1, cas_hit=bool(rng.integers(0, 2)))
            new += [(a, None), (b, None)]
        elif kind in ("write_read", "write_write"):
            span = n if kind == "write_read" else n + int(rng.integers(0, 2)) * int(rng.choice(lens))
            region = mr("fmid", dst.take(span, mis), span, "remote")
            a = FWR("WRITE", n, p + "src_l", src_off(n), region, 0)
            if kind == "write_read":
                b = FWR("READ", n, mr("fback", dst.take(n, int(rng.choice(M.MIS))), n, "local"), 0, region, 0, fence=True)
            else:
                m = int(rng.choice([x for x in lens if x <= span]))
                off = int(rng.integers(0, min(n - 1, span - m) + 1))     # starts inside the first WRITE's bytes
                b = FWR("WRITE", m, p + "src_l", src_off(m), region, off, fence=True)
            new += [(a, None), (b, None)]
        else:
            mid = mr("fmid", dst.take(n, mis), n, "local")
            a = FWR("READ", n, mid, 0, p + "src_r", src_off(n))
            if kind == "read_write":
                b = FWR("WRITE", n, mid, 0, mr("fout", dst.take(n, int(rng.choice(M.MIS))), n, "remote"), 0, fence=True)
                new += [(a, None), (b, None)]
            else:
                rv = mr("frcv", dst.take(n, int(rng.choice(M.MIS))), n, "remote")
                new += [(a, None), (FWR("SEND", n, mid, 0, fence=True), Recv(rv, 0, n))]
    for w, _ in new:
        w.signaled = bool(rng.integers(0, 4)) or w.fence
    last = len(qp.wrs) - 1
    at = sorted(int(x) for x in rng.integers(0, max(last, 0) + 1, len(new) // 2))
    return new, at, mrs, dst.top + 64


def _splice(prog, qi, new, at):
    """Insert pair j in front of original WR at[j]; receives keep the order of the WRs that consume them."""
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
            for x, r in new[2 * j:2 * j + 2]:
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
    if not cfg.get("fences"):
        return prog
    for qi in range(len(prog.qps)):
        new, at, mrs, dst_n = _pairs_for(seed, qi, prog.cfg, prog)
        b = prog.bufs[f"q{qi}.DST"]
        tail = np.random.default_rng([seed, qi, 0xD57]).integers(0, 256, dst_n - b.init.size, dtype=np.uint8)
        b.init = np.concatenate([b.init, tail])
        prog.mrs.update(mrs)
        _splice(prog, qi, new, at)
    M.run_model(prog, host_native_atomics=prog.cfg.get("host_native_atomics", True), resolve_cas=True)
    for qp in prog.qps:
        for w in qp.wrs:
            if w.op == "CS" and w.compare is None:       # never executed (flushed): any value
                w.compare = 0
    return prog


# ---------------------------------------------------------------------------------------------------------------- wires
class _FenceQp:
    """A queue pair that posts the WRs of one program QP in order, each with that WR's fence flag.  rc_model.run_program
    makes exactly one post call per WR, in program order, so the n-th call belongs to WR n.  Everything else is the QP's."""
    _POSTS = ("post_raw", "post_write", "post_read", "post_send", "post_write_inline", "post_send_inline",
              "post_fetch_add", "post_cmp_swap")

    def __init__(self, qp, wrs):
        self._qp, self._wrs, self._next = qp, wrs, 0

    def __getattr__(self, name):
        attr = getattr(self._qp, name)
        if name not in self._POSTS:
            return attr

        def post(*a, **kw):
            w = self._wrs[self._next]
            self._next += 1
            return attr(*a, fence=fenced(w), **kw)
        return post


def with_fences(wire):
    """Make ``wire`` (an rc_model wire) post every WR with its fence flag."""
    setup = wire.setup

    def fenced_setup(prog):
        W = setup(prog)
        wire.qps = [_FenceQp(q, prog.qps[i].wrs) for i, q in enumerate(wire.qps)]
        return W
    wire.setup = fenced_setup
    return wire


def check_seed(seed, cfg, make_wire, timeout_s=30.0):
    """rc_model.check_seed for fenced programs: generate, run on a fresh wire that posts the flags, compare."""
    prog = generate(seed, cfg)
    wire = with_fences(make_wire())
    try:
        return prog, M.run_program(prog, wire, timeout_s)
    finally:
        wire.close()
