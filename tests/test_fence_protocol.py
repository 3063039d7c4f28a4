"""An interleaving model of the softhca engine's fence gate (engine.cuh: fence_gated, gate_open, the gated ticket in
try_claim's commit and offer scan, and in claim_batch), walked over every interleaving of its actors.

WQE F of a QP carries the fence; WQEs 0..F-1 before it each move one chunk, F moves ``m`` chunks.  Every access to a
shared word is one atomic step.  Actors:

* the committer of F reads the retire word and, with the gate open, moves chunk 0 itself (a single claim; a batch claim
  arms a drawable ticket), else arms a GATED ticket; then it publishes the commit (parse_seq);
* the movers write the earlier WQEs' chunks; the retirer advances the retire word over finished WQEs, in order;
* helpers scan: see the commit, read F's ticket, stop the offer at a gated ticket and re-check the gate (open: one CAS
  resets the chunk counter), draw chunks (fetch-add), and move the offer past a ticket that looks fully drawn.

With one engine CTA the committer, the retirer and the helper are one thread that never blocks (its own mover is a
separate actor, as on the GPU); with several they are separate CTAs.  Checked in every reachable state: F's chunks are
drawn at most once each and never before the retire word reaches F; and from every reachable state the run can still
draw all of them (nothing is lost).  The negative controls drop the gate re-check or the offer stop; each must fail.
"""
import itertools

import pytest

OPEN, GATED = "open", "gated"


def _explore(F, m, ctas, batch, recheck=True, offer_stop=True):
    """Returns (reachable states, violations, states from which F can no longer be fully drawn)."""
    # shared: rw (retire word), fin (earlier WQEs written), ticket (None | (kind, next)), committed, offer, drawn, bad
    # actors' program counters: committer, helper(s); the one-CTA case runs committer, retirer and helper in one thread
    init = dict(rw=0, fin=(False,) * F, ticket=None, committed=False, offer=F, drawn=0, bad=False,
                cpc=0, cr=None, hpc=(0,) * (1 if ctas == 1 else 2), ht=(None,) * (1 if ctas == 1 else 2))

    def freeze(s):
        return tuple(sorted(s.items()))

    def draw(s):
        s["drawn"] += 1
        if s["rw"] != F:
            s["bad"] = True          # a chunk of F moved before every earlier WQE finished

    def committer_step(s):
        pc = s["cpc"]
        if pc == 0:
            s["cr"] = s["rw"]; s["cpc"] = 1
        elif pc == 1:
            if s["cr"] == F:
                if batch:
                    s["ticket"] = (OPEN, 0)
                else:
                    draw(s)                             # the claimer moves chunk 0 itself
                    s["ticket"] = (OPEN, 1) if m > 1 else None
            else:
                s["ticket"] = (GATED, 0)
            s["cpc"] = 2
        elif pc == 2:
            s["committed"] = True; s["cpc"] = 3
        return pc < 3

    def retire_step(s):
        if s["rw"] < F and s["fin"][s["rw"]]:
            s["rw"] += 1
            return True
        return False

    def helper_step(s, k):
        pcs, hts = list(s["hpc"]), list(s["ht"])
        pc = pcs[k]
        if pc == 0:                                     # scan: is F committed and still at or after the offer?
            if s["committed"] and s["offer"] <= F:
                pcs[k] = 1
        elif pc == 1:                                   # load F's ticket
            t = s["ticket"]
            hts[k] = t
            if t is None:                               # single chunk taken by its claimer: looks drawn
                s["offer"] = max(s["offer"], F + 1); pcs[k] = 0
            elif t[0] == GATED:
                if not offer_stop:
                    s["offer"] = max(s["offer"], F + 1)  # avail == 0 counts toward the lead
                pcs[k] = 2 if recheck else 0
            elif t[1] < m:
                pcs[k] = 3
            else:
                s["offer"] = max(s["offer"], F + 1); pcs[k] = 0
        elif pc == 2:                                   # gate re-check, then CAS open
            if s["rw"] == F:
                if s["ticket"] == hts[k]:
                    s["ticket"] = (OPEN, 0)
                pcs[k] = 3
            else:
                pcs[k] = 0
        elif pc == 3:                                   # draw: fetch-add on the chunk counter
            t = s["ticket"]
            if t[0] == OPEN:
                s["ticket"] = (OPEN, t[1] + 1)
                if t[1] < m:
                    draw(s)
            pcs[k] = 0
        s["hpc"], s["ht"] = tuple(pcs), tuple(hts)
        return True

    def moves(s):
        """(label, successor) for every enabled step."""
        out = []
        for e in range(F):
            if not s["fin"][e]:
                n = dict(s); n["fin"] = s["fin"][:e] + (True,) + s["fin"][e + 1:]
                out.append(n)
        if ctas == 1:
            # one thread: commit first, then loop { retire what its mover finished; scan }
            n = dict(s)
            if committer_step(n):
                out.append(n)
            else:
                n = dict(s)
                if retire_step(n):
                    out.append(n)
                n = dict(s)
                helper_step(n, 0)
                out.append(n)
        else:
            n = dict(s)
            if committer_step(n):
                out.append(n)
            n = dict(s)
            if retire_step(n):
                out.append(n)
            for k in range(len(s["hpc"])):
                n = dict(s)
                helper_step(n, k)
                out.append(n)
        return out

    seen, edges, stack = {freeze(init): init}, {}, [init]
    while stack:
        s = stack.pop()
        key = freeze(s)
        edges[key] = []
        for n in moves(s):
            nk = freeze(n)
            edges[key].append(nk)
            if nk not in seen:
                seen[nk] = n
                stack.append(n)
    violations = [s for s in seen.values() if s["bad"] or s["drawn"] > m]
    # liveness: every state must still reach one where all of F's chunks are drawn
    good = {k for k, s in seen.items() if s["drawn"] == m}
    rev = {}
    for k, succ in edges.items():
        for n in succ:
            rev.setdefault(n, []).append(k)
    live, work = set(good), list(good)
    while work:
        k = work.pop()
        for p in rev.get(k, ()):
            if p not in live:
                live.add(p)
                work.append(p)
    stuck = [seen[k] for k in seen if k not in live]
    return seen, violations, stuck


CASES = list(itertools.product([1, 2], [1, 2], [1, 3], [False, True]))   # earlier WQEs, chunks of F, CTAs, batch


@pytest.mark.parametrize("F,m,ctas,batch", CASES, ids=[f"F{f}-m{m}-cta{c}-{'batch' if b else 'single'}" for f, m, c, b in CASES])
def test_gate_draws_every_chunk_once_and_only_after_the_retirer(F, m, ctas, batch):
    seen, violations, stuck = _explore(F, m, ctas, batch)
    assert not violations, violations[:2]
    assert not stuck, stuck[:2]
    # the walk reached both a closed gate and a gate opened by a helper
    assert any(s["ticket"] is not None and s["ticket"][0] == GATED for s in seen.values())
    assert any(s["drawn"] == m for s in seen.values())


@pytest.mark.parametrize("ctas", [1, 3])
def test_without_the_recheck_a_gated_wqe_is_lost(ctas):
    _, violations, stuck = _explore(2, 1, ctas, batch=True, recheck=False)
    assert not violations and stuck


@pytest.mark.parametrize("ctas", [1, 3])
def test_without_the_offer_stop_a_gated_wqe_is_lost(ctas):
    _, violations, stuck = _explore(2, 2, ctas, batch=True, offer_stop=False)
    assert not violations and stuck
