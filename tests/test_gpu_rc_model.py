"""Both wires against the RC reference model (tests/rc_model.py) on one H100: random programs of WRITE, READ, SEND,
WRITE_IMM, inline, atomics and NOP, unsignaled runs, one fault in some programs, on 1-4 QPs.

The software HCA runs a covering set of configs: engine CTAs, the plain or the profiled mover, the QP's chunk size,
queues and data in device or pinned host memory, and everything pre-posted before a one-shot engine (batched claims) or
posted while the engine runs (single claims).  Besides bytes, completions and QP state, each run checks that the engine
left cleanly and moved exactly the number of bulk chunks the model predicts, so a program provably went down the copy
paths it was generated for.  Every config also builds WRs longer than the maximum message length (``cfg["max_msg"]``),
which must fail before any key is looked at.  The mock ConnectX runs the same kind of programs with its data in HBM.  ``RN_RC_SEED=<n>`` replays one seed; ``RN_RC_SOAK=<n>`` runs n seeds per config."""
import time

import pytest

import rc_model as M

pytestmark = pytest.mark.gpu

K = 1 << 10
# (ctas, profiled mover, chunk_bytes, queue memory, data memory, oneshot)
CONFIGS = [
    (1, False, 16 * K, "host", "dev", False),
    (3, False, 20 * K + 16, "dev", "dev", True),
    (32, False, 64 * K, "host", "host", False),
    (32, False, 512 * K, "dev", "dev", False),
    (3, True, 64 * K, "host", "dev", True),
    (1, False, 20 * K + 16, "host", "host", True),
    (32, False, 16 * K, "dev", "host", True),
    (3, False, 512 * K, "host", "dev", False),
    (1, False, 64 * K, "dev", "dev", False),
    (32, False, 20 * K + 16, "host", "dev", False),
    (3, False, 512 * K, "host", "host", False),
    (32, True, 16 * K, "dev", "dev", True),
]


def _seeds(n, base):
    s = M.replay_seed()
    return [s] if s is not None else [base + i for i in range(M.soak_seeds(n))]


@pytest.mark.parametrize("ctas,prof,chunk,qmem,dmem,oneshot", CONFIGS,
                         ids=[f"c{c}-{'prof-' if p else ''}k{k // K}-q{q}-d{d}-{'oneshot' if o else 'live'}" for c, p, k, q, d, o in CONFIGS])
def test_softhca_matches_the_model(monkeypatch, ctas, prof, chunk, qmem, dmem, oneshot):
    if prof:
        monkeypatch.setenv("RN_ENGINE_PROFILE", "1")
    else:
        monkeypatch.delenv("RN_ENGINE_PROFILE", raising=False)
    cfg = {"wire": "softhca", "max_wrs": 150, "max_len": 4 << 20, "big_budget": 12 << 20, "ctas": ctas,
           "chunk_bytes": chunk, "data_mem": dmem, "allow_rnr": not oneshot, "max_msg": M.MAX_MSG}
    t0 = time.monotonic()
    bulk = 0
    for seed in _seeds(4, 1000 * CONFIGS.index((ctas, prof, chunk, qmem, dmem, oneshot))):
        _, model = M.check_seed(seed, cfg, lambda: M.SoftHcaWire(0, ctas, chunk, qmem, oneshot))
        bulk += sum(o.bulk_chunks for o in model.qps)
    print(f"{ctas} CTAs, {'profiled' if prof else 'plain'} mover, chunk {chunk}: {bulk} bulk chunks, {time.monotonic() - t0:.1f} s")


def test_mock_connectx_matches_the_model_on_hbm():
    cfg = {"wire": "verbs", "max_wrs": 100, "max_len": 1 << 20, "big_budget": 4 << 20, "allow_rnr": True, "max_msg": M.MAX_MSG}
    for seed in _seeds(6, 50_000):
        M.check_seed(seed, cfg, lambda: M.VerbsWire(device=0))
