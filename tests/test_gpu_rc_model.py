"""Both wires against the RC reference model (tests/rc_model.py) on one H100: random programs of WRITE, READ, SEND,
WRITE_IMM, inline, atomics and NOP, unsignaled runs, one fault in some programs, on 1-4 QPs.

The software HCA runs a covering set of configs: engine CTAs, the mover's store/load split (RN_ENGINE_STORES_IN_FLIGHT),
the profiled mover, the QP's chunk size, queues and data in device or pinned host memory, and everything pre-posted
before a one-shot engine (batched claims) or posted while the engine runs (single claims).  Besides bytes, completions and
QP state, each run checks that the engine left cleanly and moved exactly the number of bulk chunks the model predicts, so
a program provably went down the copy paths it was generated for.  The mock ConnectX runs the same kind of programs with
its data in HBM.  ``RN_RC_SEED=<n>`` replays one seed; ``RN_RC_SOAK=<n>`` runs n seeds per config."""
import time

import pytest

import rc_model as M

pytestmark = pytest.mark.gpu

K = 1 << 10
# (ctas, stores in flight or "prof", chunk_bytes, queue memory, data memory, oneshot)
CONFIGS = [
    (1, 2, 16 * K, "host", "dev", False),
    (3, 4, 20 * K + 16, "dev", "dev", True),
    (32, 6, 64 * K, "host", "host", False),
    (32, 8, 512 * K, "dev", "dev", False),
    (3, "prof", 64 * K, "host", "dev", True),
    (1, 8, 20 * K + 16, "host", "host", True),
    (32, 2, 16 * K, "dev", "host", True),
    (3, 6, 512 * K, "host", "dev", False),
    (1, 4, 64 * K, "dev", "dev", False),
    (32, 4, 20 * K + 16, "host", "dev", False),
    (3, 2, 512 * K, "host", "host", False),
    (32, "prof", 16 * K, "dev", "dev", True),
]


def _seeds(n, base):
    s = M.replay_seed()
    return [s] if s is not None else [base + i for i in range(M.soak_seeds(n))]


@pytest.mark.parametrize("ctas,sif,chunk,qmem,dmem,oneshot", CONFIGS,
                         ids=[f"c{c}-s{s}-k{k // K}-q{q}-d{d}-{'oneshot' if o else 'live'}" for c, s, k, q, d, o in CONFIGS])
def test_softhca_matches_the_model(monkeypatch, ctas, sif, chunk, qmem, dmem, oneshot):
    if sif == "prof":
        monkeypatch.setenv("RN_ENGINE_PROFILE", "1")
        monkeypatch.delenv("RN_ENGINE_STORES_IN_FLIGHT", raising=False)
    else:
        monkeypatch.delenv("RN_ENGINE_PROFILE", raising=False)
        monkeypatch.setenv("RN_ENGINE_STORES_IN_FLIGHT", str(sif))
    cfg = {"wire": "softhca", "max_wrs": 150, "max_len": 4 << 20, "big_budget": 12 << 20, "ctas": ctas,
           "chunk_bytes": chunk, "data_mem": dmem, "allow_rnr": not oneshot}
    t0 = time.monotonic()
    bulk = 0
    for seed in _seeds(4, 1000 * CONFIGS.index((ctas, sif, chunk, qmem, dmem, oneshot))):
        _, model = M.check_seed(seed, cfg, lambda: M.SoftHcaWire(0, ctas, chunk, qmem, oneshot))
        bulk += sum(o.bulk_chunks for o in model.qps)
    print(f"{ctas} CTAs, sif {sif}, chunk {chunk}: {bulk} bulk chunks, {time.monotonic() - t0:.1f} s")


def test_mock_connectx_matches_the_model_on_hbm():
    cfg = {"wire": "verbs", "max_wrs": 100, "max_len": 1 << 20, "big_budget": 4 << 20, "allow_rnr": True}
    for seed in _seeds(6, 50_000):
        M.check_seed(seed, cfg, lambda: M.VerbsWire(device=0))
