"""Scatter-gather work requests against the RC reference model on one H100 (tests/rc_sgl_model.py): the hand-worked
programs of tests/test_rc_sgl.py -- including a hand-built two-segment WQE with a zero-length segment -- and random
programs with list WRs spliced in (``cfg["sgl"]``), on the software HCA across engine CTAs, chunk sizes, queue and data
memory and one-shot or live engines, and on the mock ConnectX with its data in HBM.  Besides bytes, completions and QP
state, every softhca run checks that the engine moved exactly the bulk chunks the model predicts for lists cut per
entry.  ``RN_RC_SEED=<n>`` replays one seed; ``RN_RC_SOAK=<n>`` runs n seeds per config."""
import pytest

import rc_model as M
import rc_sgl_model as S
from rc_sgl_model import GWR
from test_rc_sgl import DIRECTED, _prog

pytestmark = pytest.mark.gpu

K = 1 << 10
# (ctas, chunk_bytes, queue memory, data memory, oneshot)
CONFIGS = [
    (1, 16 * K, "host", "dev", False),
    (3, 20 * K + 16, "dev", "dev", True),
    (32, 64 * K, "host", "host", False),
    (32, 512 * K, "dev", "dev", False),
    (3, 512 * K, "host", "dev", False),
    (32, 16 * K, "dev", "host", True),
]


def _seeds(n, base):
    s = M.replay_seed()
    return [s] if s is not None else [base + i for i in range(M.soak_seeds(n))]


@pytest.mark.parametrize("name", sorted(DIRECTED))
@pytest.mark.parametrize("ctas", [1, 32])
def test_softhca_runs_directed_programs(name, ctas):
    wrs, recvs = DIRECTED[name]
    p = _prog([GWR(**vars(w)) for w in wrs], recvs, {"wire": "softhca", "ctas": ctas, "max_msg": M.MAX_MSG})
    wire = M.SoftHcaWire(0, ctas, 1 << 16, "host", False)
    try:
        S.run_program(p, wire)
    finally:
        wire.close()


@pytest.mark.parametrize("ctas,chunk,qmem,dmem,oneshot", CONFIGS,
                         ids=[f"c{c}-k{k // K}-q{q}-d{d}-{'oneshot' if o else 'live'}" for c, k, q, d, o in CONFIGS])
def test_softhca_matches_the_model_on_sgl_programs(ctas, chunk, qmem, dmem, oneshot):
    cfg = {"wire": "softhca", "max_wrs": 150, "max_len": 4 << 20, "big_budget": 12 << 20, "ctas": ctas, "chunk_bytes": chunk,
           "data_mem": dmem, "allow_rnr": not oneshot, "max_msg": M.MAX_MSG, "sgl": True}
    for seed in _seeds(4, 7000 + 100 * CONFIGS.index((ctas, chunk, qmem, dmem, oneshot))):
        S.check_seed(seed, cfg, lambda: M.SoftHcaWire(0, ctas, chunk, qmem, oneshot))


def test_mock_connectx_matches_the_model_on_sgl_programs_in_hbm():
    cfg = {"wire": "verbs", "max_wrs": 100, "max_len": 1 << 20, "big_budget": 4 << 20, "allow_rnr": True, "max_msg": M.MAX_MSG,
           "sgl": True}
    for seed in _seeds(6, 60_000):
        S.check_seed(seed, cfg, lambda: M.VerbsWire(device=0))
