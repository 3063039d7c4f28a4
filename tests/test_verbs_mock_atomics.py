"""RDMA atomics on the verbs wire, against the in-tree mock ConnectX (two ports, host memory, CPU only): fetch-and-add
and compare-and-swap results, the remote-atomic access check with the flush that follows an error, and alignment."""
import numpy as np
import pytest

import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, wire as W

H = W.MEM_HOST_PINNED


@pytest.fixture
def pair():
    lib = N.load()
    if lib.rn_verbs_available() < 2 or lib.rn_verbs_is_mock() != 1:
        pytest.skip("needs the mock verbs provider with two ports")
    c0, c1 = rn.Context(device=None, wire="verbs", nic=0), rn.Context(device=None, wire="verbs", nic=1)
    q0 = c0.create_qp(c0.create_cq(64, H), c0.create_cq(64, H), 16, 16, H)
    q1 = c1.create_qp(c1.create_cq(64, H), c1.create_cq(64, H), 16, 16, H)
    q0.connect(q1)
    yield c0, c1, q0, q1
    c0.close()
    c1.close()


def test_fetch_add_returns_the_old_value_and_adds(pair):
    c0, c1, q0, _ = pair
    fetch, target = np.zeros(4, dtype=np.uint64), np.array([40, 2 ** 64 - 1, 0, 0], dtype=np.uint64)
    mf, mt = c0.reg_mr(fetch), c1.reg_mr(target)
    q0.post_fetch_add(mf, mt, 2)
    q0.post_fetch_add(mf, mt, 5, local_off=8)
    q0.post_fetch_add(mf, mt, 1, local_off=16, remote_off=8)          # wraps around
    wcs = q0.scq.wait(3)
    assert all(w.status == "OK" and w.byte_cnt == 8 for w in wcs)
    assert list(fetch[:3]) == [40, 42, 2 ** 64 - 1]
    assert list(target[:2]) == [47, 0]


def test_cmp_swap_succeeds_on_match_and_leaves_memory_on_mismatch(pair):
    c0, c1, q0, _ = pair
    fetch, target = np.zeros(2, dtype=np.uint64), np.array([7], dtype=np.uint64)
    mf, mt = c0.reg_mr(fetch), c1.reg_mr(target)
    q0.post_cmp_swap(mf, mt, compare=7, swap=0xABCDEF0123456789)
    assert q0.scq.wait(1)[0].status == "OK"
    assert fetch[0] == 7 and target[0] == 0xABCDEF0123456789
    q0.post_cmp_swap(mf, mt, compare=7, swap=1, local_off=8)
    assert q0.scq.wait(1)[0].status == "OK"
    assert fetch[1] == 0xABCDEF0123456789 and target[0] == 0xABCDEF0123456789


def test_no_remote_atomic_access_is_a_remote_access_error_and_flushes(pair):
    c0, c1, q0, q1 = pair
    fetch, target = np.zeros(2, dtype=np.uint64), np.array([3], dtype=np.uint64)
    mf = c0.reg_mr(fetch)
    mt = c1.reg_mr(target, access=W.ACC_ALL & ~W.ACC_REMOTE_ATOMIC)
    q0.post_fetch_add(mf, mt, 1)
    q0.post_fetch_add(mf, mt, 1, local_off=8)
    wcs = q0.scq.wait(2)
    assert wcs[0].is_error and wcs[0].status == "REMOTE_ACCESS_ERR"
    assert wcs[1].is_error and wcs[1].status == "WR_FLUSH_ERR"
    assert target[0] == 3 and not fetch.any()
    assert q0.state == "ERR"


def test_misaligned_target_is_an_invalid_request(pair):
    c0, c1, q0, _ = pair
    fetch, target = np.zeros(1, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    mf, mt = c0.reg_mr(fetch), c1.reg_mr(target)
    q0.post_fetch_add(mf, mt, 1, remote_off=4)
    wc = q0.scq.wait(1)[0]
    assert wc.is_error and wc.status == "REMOTE_INVAL_REQ_ERR"
    assert not target.any()
