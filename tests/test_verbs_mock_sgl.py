"""Scatter-gather lists on the verbs wire, against the in-tree mock ConnectX (two ports, host memory, CPU only):
ibv_post_send with two SGEs for every opcode that takes a list, the provider's refusals (more SGEs than granted, an
atomic with two, inline past 28 bytes), zero-length entries dropped, two inline SGEs concatenated, and the granted
max_send_sge."""
import ctypes as C

import numpy as np
import pytest

import rocnrdma_b200 as rn
from rocnrdma_b200 import _native as N, wire as W
from rocnrdma_b200.api import MemoryRegion

H = W.MEM_HOST_PINNED
EINVAL = 22


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


def _bufs(c, *sizes, seed=1):
    rng = np.random.default_rng(seed)
    arrs = [rng.integers(0, 256, n, dtype=np.uint8) for n in sizes]
    return arrs, [c.reg_mr(a) for a in arrs]


def _raw(lib, q, op, entries, raddr=0, rkey=0, flags=1):
    arr = (N.RnSge * max(len(entries), 1))()
    for i, (a, k, n) in enumerate(entries):
        arr[i].addr, arr[i].lkey, arr[i].bytes = a, k, n
    wr = C.c_uint64()
    return lib.rn_verbs_post_sg(q._vq, op, arr, len(entries), raddr, rkey, flags, 0, C.byref(wr))


def test_max_send_sge_is_granted_and_reported(pair):
    c0, _, q0, _ = pair
    assert c0._lib.rn_verbs_qp_max_sge(q0._vq) == 2
    assert q0.max_send_sge == 2


@pytest.mark.parametrize("imm", [None, 0xBEEF])
def test_gather_write_lands_concatenated(pair, imm):
    c0, c1, q0, q1 = pair
    (a, b), (ma, mb) = _bufs(c0, 300, 200)
    dst = np.zeros(600, dtype=np.uint8)
    md = c1.reg_mr(dst)
    if imm is not None:
        rbuf = np.zeros(8, dtype=np.uint8)
        q1.post_recv(c1.reg_mr(rbuf))
    q0.post_write_sg([(ma, 10, 100), (mb, 7, 60)], md, dst_off=50, imm=imm)
    wc = q0.scq.wait(1)[0]
    assert wc.status == "OK" and wc.byte_cnt == 160
    assert bytes(dst[50:150]) == bytes(a[10:110]) and bytes(dst[150:210]) == bytes(b[7:67])
    assert not dst[:50].any() and not dst[210:].any()
    if imm is not None:
        rwc = q1.rcq.wait(1)[0]
        assert rwc.status == "OK" and rwc.imm == imm and rwc.byte_cnt == 160


def test_scatter_read_splits_the_remote_range(pair):
    c0, c1, q0, _ = pair
    (src,), (ms,) = _bufs(c1, 512, seed=2)
    x, y = np.zeros(128, dtype=np.uint8), np.zeros(128, dtype=np.uint8)
    mx, my = c0.reg_mr(x), c0.reg_mr(y)
    q0.post_read_sg([(mx, 3, 40), (my, 9, 90)], ms, remote_off=100)
    wc = q0.scq.wait(1)[0]
    assert wc.status == "OK" and wc.byte_cnt == 130
    assert bytes(x[3:43]) == bytes(src[100:140]) and bytes(y[9:99]) == bytes(src[140:230])
    assert not x[:3].any() and not x[43:].any() and not y[:9].any() and not y[99:].any()


@pytest.mark.parametrize("imm", [None, 0x5150])
def test_gather_send_lands_in_one_receive(pair, imm):
    c0, c1, q0, q1 = pair
    (a, b), (ma, mb) = _bufs(c0, 64, 64, seed=3)
    rbuf = np.zeros(128, dtype=np.uint8)
    q1.post_recv(c1.reg_mr(rbuf))
    q0.post_send_sg([(ma, 0, 33), (mb, 1, 20)], imm=imm)
    assert q0.scq.wait(1)[0].byte_cnt == 53
    rwc = q1.rcq.wait(1)[0]
    assert rwc.status == "OK" and rwc.byte_cnt == 53 and (imm is None or rwc.imm == imm)
    assert bytes(rbuf[:33]) == bytes(a[:33]) and bytes(rbuf[33:53]) == bytes(b[1:21]) and not rbuf[53:].any()


def test_three_sges_fail_with_einval_naming_the_work_request(pair):
    c0, c1, q0, _ = pair
    lib = c0._lib
    (a,), (ma,) = _bufs(c0, 64)
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    e = [(ma.addr, ma.lkey, 8)] * 3
    assert _raw(lib, q0, W.OP_RDMA_WRITE, e, md.addr, md.rkey) == -EINVAL
    assert "bad_wr is this work request" in lib.rn_verbs_why().decode()
    with pytest.raises(ValueError):
        q0.post_write_sg([(ma, 0, 8)] * 3, md)
    with pytest.raises(ValueError):
        q0.post_write_sg([], md)
    with pytest.raises(ValueError):
        q0.post_write_sg([(ma, 0, 1 << 32)], md)
    q0.post_write_sg([(ma, 0, 4), (ma, 4, 4)], md)          # nothing was queued by the refused posts
    wc = q0.scq.wait(1)[0]
    assert wc.status == "OK" and wc.byte_cnt == 8 and bytes(dst[:8]) == bytes(a[:8])


def test_atomic_with_two_sges_fails_with_einval(pair):
    c0, c1, q0, _ = pair
    lib = c0._lib
    f = np.zeros(16, dtype=np.uint8)
    mf = c0.reg_mr(f)
    t = np.zeros(8, dtype=np.uint64)
    mt = c1.reg_mr(t, access=W.ACC_ALL)
    for op in (W.OP_ATOMIC_FA, W.OP_ATOMIC_CS):
        assert _raw(lib, q0, op, [(mf.addr, mf.lkey, 8), (mf.addr + 8, mf.lkey, 8)], mt.addr, mt.rkey) == -EINVAL
        assert "bad_wr is this work request" in lib.rn_verbs_why().decode()


def test_zero_length_entries_are_dropped(pair):
    c0, c1, q0, _ = pair
    lib = c0._lib
    (a, b), (ma, mb) = _bufs(c0, 64, 64, seed=4)
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    # the empty entry's key is not even valid: dropped at post time, it is never looked at
    assert _raw(lib, q0, W.OP_RDMA_WRITE, [(0xDEAD0000, 0xFFFFFF00, 0), (mb.addr + 5, mb.lkey, 11)], md.addr + 2, md.rkey) == 0
    q0.post_write_sg([(ma, 0, 6), (mb, 0, 0)], md, dst_off=20)
    wcs = q0.scq.wait(2)
    assert [w.status for w in wcs] == ["OK", "OK"] and [w.byte_cnt for w in wcs] == [11, 6]
    assert bytes(dst[2:13]) == bytes(b[5:16]) and bytes(dst[20:26]) == bytes(a[:6])
    assert not dst[:2].any() and not dst[13:20].any() and not dst[26:].any()


def test_two_inline_sges_are_concatenated(pair):
    c0, c1, q0, _ = pair
    lib = c0._lib
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    x, y = C.create_string_buffer(b"0123456789", 10), C.create_string_buffer(b"abcdefghijklmnopqr", 18)
    e = [(C.addressof(x), 0, 10), (C.addressof(y), 0, 18)]
    assert _raw(lib, q0, W.OP_RDMA_WRITE, e, md.addr + 4, md.rkey, flags=1 | 4) == 0
    wc = q0.scq.wait(1)[0]
    assert wc.status == "OK" and wc.byte_cnt == 28
    assert bytes(dst[4:32]) == b"0123456789abcdefghijklmnopqr" and not dst[:4].any() and not dst[32:].any()
    # 29 bytes in two SGEs is past the inline limit
    z = C.create_string_buffer(19)
    assert _raw(lib, q0, W.OP_RDMA_WRITE, [(C.addressof(x), 0, 10), (C.addressof(z), 0, 19)], md.addr, md.rkey,
                flags=1 | 4) == -EINVAL


def test_second_entry_key_error_is_a_local_protection_error(pair):
    c0, c1, q0, _ = pair
    (a,), (ma,) = _bufs(c0, 64)
    dst = np.zeros(64, dtype=np.uint8)
    md = c1.reg_mr(dst)
    bad = MemoryRegion(c0, ma.addr, 64, ma.lkey ^ 0x100, W.ACC_ALL)     # entry 1 under a key nobody registered
    q0.post_write_sg([(ma, 0, 8), (bad, 0, 8)], md)
    wc = q0.scq.wait(1)[0]
    assert wc.status != "OK" and W.SYNDROMES.get(wc.syndrome) == "LOCAL_PROT_ERR"
    assert not dst.any()
