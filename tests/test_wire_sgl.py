"""Two-entry scatter-gather WQEs on the wire: exact bytes from the Python mirror, the native encoder against the mirror,
decode round trips through both decoders, the malformed lists the decoders refuse, zero-length entries collapsing to the
one-entry WQE, per-segment saturation, and the layout against DOCA GPUNetIO's header (csrc/wire/mlx5_wire.h)."""
import ctypes as C
import shutil
import struct
import subprocess
from pathlib import Path

import pytest

from rocnrdma_b200 import wire as W

ROOT = Path(__file__).resolve().parent.parent
RDMA_OPS = (W.OP_RDMA_WRITE, W.OP_RDMA_WRITE_IMM, W.OP_RDMA_READ)
SEND_OPS = (W.OP_SEND, W.OP_SEND_IMM)
E0, E1 = (0x00007F0000001000, 0x00000101, 0x40), (0x00007F0000A00003, 0x00000202, 0x1234)


def _lib():
    from rocnrdma_b200 import _native as N
    return N, N.load()


def _native_build(op, idx, qpn, sges, raddr=0, rkey=0, flags=W.CTRL_CQ_UPDATE, imm=0):
    N, lib = _lib()
    arr = (N.RnSge * len(sges))()
    for i, (a, k, n) in enumerate(sges):
        arr[i].addr, arr[i].lkey, arr[i].bytes = a, k, n
    buf = (C.c_uint8 * 64)()
    lib.rn_wire_build_sg_wqe(buf, op, idx, qpn, arr, len(sges), raddr, rkey, flags, imm)
    return bytes(buf)


def _mirror(op, idx, qpn, sges, raddr=0, rkey=0, flags=W.CTRL_CQ_UPDATE, imm=0):
    if op in SEND_OPS:
        return W.send_sg_wqe(op, idx, qpn, sges, flags, imm)
    return W.rdma_sg_wqe(op, idx, qpn, sges, raddr, rkey, flags, imm)


def _decode_sg(w):
    _, lib = _lib()
    out = (C.c_uint64 * 17)()
    ok = lib.rn_wire_decode_wqe_sg((C.c_uint8 * 64)(*w), out)
    return ok, list(out)


@pytest.mark.parametrize("op", RDMA_OPS)
def test_two_entry_rdma_wqe_bytes(op):
    imm = 0xCAFEF00D if op == W.OP_RDMA_WRITE_IMM else 0
    w = W.rdma_sg_wqe(op, 0x0102, 0x0A0B0C, [E0, E1], raddr=0x7F0000002000, rkey=0x303, imm=imm)
    assert len(w) == 64
    assert w[0:16] == bytes([0x00, 0x01, 0x02, op, 0x0A, 0x0B, 0x0C, 4, 0, 0, 0, 0x08]) + struct.pack(">I", imm)
    assert w[16:32] == bytes.fromhex("00007f0000002000" "00000303" "00000000")
    assert w[32:48] == bytes.fromhex("00000040" "00000101" "00007f0000001000")
    assert w[48:64] == bytes.fromhex("00001234" "00000202" "00007f0000a00003")
    assert _native_build(op, 0x0102, 0x0A0B0C, [E0, E1], 0x7F0000002000, 0x303, W.CTRL_CQ_UPDATE, imm) == w


@pytest.mark.parametrize("op", SEND_OPS)
def test_two_entry_send_wqe_bytes(op):
    w = W.send_sg_wqe(op, 5, 0x100, [E0, E1], fm_ce_se=0, imm=0x01020304)
    assert w[0:16] == bytes([0, 0, 5, op, 0, 1, 0, 3, 0, 0, 0, 0, 1, 2, 3, 4])
    assert w[16:32] == bytes.fromhex("00000040" "00000101" "00007f0000001000")
    assert w[32:48] == bytes.fromhex("00001234" "00000202" "00007f0000a00003")
    assert w[48:] == bytes(16)
    assert _native_build(op, 5, 0x100, [E0, E1], flags=0, imm=0x01020304) == w


def test_native_encoder_matches_python_mirror():
    k = 0
    for op in RDMA_OPS + SEND_OPS:
        for n0, n1 in ((1, 1), (15, 16), (4096, 1 << 20), (0x7FFFFFFF, 0x7FFFFFFF), (1 << 30, 5)):
            sges = [(2 ** 64 - 1 - k, 0xFFFFFFFF - k, n0), (0x1000 + 7 * k, 0x100 + k, n1)]
            fl = [0, W.CTRL_CQ_UPDATE, W.CTRL_CQ_UPDATE | W.CTRL_FENCE][k % 3]
            args = (op, 0xFFFF - k, 0xFFFFFF - k, sges, 2 ** 63 + k, 0xABCD0000 + k, fl, 0x01020304 + k)
            assert _native_build(*args) == _mirror(*args), (op, n0, n1)
            k += 1


@pytest.mark.parametrize("op", RDMA_OPS + SEND_OPS)
def test_decode_round_trip(op):
    w = _mirror(op, 77, 0x4242, [E0, E1], 0x1122334455667788, 0x0A0B0C0D, W.CTRL_CQ_UPDATE, 9)
    rdma = op in RDMA_OPS
    ra, rk = (0x1122334455667788, 0x0A0B0C0D) if rdma else (0, 0)
    v = W.decode_wqe(w)
    assert v.sges == [E0, E1] and v.nbytes == E0[2] + E1[2] and v.ds == (4 if rdma else 3)
    assert (v.opcode, v.wqe_idx, v.qpn, v.raddr, v.rkey, v.laddr, v.lkey) == (op, 77, 0x4242, ra, rk, E0[0], E0[1])
    ok, out = _decode_sg(w)
    assert ok == 1
    assert out == [op, 77, 0x4242, v.ds, W.CTRL_CQ_UPDATE, 9, ra, rk, E0[0], E0[1], E0[2] + E1[2], 0, 0, 2, E0[2], E1[0], E1[1]]
    # the 13-field hook keeps its fields (bytes is the total) and accepts the WQE
    out13 = (C.c_uint64 * 13)()
    assert _lib()[1].rn_wire_decode_wqe((C.c_uint8 * 64)(*w), out13) == 1 and list(out13) == out[:13]


def test_one_entry_wqes_decode_with_one_entry():
    for w in (W.rdma_wqe(W.OP_RDMA_WRITE, 1, 2, 0x1000, 3, 0x2000, 4, 64), W.send_wqe(W.OP_SEND, 1, 2, 0x1000, 3, 12)):
        ok, out = _decode_sg(w)
        assert ok == 1 and out[13:] == [1, 0, 0, 0]
        assert W.decode_wqe(w).sges == [(0x1000, 3, out[10])]


@pytest.mark.parametrize("op", RDMA_OPS + SEND_OPS)
@pytest.mark.parametrize("lens", [(0, 0x55), (0x55, 0), (0, 0)])
def test_zero_length_entries_collapse_to_the_one_entry_wqe(op, lens):
    sges = [(E0[0], E0[1], lens[0]), (E1[0], E1[1], lens[1])]
    kept = [e for e in sges if e[2]] or [(E0[0], E0[1], 0)]
    a, k, n = kept[0]
    one = (W.send_wqe(op, 9, 0x77, a, k, n, W.CTRL_CQ_UPDATE, 3) if op in SEND_OPS
           else W.rdma_wqe(op, 9, 0x77, a, k, 0x5000, 0x66, n, W.CTRL_CQ_UPDATE, 3))
    assert _native_build(op, 9, 0x77, sges, 0x5000, 0x66, W.CTRL_CQ_UPDATE, 3) == one
    assert _mirror(op, 9, 0x77, sges, 0x5000, 0x66, W.CTRL_CQ_UPDATE, 3) == one
    # a one-entry list is the one-entry WQE too
    assert _native_build(op, 9, 0x77, [kept[0]], 0x5000, 0x66, W.CTRL_CQ_UPDATE, 3) == one


def test_each_segment_saturates_on_its_own():
    w = _native_build(W.OP_RDMA_WRITE, 1, 2, [(0x1000, 1, 0xFFFFFFFF), (0x2000, 2, 0x80000000)], 0x3000, 3)
    assert w[32:36] == struct.pack(">I", W.MAX_BYTE_COUNT) and w[48:52] == struct.pack(">I", W.MAX_BYTE_COUNT)
    ok, out = _decode_sg(w)
    assert ok == 1 and out[10] == 2 * W.MAX_BYTE_COUNT and out[10] > W.MAX_MSG   # the total fits 32 bits, and fails as too long
    assert W.decode_wqe(w).nbytes == 2 * W.MAX_BYTE_COUNT


def test_hand_built_zero_length_segment_decodes():
    """Posters drop zero-length entries, but a two-segment WQE with one must still decode (both wires agree on it)."""
    b = bytearray(W.rdma_sg_wqe(W.OP_RDMA_WRITE, 1, 2, [E0, E1], 0x3000, 3))
    b[48:52] = bytes(4)
    ok, out = _decode_sg(bytes(b))
    assert ok == 1 and out[13] == 2 and out[10] == E0[2] and out[14] == E0[2]


def _with(w, off, data):
    b = bytearray(w)
    b[off:off + len(data)] = data
    return bytes(b)


def _bad_wqes():
    wr = W.rdma_sg_wqe(W.OP_RDMA_WRITE, 3, 5, [E0, E1], 0x1000, 7)
    sd = W.send_sg_wqe(W.OP_SEND, 3, 5, [E0, E1])
    return {
        "rdma_second_inline": _with(wr, 48, struct.pack(">I", 0x80000000 | 8)),
        "read_second_inline": _with(W.rdma_sg_wqe(W.OP_RDMA_READ, 3, 5, [E0, E1], 0x1000, 7), 48, struct.pack(">I", 0x80000008)),
        "send_second_inline": _with(sd, 32, struct.pack(">I", 0x80000000 | 8)),
        "rdma_ds5": _with(wr, 7, b"\x05"),
        "send_ds4": _with(sd, 7, b"\x04"),
        "rdma_ds2": _with(wr, 7, b"\x02"),
        "send_ds1": _with(sd, 7, b"\x01"),
    }


@pytest.mark.parametrize("case", list(_bad_wqes()))
def test_native_decoder_rejects_malformed_lists(case):
    _, lib = _lib()
    w = _bad_wqes()[case]
    assert _decode_sg(w)[0] == 0
    assert lib.rn_wire_decode_wqe((C.c_uint8 * 64)(*w), (C.c_uint64 * 13)()) == 0
    if "inline" in case:                    # the mirror checks the second segment's flag
        with pytest.raises(ValueError):
            W.decode_wqe(w)


# ---------------------------------------------------------------- against DOCA GPUNetIO's header
SRC = ROOT / "tests" / "native" / "sgl_crosscheck.cc"


def _compile(tmp_path, include_dir, hdr):
    exe = tmp_path / "sgl_crosscheck"
    cmd = ["g++", "-std=c++17", "-fpermissive", "-w", f"-I{include_dir}", f'-DDOCA_VERBS_DEF_H="{hdr}"', str(SRC), "-o", str(exe)]
    return exe, subprocess.run(cmd, capture_output=True, text=True, timeout=120)


def _doca():
    from test_wire_crosscheck import _doca_header
    hdr = _doca_header()
    if hdr is None or shutil.which("g++") is None:
        pytest.skip("the NCCL wheel in this image does not ship doca_gpunetio_verbs_def.h, or no host compiler")
    return hdr


def test_data_segment_and_two_entry_segment_counts_agree_with_doca_gpunetio(tmp_path):
    exe, r = _compile(tmp_path, ROOT / "rocnrdma_b200" / "csrc", _doca())
    assert r.returncode == 0, r.stderr[-3000:]
    assert subprocess.run([str(exe)], timeout=60).returncode == 0


def test_the_sgl_crosscheck_can_fail(tmp_path):
    """Negative control: a third entry per WQE and the same translation unit must stop compiling."""
    hdr = _doca()
    src = (ROOT / "rocnrdma_b200" / "csrc" / "wire" / "mlx5_wire.h").read_text()
    old = "  MAX_SGE = 2,"
    assert old in src
    (tmp_path / "wire").mkdir()
    (tmp_path / "wire" / "mlx5_wire.h").write_text(src.replace(old, "  MAX_SGE = 3,", 1))
    _, r = _compile(tmp_path, tmp_path, hdr)
    assert r.returncode != 0 and "fills one WQEBB" in r.stderr
