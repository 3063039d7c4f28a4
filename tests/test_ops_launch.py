"""The ops launch layer without a GPU: the scratch map, the result-record decoder, and the arguments every wrapper that
takes CPU tensors passes to its native entry point.

The wrappers run against a fake native library that records each ``rn_k_*`` call, a stub stream and a context whose
mapped scratch is a ctypes buffer.  Addresses are recorded as offsets into the buffer they point at (the mapped or
device scratch, a tensor), so the recorded calls are the same on every run; they are pinned in
``tests/golden/ops_launch_calls.json``."""
import ctypes as C
import dataclasses
import inspect
import json
import os

import pytest
import torch

from rocnrdma_b200 import _native as N, ops, wire as W
from rocnrdma_b200.api import Context
from rocnrdma_b200.ops import gemm as G, gemm_mx as MX, launch as L, pack as P, rdma as R
from rocnrdma_b200.parallel import ring_fp8

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ops_launch_calls.json")
MAPPED_BYTES, DEV_BYTES = 256 << 10, 2 << 20
DEV_BASE = 0xD000_0000_0000
STREAM = 0x5151
# the wrappers allocate these arguments themselves (checksum's and compare's result word): not pinned
_UNPINNED = {"rn_k_checksum": (3,), "rn_k_compare": (4,)}


# ---------------------------------------------------------------- the scratch map
# every default before the map existed: result-record offsets in the mapped scratch, device-scratch slots
DEFAULT_OFFSETS = {"rdma_stream": 0, "slot_results": 4096, "recv_consume": 8192, "shared_post_stress": 12288,
                   "atomic_stream": 16384, "put_signal": 20480, "signal_wait": 20544, "put_inline": 24576,
                   "cq_watch": 30720, "write_read": 32768, "gather_stream": 36864, "read_records": 40960,
                   "ring_results": 128 << 10}
DEFAULT_SLOTS = {"pack": 0, "unpack": 1, "gemm_send": 2, "gemm_mxfp8": 3, "reduce": 4}
SIGNATURE_DEFAULTS = [
    (ops.write_read, "scratch_off", 32768), (ops.recv_consume, "scratch_off", 8192),
    (ops.atomic_stream, "scratch_off", 16384), (ops.put_signal, "scratch_off", 20480),
    (ops.put_inline, "scratch_off", 24576), (ops.gather_stream, "scratch_off", 36864),
    (ops.signal_wait, "scratch_off", 20544), (ops.cq_watch, "scratch_off", 30720),
    (ops.read_records, "scratch_off", 40960), (ops.pack_fp8_write, "scratch_slot", 0),
    (ops.unpack_fp8, "scratch_slot", 1), (ops.gemm_send, "scratch_slot", 2), (ops.gemm_mxfp8, "scratch_slot", 3),
    (ops.reduce_fp8, "scratch_slot", 4)]


def test_the_map_keeps_every_default():
    assert {k: r.offset for k, r in L.MAPPED.items()} == DEFAULT_OFFSETS
    assert L.SLOT == DEFAULT_SLOTS
    assert L.SHARED_POST_STRESS_COUNTER.offset == 900 << 10
    for fn, name, value in SIGNATURE_DEFAULTS:
        assert inspect.signature(fn).parameters[name].default == value, fn.__name__
    assert [L.result_offset(s) for s in range(L.N_SLOTS)] == [4096 + 64 * s for s in range(L.N_SLOTS)]
    assert L.ring_result_offset(3, 5) == (128 << 10) + 3 * 4096 + 64 * 5
    assert ring_fp8.MAX_IN_PROCESS == 8


def test_regions_fit_and_do_not_overlap():
    assert L.MAPPED_BYTES == 256 << 10 and L.SLOT_BYTES * L.N_SLOTS == 2 << 20
    # at its largest: 64 QPs of the multi-QP launches, 8 slots of the per-slot and ring records
    assert L.MAPPED["atomic_stream"].nbytes == 64 * 64 and L.MAPPED["slot_results"].nbytes == 64 * 8
    assert L.MAPPED["ring_results"].nbytes == 8 * L.RING_SLOT_BYTES
    regions = sorted(L.MAPPED.values())
    assert all(r.offset % 64 == 0 and r.offset + r.nbytes <= L.MAPPED_BYTES for r in regions)
    for a, b in zip(regions, regions[1:]):
        assert a.offset + a.nbytes <= b.offset, (a, b)
    # device scratch: distinct slots; shared_post_stress's counter lies in gemm_mxfp8's slot and no other default's
    slots = list(L.SLOT.values())
    assert len(set(slots)) == len(slots) and all(0 <= s < L.N_SLOTS for s in slots)
    c = L.SHARED_POST_STRESS_COUNTER
    assert c.offset + c.nbytes <= L.N_SLOTS * L.SLOT_BYTES
    assert c.offset // L.SLOT_BYTES == (c.offset + c.nbytes - 1) // L.SLOT_BYTES == L.SLOT["gemm_mxfp8"]
    # the ring's records of one slot hold the 2N + 3 records of an 8-rank plan
    assert 2 * ring_fp8.MAX_IN_PROCESS + 3 <= L.RING_SLOT_BYTES // 64


def test_a_callers_offset_is_checked_once():
    for off in (0, 8256, 40960 + 64 * 7, L.MAPPED_BYTES - 64):
        assert L.scratch_offset(off) == off and L.result_offset(5, off) == off
    assert L.scratch_offset(L.MAPPED_BYTES - 64 * 64, 64) == L.MAPPED_BYTES - 64 * 64
    for off, n in ((-64, 1), (8200, 1), (L.MAPPED_BYTES, 1), (L.MAPPED_BYTES - 64, 2)):
        with pytest.raises(ValueError, match="multiple of 64"):
            L.scratch_offset(off, n)
    with pytest.raises(ValueError, match="multiple of 64"):
        L.result_offset(0, 100)


def test_every_slot_is_checked(fake):
    lib, ctx = fake
    a = torch.zeros(128, 64, dtype=torch.bfloat16)
    b, c = torch.zeros(256, 64, dtype=torch.bfloat16), torch.zeros(128, 256, dtype=torch.bfloat16)
    op = MX.MxOperand.from_tensors(torch.zeros(256, 64, dtype=torch.uint8), torch.zeros(256, 2, dtype=torch.uint8))
    mc = torch.zeros(256, 256, dtype=torch.bfloat16)
    for slot in (-1, 8):
        with pytest.raises(ValueError, match="scratch_slot"):
            ops.gemm_send(ctx, a, b, c, scratch_slot=slot)
        with pytest.raises(ValueError, match="scratch_slot"):
            ops.gemm_mxfp8(ctx, op, op, mc, scratch_slot=slot)
        with pytest.raises(ValueError, match="scratch_slot"):
            L.counters(ctx, 1, slot)
    with pytest.raises(ValueError, match="counters need"):
        L.counters(ctx, L.SLOT_BYTES // 4, 0)
    # a_ready is checked as every other arrival-word tensor: here it is not on the context's GPU
    with pytest.raises(ValueError, match="one word per record"):
        ops.gemm_mxfp8(ctx, op, op, mc, a_ready=torch.ones(1, dtype=torch.int64))
    assert lib.calls == []


# ---------------------------------------------------------------- record words
def _record(status: int, *words) -> C.Array:
    """A 64-byte result record: ``status``, then distinct words (t_start, t_end, ...), after ``words`` if given."""
    w = list(words) + [1000 + 111 * i for i in range(len(words), 7)]
    buf = (C.c_uint8 * 64)()
    (C.c_int64 * 8).from_buffer(buf)[:] = [status] + w
    return buf


STATUSES = {0: "OK", -1: "TIMEOUT", -2: "CQE_ERROR", -3: "QP_ERROR", 5: "5"}


@pytest.mark.parametrize("code", sorted(STATUSES))
def test_every_parser_reads_the_status_word(code):
    v = _record(code)
    name = STATUSES[code]
    assert R.parse_stream_out(v, 1, 64).status == [name]
    for parse in (R.parse_recv, R.parse_cq_watch, R.parse_signal_wait, R.parse_read_records, P.parse_unpack):
        assert parse(v)["status"] == name
    assert P.parse_reduce(v).status == name
    assert G.parse(v, 1, 2, 3).status == name
    assert R.WAIT_STATUS.get(code, str(code)) == name


def test_parsers_return_what_they_returned_before():
    v = _record(-1)
    t0, t1 = 1000, 1111
    assert R.parse_recv(v) == dict(status="TIMEOUT", device_ns=t1 - t0, t_start_ns=t0, t_end_ns=t1, seen=1222, bytes=1333)
    # a dict may gain the header's keys, never lose or change one
    assert R.parse_cq_watch(v) == dict(status="TIMEOUT", seen=1222, mismatches=1333, error_cqes=1444, device_ns=111,
                                       t_start_ns=t0, t_end_ns=t1)
    assert R.parse_signal_wait(v) == dict(status="TIMEOUT", seen=1222, mismatches=1333, device_ns=111, t_start_ns=t0,
                                          t_end_ns=t1)
    assert R.parse_read_records(v) == dict(status="TIMEOUT", done=1222, device_ns=111, t_start_ns=t0, t_end_ns=t1,
                                           first_idx=1333, last_idx=1444, cons=1555)
    assert P.parse_unpack(v) == dict(status="TIMEOUT", device_ns=111, records_seen=1222, records_forwarded=1333,
                                     t_first_post_ns=1444, t_start_ns=t0, t_end_ns=t1)
    assert P.parse_reduce(v) == P.ReduceResult("TIMEOUT", t0, t1, 1222, 1333, 1444, 1555, 0)
    assert P.parse_reduce(v, 99) == P.ReduceResult("TIMEOUT", t0, t1, 1222, 1333, 1444, 1555, 99)
    g = G.parse(v, 4, 5, 6)
    assert g == G.GemmResult("TIMEOUT", t0, t1, 1222, 1333, 1444, 4, 5, 6, variant=1555, stream_k=True)
    assert type(g.variant) is int and type(g.stream_k) is bool
    assert not G.parse(_record(0, 1, 2, 3, 4, 5, 6, 0), 1, 1, 1).stream_k
    two = (C.c_uint8 * 128)()
    two[:64], two[64:] = bytes(_record(-2, 10, 20, 3)), bytes(_record(0, 5, 40, 7))
    s = R.parse_stream_out(two, 2, 4096)
    assert s == R.StreamResult(["CQE_ERROR", "OK"], [10, 5], [20, 40], [3, 7], 4096)
    assert s.device_ns == 35 and not s.ok


# ---------------------------------------------------------------- the recorded launches
class FakeLib:
    """The native entry points a wrapper calls: ``rn_k_*`` are recorded, addresses as offsets into known regions."""

    def __init__(self, regions):
        self.calls, self.regions = [], regions

    def sym(self, x):
        if isinstance(x, C.Array):
            return [self.sym(v) for v in x]
        if isinstance(x, int) and not isinstance(x, bool):
            for name, base, size in self.regions:
                if base <= x < base + size:
                    return f"{name}+{x - base}"
        return x

    def rn_set_device(self, dev):
        return 0

    def rn_hca_dev_scratch(self, h, size):
        size._obj.value = DEV_BYTES
        return DEV_BASE

    def __getattr__(self, name):
        if not name.startswith("rn_k_"):
            raise AttributeError(name)

        def call(*args):
            args = [self.sym(a) for a in args]
            for i in _UNPINNED.get(name, ()):
                args[i] = "<allocated>"
            self.calls.append([name, args])
            return 0
        return call


class FakeStream:
    cuda_stream = STREAM

    def synchronize(self):
        pass


class FakeCtx:
    """A context whose mapped scratch is a ctypes buffer; scratch and device-scratch lookups are Context's own."""
    device, auto_sweep, wire, _vdev, _h = 0, False, "softhca", None, 1
    scratch, dev_scratch, dev_scratch_bytes, max_msg_bytes = (Context.scratch, Context.dev_scratch,
                                                              Context.dev_scratch_bytes, Context.max_msg_bytes)

    def __init__(self, lib):
        self._lib = lib
        self.buf = (C.c_uint8 * MAPPED_BYTES)()
        self._scratch_ptr, self._scratch_size = C.addressof(self.buf), MAPPED_BYTES
        # every record a wrapper might read holds distinct words, and every fifth one each status code
        w = (C.c_int64 * (MAPPED_BYTES // 8)).from_buffer(self.buf)
        for i in range(len(w)):
            w[i] = (0, -1, -2, -3, 9)[(i // 8) % 5] if i % 8 == 0 else 100 * i + i % 8


@dataclasses.dataclass
class Obj:
    """A queue pair, CQ or memory region: only the fields the wrappers read."""
    ctx: object = None
    dev_ptr: int = 0
    addr: int = 0
    length: int = 0
    lkey: int = 0
    rkey: int = 0
    sq_depth: int = 0
    scq: object = None
    depth: int = 0


class Values:
    """put_inline's values: a contiguous CUDA tensor that is never read on the host."""
    is_cuda = True

    def __init__(self, t):
        self.t = t

    def __getattr__(self, name):
        return getattr(self.t, name)


def _result(r, lib):
    if r is None:
        return None
    if isinstance(r, tuple):
        view, ws = r
        return ["view", lib.sym(C.addressof(view)), len(view), ws.cuda_stream]
    if dataclasses.is_dataclass(r):
        return [type(r).__name__, {k: v for k, v in vars(r).items()}]
    return r


@pytest.fixture
def fake(monkeypatch):
    """(fake native library, context) with the library and a stub stream in place."""
    for var in ("RN_GEMM_CTA_GROUP", "RN_GEMM_DENSE_PROBE", "RN_GEMM_NO_STREAMK", "RN_MX_CTA_GROUP"):
        monkeypatch.delenv(var, raising=False)
    lib = FakeLib([])
    ctx = FakeCtx(lib)
    lib.regions = [("scratch", ctx._scratch_ptr, MAPPED_BYTES), ("dev", DEV_BASE, DEV_BYTES)]
    monkeypatch.setattr(N, "load", lambda: lib)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: FakeStream())
    return lib, ctx


def _launches(lib, ctx):
    """(label, native calls, result) of every case, in order."""
    g = torch.Generator().manual_seed(3)
    T = {
        "u8": torch.zeros(1 << 16, dtype=torch.uint8),
        "u8b": torch.zeros(1 << 16, dtype=torch.uint8),
        "i64": torch.zeros(64, dtype=torch.int64),
        "bf": torch.randn(2 * P.TILE_ELEMS, generator=g).to(torch.bfloat16),
        "bf_out": torch.zeros(2 * P.TILE_ELEMS, dtype=torch.bfloat16),
        "stg": torch.zeros(P.staging_bytes(2 * P.TILE_ELEMS, P.TILE_ELEMS), dtype=torch.uint8),
        "ga": torch.zeros(128, 64, dtype=torch.bfloat16),
        "gb": torch.zeros(256, 64, dtype=torch.bfloat16),
        "gc": torch.zeros(128, 256, dtype=torch.bfloat16),
        "gc8": torch.zeros(G.panel_record_bytes(256), dtype=torch.uint8),
        "vals": torch.zeros(4, 16, dtype=torch.uint8),
        "mq": torch.zeros(256, 64, dtype=torch.uint8),
        "ms": torch.zeros(256, 2, dtype=torch.uint8),
        "mc": torch.zeros(256, 256, dtype=torch.bfloat16),
    }
    lib.regions += [(k, t.data_ptr(), t.numel() * t.element_size()) for k, t in T.items()]
    cq = Obj(ctx=ctx, dev_ptr=0xC0, depth=64)
    q0, q1, q2 = (Obj(ctx=ctx, dev_ptr=0xA0 + i, sq_depth=32, scq=cq) for i in range(3))
    mr = {k: Obj(ctx=ctx, addr=(0x10 + i) << 32, length=1 << 20, lkey=0x100 + i, rkey=0x200 + i)
          for i, k in enumerate(("a", "b", "c", "sig", "fetch"))}
    a, b, c, sig, fetch = (mr[k] for k in ("a", "b", "c", "sig", "fetch"))
    stg_mr = Obj(ctx=ctx, addr=T["stg"].data_ptr(), length=T["stg"].numel(), lkey=0x300, rkey=0x301)
    pair = lambda k: (T[k].data_ptr(), T[k].numel())  # noqa: E731
    a_op = MX.MxOperand.from_tensors(T["mq"], T["ms"])
    b_op = MX.MxOperand.from_tensors(T["mq"], T["ms"])
    rb = P.record_bytes(P.TILE_ELEMS)
    cases = [
        ("rdma_stream lone", lambda: ops.rdma_stream(q0, W.OP_RDMA_WRITE, a, b, 4096, iters=3)),
        ("rdma_stream listed", lambda: ops.rdma_stream(
            [q0, q1], W.OP_RDMA_READ, a, b, 65536, iters=5, window=8, signal_every=2, burst=2, stride=1 << 20,
            slot_stride=4096, nslots=3, timeout_ms=500, post_only=True, fence_every=3)),
        ("rdma_stream no dst, async", lambda: ops.rdma_stream(q1, W.OP_SEND, a, None, 100, sync=False)),
        ("rdma_stream out=", lambda: ops.rdma_stream([q0, q1], W.OP_RDMA_WRITE, a, b, 8, sync=False,
                                                     out=ctx.scratch(128, offset=1024))),
        ("write_read", lambda: ops.write_read(q0, a, b, c, 4096, iters=2, mode="wait")),
        ("write_read one_call", lambda: ops.write_read(q1, a, b, c, 64, mode="one_call", timeout_ms=0,
                                                       scratch_off=32768 + 128)),
        ("fill_random", lambda: ops.fill_random(T["u8"], seed=3) is T["u8"]),
        ("fill_bf16", lambda: ops.fill_bf16(T["bf_out"], seed=2, scale=0.5) is T["bf_out"]),
        ("checksum", lambda: ops.checksum(T["u8"])),
        ("compare", lambda: ops.compare(T["u8"], T["u8b"])),
        ("compare nbytes", lambda: ops.compare(T["u8"], T["u8b"], nbytes=100)),
        ("l2_flush", lambda: ops.l2_flush(T["u8"], 7)),
        ("recv_consume", lambda: ops.recv_consume(q0, 5)),
        ("recv_consume stamps prepost", lambda: ops.recv_consume(
            q1, 4, max_imm=8, stamps=T["i64"], prepost_mr=a, prepost_bytes=0, scratch_off=8256, sync=False)),
        ("shared_post_stress", lambda: R.shared_post_stress(q0, a, b, ctas=4, per_cta=8)),
        ("atomic_stream fa", lambda: ops.atomic_stream(q0, "fa", sig, fetch, 4, add=-1)),
        ("atomic_stream cs chain", lambda: ops.atomic_stream(
            [q0, q1, q2], "cs", sig, fetch, 4, compare=5, swap=6, chain=True, target_stride=8, window=4, burst=2,
            signal_every=2, timeout_ms=300, scratch_off=16384 + 64 * 4, sync=False)),
        ("put_signal", lambda: ops.put_signal(q0, a, b, 256, sig, sig_off=8, fetch_mr=fetch, add=3, iters=4,
                                              window=2, slot_stride=256, nslots=4)),
        ("put_inline plain", lambda: ops.put_inline(q0, Values(T["vals"].reshape(-1)), b, 8, iters=3)),
        ("put_inline signal", lambda: ops.put_inline(
            [q0, q1], Values(T["vals"]), b, 16, iters=2, window=4, burst=2, signal_every=2, slot_stride=32, nslots=2,
            sig_mr=sig, sig_off=16, fetch_mr=fetch, add=2, sync=False, scratch_off=24576 + 64)),
        ("gather_stream", lambda: ops.gather_stream(q0, W.OP_RDMA_WRITE, a, b, c, 4096, 1000)),
        ("gather_stream send one_call", lambda: ops.gather_stream(
            [q0, q1], W.OP_SEND, a, b, None, 2048, 0, iters=3, window=2, stride=8192, slot_stride=2048, nslots=2,
            via="one_call", scratch_off=36864 + 128, sync=False)),
        ("signal_wait", lambda: ops.signal_wait(ctx, pair("i64"), 5)),
        ("signal_wait mr check", lambda: ops.signal_wait(
            ctx, sig, 3, stamps=T["i64"], check=(pair("u8"), pair("u8b"), 64, 128), timeout_ms=50, sync=False,
            scratch_off=20544 + 64)),
        ("cq_watch", lambda: ops.cq_watch(cq, 4, pair("u8"), pair("u8b"), 4096, 2, 4096, 1024)),
        ("cq_watch tail", lambda: ops.cq_watch(cq, 2, T["u8"], T["u8b"], 1024, 4, 1024, 512, tail=256, sync=False,
                                               scratch_off=30720 + 64)),
        ("read_records", lambda: ops.read_records(q0, a, b, 4096, 8)),
        ("read_records strided", lambda: ops.read_records(
            q1, a, b, 1024, 4, src_off=64, src_stride=2048, dst_off=128, window=0, burst=2, signal_every=2,
            sync=False, scratch_off=40960 + 64 * 3)),
        ("pack_fp8_write local", lambda: ops.pack_fp8_write(ctx, T["bf"], stg_mr, chunk_elems=P.TILE_ELEMS)),
        ("pack_fp8_write posting", lambda: ops.pack_fp8_write(
            ctx, T["bf"], stg_mr, qp=q0, dst_mr=b, chunk_elems=P.TILE_ELEMS, with_imm=True, signal_every=2, grid=3,
            post_only=True, direct=True, scratch_slot=5)),
        ("pack_fp8_write result_off", lambda: ops.pack_fp8_write(
            ctx, T["bf"], stg_mr, qp=q1, dst_mr=b, chunk_elems=2 * P.TILE_ELEMS, sync=False, result_off=(128 << 10) + 64)),
        ("unpack_fp8", lambda: ops.unpack_fp8(ctx, T["stg"], T["bf_out"], P.TILE_ELEMS)),
        ("unpack_fp8 cq", lambda: ops.unpack_fp8(ctx, T["stg"], T["bf_out"], P.TILE_ELEMS, qp=q1, grid=2,
                                                 timeout_ms=10, scratch_slot=6)),
        ("unpack_fp8 forward", lambda: ops.unpack_fp8(
            ctx, T["stg"][rb:], T["bf_out"][P.TILE_ELEMS:], P.TILE_ELEMS, fwd_qp=q0, fwd_src_mr=stg_mr, fwd_dst_mr=b,
            fwd_dst_off=2 * rb, with_imm=True, imm_base=7, signal_every=2, post_only=True, sync=False,
            result_off=(128 << 10) + 4096)),
        ("gemm_send", lambda: ops.gemm_send(ctx, T["ga"], T["gb"], T["gc"])),
        ("gemm_send fp8 posting", lambda: ops.gemm_send(
            ctx, T["ga"], T["gb"], T["gc8"], c_mr=c, qp=q0, dst_mr=b, out_fp8=True, with_imm=True, signal_every=2,
            cta_group=3, group_m=2, grid=4, post_only=True, stream_k=True, scratch_slot=6, sync=False)),
        ("gemm_send plain_stores", lambda: ops.gemm_send(ctx, T["ga"], T["gb"], T["gc"], plain_stores=True, cta_group=1,
                                                         timeout_ms=7)),
        ("gemm_mxfp8", lambda: ops.gemm_mxfp8(ctx, a_op, b_op, T["mc"])),
        ("gemm_mxfp8 async", lambda: ops.gemm_mxfp8(ctx, a_op, b_op, T["mc"], grid=8, cta_group=1, scratch_slot=7,
                                                    timeout_ms=9, sync=False)),
    ]
    out = []
    for label, fn in cases:
        lib.calls = []
        r = fn()
        out.append([label, lib.calls, _result(r, lib)])
    return out


def test_wrappers_pass_the_arguments_they_passed_before(fake):
    got = json.loads(json.dumps(_launches(*fake)))
    with open(GOLDEN) as f:
        want = json.load(f)
    assert [c[0] for c in got] == [c[0] for c in want]
    header = {"t_start_ns", "t_end_ns", "device_ns"}
    for g, w in zip(got, want):
        if isinstance(w[2], dict):      # a returned dict may gain the header's keys, never lose or change one
            extra = g[2].keys() - w[2].keys()
            assert extra <= header, g[0]
            g[2] = {k: v for k, v in g[2].items() if k not in extra}
        assert g == w, g[0]
