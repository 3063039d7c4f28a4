"""Verbs-shaped public API over the native software HCA.

    ctx = Context(device=0)                      # ~ ibv_open_device + alloc_pd
    mr  = ctx.reg_mr(tensor)                     # ~ ibv_reg_mr on a GPU pointer (the reference's whole purpose)
    cq  = ctx.create_cq(1024)
    qp  = ctx.create_qp(cq)                      # RC queue pair
    qp.connect(peer_qp)                          # RESET->INIT->RTR->RTS both ways
    ctx.engine_start(ctas=32)                    # the DMA engine (the "NIC")
    qp.post_write(src_mr, dst_mr, nbytes)        # host-posted   (baseline: SURVEY.md B2)
    ops.rdma_stream(qp, ...)                     # GPU-posted    (product:  SURVEY.md P1)

Two wires sit under the same objects (``Context(wire=...)``):

* ``softhca`` -- the software HCA: queues in GPU or pinned memory, a persistent sm_90a kernel moves
  the bytes.  What runs when the box exposes no NIC.
* ``verbs``   -- a ConnectX through libibverbs / mlx5dv (``csrc/verbs/verbs_dl.cc``): ``reg_mr`` is
  ``ibv_reg_dmabuf_mr`` / ``ibv_reg_mr`` on the GPU pointer, host-posted verbs are ``ibv_post_send``,
  and ``loopback_qp(mem=MEM_DEVICE)`` hands the raw mlx5 queues to the GPU so the same kernels post
  to the NIC.  ``auto`` picks it when a real HCA is reachable.

Reference parity: ``reg_mr`` is what amdp2p's seven peer-memory callbacks make
possible (amdp2p.c:363-371); revocation (``MemoryRegion.revoke``) is
free_callback (amdp2p.c:88-109).  Everything below registration has no
counterpart there.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional

import os

from . import _native as N
from . import wire as W

# ibv_wc_status -> the syndrome names the softhca wire reports (wire.SYNDROMES), so callers see one vocabulary
_WC_STATUS = {0: "OK", 1: "LOCAL_LENGTH_ERR", 2: "LOCAL_QP_OP_ERR", 4: "LOCAL_PROT_ERR", 5: "WR_FLUSH_ERR", 6: "MW_BIND_ERR",
              7: "BAD_RESP_ERR", 8: "LOCAL_ACCESS_ERR", 9: "REMOTE_INVAL_REQ_ERR", 10: "REMOTE_ACCESS_ERR", 11: "REMOTE_OP_ERR",
              12: "TRANSPORT_RETRY_EXC_ERR", 13: "RNR_RETRY_EXC_ERR", 16: "REMOTE_ABORTED_ERR", 21: "GENERAL_ERR"}
_IBV_WC_RECV, _IBV_WC_RECV_RDMA_WITH_IMM = 128, 129


def resolve_wire(wire: str = "auto") -> str:
    """'auto' -> 'verbs' when a REAL HCA is usable (libibverbs loads, /dev/infiniband is there, a device
    exists), else 'softhca'.  The mock provider is never picked automatically: ask for it with
    ``wire="verbs"`` (or ROCNRDMA_WIRE=verbs) after ``_native.use_mock_verbs()``."""
    wire = os.environ.get("ROCNRDMA_WIRE", wire) if wire == "auto" else wire
    if wire not in ("auto", "softhca", "verbs"):
        raise ValueError(f"wire={wire!r}: expected auto | softhca | verbs")
    if wire != "auto":
        return wire
    lib = N.load()
    return "verbs" if lib.rn_verbs_available() > 0 and not lib.rn_verbs_is_mock() else "softhca"


def _ptr_len(buf, nbytes=None):
    """Accept a torch tensor, a (ptr, nbytes) tuple, or an object with __cuda_array_interface__."""
    if isinstance(buf, tuple):
        return int(buf[0]), int(buf[1])
    if hasattr(buf, "data_ptr"):
        n = buf.numel() * buf.element_size()
        return int(buf.data_ptr()), int(n if nbytes is None else nbytes)
    if hasattr(buf, "ctypes"):  # numpy
        return int(buf.ctypes.data), int(buf.nbytes if nbytes is None else nbytes)
    raise TypeError(f"cannot take the address of {type(buf)!r}")


@dataclass
class WorkCompletion:
    qpn: int
    wqe_counter: int
    opcode: int
    byte_cnt: int
    imm: int
    syndrome: int
    wqe_opcode: int
    is_error: bool
    status_name: Optional[str] = None      # verbs wire: the ibv_wc_status, in the same vocabulary
    wr_id: int = 0

    @property
    def status(self) -> str:
        return self.status_name or W.SYNDROMES.get(self.syndrome, hex(self.syndrome))


class MemoryRegion:
    """A registered range (what ``ibv_reg_mr`` returns): ``addr``/``length``, one key used as lkey and rkey (mlx5 style), access bits; ``state`` follows PINNED -> REVOKED -> FREE."""
    def __init__(self, ctx: "Context", addr: int, length: int, key: int, access: int, keepalive=None, rkey: Optional[int] = None,
                 vmr=None):
        self.ctx, self.addr, self.length, self.key, self.access = ctx, addr, length, key, access
        self.lkey = key
        self.rkey = key if rkey is None else rkey
        self._keepalive = keepalive
        self._live = True
        self._vmr = vmr               # verbs wire: the ibv_mr handle
        self.dmabuf_fd = -1
        self.mode = "direct"

    @property
    def state(self) -> str:
        """FREE / PINNED / REVOKED, read from the HCA."""
        if self._vmr is not None or self.ctx.wire == "verbs":
            return "PINNED" if self._live else "FREE"
        return ["FREE", "PINNED", "REVOKED"][self.ctx._lib.rn_mr_state(self.ctx._h, self.key)]

    @property
    def driver_revoked(self) -> bool:
        """True when the revocation came from the driver's side (the allocation vanished), not from ``revoke()``."""
        return self.ctx.wire == "softhca" and bool(self.ctx._lib.rn_mr_driver_revoked(self.ctx._h, self.key))

    def revoke(self):
        """The backing memory is going away: stop translating now (the engine fails
        any WQE that names this key with a protection error)."""
        if self.ctx.wire == "verbs":
            raise N.NativeError("revocation on the verbs wire is the GPU driver's call (free the memory): "
                                "the peer-memory client's free callback invalidates the MR (kmod/b200p2p.c)")
        N.check(self.ctx._lib.rn_mr_revoke(self.ctx._h, self.key), "mr_revoke")

    def dereg(self):
        """Release the MKey slot (and the dma-buf pin, if any).  Safe after ``revoke``."""
        if not self._live:
            return
        if self._vmr is not None:
            rc = self.ctx._lib.rn_verbs_dereg_mr(self._vmr)
            self._vmr = None
            if self.dmabuf_fd >= 0:
                self.ctx._lib.rn_dmabuf_close(self.dmabuf_fd)
                self.dmabuf_fd = -1
            if rc:
                raise N.NativeError(f"ibv_dereg_mr failed ({rc})")
        else:
            N.check(self.ctx._lib.rn_dereg_mr(self.ctx._h, self.key), "dereg_mr")
        self._live = False
        self._keepalive = None

    def __repr__(self):
        return f"MemoryRegion(addr=0x{self.addr:x}, len={self.length}, key=0x{self.key:x})"


class CompletionQueue:
    """A completion queue: 64-byte mlx5 CQEs with an owner bit, in device or pinned host memory.  Device posters poll it themselves; these methods are the host-side consumer."""
    def __init__(self, ctx, handle, depth, mem, vcq=None):
        self.ctx, self._c, self.depth, self.mem = ctx, handle, depth, mem
        self._vcq = vcq               # verbs wire: the ibv_cq handle

    @property
    def dev_ptr(self) -> int:
        if self._c is None:
            raise N.NativeError("this CQ belongs to the HCA; it has a device view only once its QP was handed to the GPU")
        return self.ctx._lib.rn_cq_dev(self._c)

    def poll(self, max_entries: int = 16) -> List[WorkCompletion]:
        """Consume up to ``max_entries`` completions that are ready now (never blocks)."""
        if self._vcq is not None:
            n_max = min(max_entries, 32)
            varr = (N.RnVWc * n_max)()
            n = self.ctx._lib.rn_verbs_poll(self._vcq, n_max, varr)
            if n < 0:
                raise N.NativeError(f"ibv_poll_cq failed ({n})")
            out = []
            for a in varr[:n]:
                recv = a.opcode >= _IBV_WC_RECV
                err = a.status != 0
                if recv:
                    opc = W.CQE_RESP_ERR if err else (W.CQE_RESP_WR_IMM if a.opcode == _IBV_WC_RECV_RDMA_WITH_IMM else
                                                      (W.CQE_RESP_SEND_IMM if a.with_imm else W.CQE_RESP_SEND))
                else:
                    opc = W.CQE_REQ_ERR if err else W.CQE_REQ
                name = _WC_STATUS.get(a.status, f"IBV_WC_{a.status}")
                out.append(WorkCompletion(a.qp_num, a.wr_id & 0xFFFF, opc, a.byte_len, a.imm, W.SYN.get(name, 0xFF if err else 0), 0,
                                          err, status_name=name, wr_id=a.wr_id))
            return out
        arr = (N.RnWc * max_entries)()
        n = self.ctx._lib.rn_poll_cq(self._c, max_entries, arr)
        if n < 0:
            raise N.NativeError(f"poll_cq failed ({n})")
        return [WorkCompletion(a.qpn, a.wqe_counter, a.opcode, a.byte_cnt, a.imm, a.syndrome, a.wqe_opcode,
                               bool(a.is_error)) for a in arr[:n]]

    def wait(self, n: int = 1, timeout_s: float = 5.0) -> List[WorkCompletion]:
        """Poll until ``n`` completions have been consumed; ``TimeoutError`` after ``timeout_s``."""
        import time
        out: List[WorkCompletion] = []
        t0 = time.monotonic()
        while len(out) < n:
            out += self.poll(n - len(out))
            if len(out) < n and time.monotonic() - t0 > timeout_s:
                raise TimeoutError(f"CQ wait: got {len(out)}/{n} completions in {timeout_s}s")
        return out


class QueuePair:
    """A reliable-connected queue pair: send queue of 64-byte WQEBBs, receive queue, doorbell record and doorbell register, in device memory (GPU posters) or pinned host memory (host posters).  RESET -> INIT -> RTR -> RTS as in IB."""
    def __init__(self, ctx, handle, scq, rcq, sq_depth, rq_depth, sq_mem):
        self.ctx, self._q, self.scq, self.rcq = ctx, handle, scq, rcq
        self.sq_depth, self.rq_depth, self.sq_mem = sq_depth, rq_depth, sq_mem
        self.qpn = ctx._lib.rn_qp_num(handle)

    @property
    def dev_ptr(self) -> int:
        return self.ctx._lib.rn_qp_dev(self._q)

    @property
    def state(self) -> str:
        """Current IB state name (RESET, INIT, RTR, RTS, SQD, SQE, ERR)."""
        return W.QP_STATE_NAMES[self.ctx._lib.rn_qp_state(self._q)]

    def modify(self, state: int):
        """``ibv_modify_qp``: checked state transition (``wire.QPS_*``); RESET rewinds every index and the doorbell."""
        N.check(self.ctx._lib.rn_modify_qp(self._q, state), "modify_qp")

    def describe(self) -> N.RnRemote:
        """What a requester must know to target this QP as a responder (receive ring, receive CQ, MKey table, QP number)."""
        r = N.RnRemote()
        N.check(self.ctx._lib.rn_qp_describe(self._q, C.byref(r)), "qp_describe")
        return r

    def connect_remote(self, remote: N.RnRemote):
        """Install an already translated description of the responder (see ``parallel.peer.connect_to``)."""
        N.check(self.ctx._lib.rn_qp_connect(self._q, C.byref(remote)), "qp_connect")

    def connect(self, peer: Optional["QueuePair"] = None):
        """Bring this QP and ``peer`` (default: itself, i.e. loopback) to RTS."""
        peer = peer or self
        N.check(self.ctx._lib.rn_qp_connect_pair(self._q, peer._q), "qp_connect_pair")
        return self

    # ---- host-posted verbs (the "ibv_post_send" baseline path)
    def _post(self, opcode, laddr, lkey, raddr, rkey, nbytes, signaled=True, imm=0) -> int:
        idx = C.c_uint64()
        flags = W.CTRL_CQ_UPDATE if signaled else 0
        self.ctx.sweep_revoked()          # a freed allocation must not be reachable through a stale key
        N.check(self.ctx._lib.rn_post_send(self._q, opcode, laddr, lkey, raddr, rkey, nbytes, flags, imm,
                                           C.byref(idx)), "post_send")
        return idx.value

    def post_write(self, src: MemoryRegion, dst: MemoryRegion, nbytes=None, src_off=0, dst_off=0, signaled=True,
                   imm=None) -> int:
        """Host-posted RDMA WRITE (``imm`` not None: WRITE_WITH_IMM, consumes a receive WQE at the responder).  Returns the WQE index."""
        n = src.length - src_off if nbytes is None else nbytes
        op = W.OP_RDMA_WRITE if imm is None else W.OP_RDMA_WRITE_IMM
        return self._post(op, src.addr + src_off, src.lkey, dst.addr + dst_off, dst.rkey, n, signaled, imm or 0)

    def post_read(self, dst_local: MemoryRegion, src_remote: MemoryRegion, nbytes=None, local_off=0, remote_off=0,
                  signaled=True) -> int:
        """Host-posted RDMA READ into ``dst_local``.  Returns the WQE index."""
        n = dst_local.length - local_off if nbytes is None else nbytes
        return self._post(W.OP_RDMA_READ, dst_local.addr + local_off, dst_local.lkey, src_remote.addr + remote_off,
                          src_remote.rkey, n, signaled)

    def post_send(self, src: MemoryRegion, nbytes=None, src_off=0, signaled=True, imm=None) -> int:
        """Host-posted SEND (``imm`` not None: SEND_WITH_IMM); lands in the responder's next receive buffer."""
        n = src.length - src_off if nbytes is None else nbytes
        op = W.OP_SEND if imm is None else W.OP_SEND_IMM
        return self._post(op, src.addr + src_off, src.lkey, 0, 0, n, signaled, imm or 0)

    def post_raw(self, opcode, laddr=0, lkey=0, raddr=0, rkey=0, nbytes=0, signaled=True, imm=0) -> int:
        """Post a WQE with arbitrary fields (error-path tests: bad keys, bad opcodes, NOP)."""
        return self._post(opcode, laddr, lkey, raddr, rkey, nbytes, signaled, imm)

    def post_recv(self, dst: MemoryRegion, nbytes=None, off=0):
        """Post one receive buffer (consumed in order by SEND / WRITE_WITH_IMM)."""
        n = dst.length - off if nbytes is None else nbytes
        N.check(self.ctx._lib.rn_post_recv(self._q, dst.addr + off, dst.lkey, n), "post_recv")

    def set_flags(self, sys_scope: Optional[bool] = None, trace: Optional[bool] = None):
        """sys_scope: force system-scope fences (peer GPU / NIC paths).  trace: stamp each
        WQE's lifecycle (post, claim, parsed, copied, cqe, seen) with %globaltimer."""
        N.check(self.ctx._lib.rn_qp_set_flags(self._q, -1 if sys_scope is None else int(sys_scope),
                                              -1 if trace is None else int(trace)), "qp_set_flags")

    def read_trace(self, nslots: Optional[int] = None) -> List[dict]:
        """Per-SQ-slot %globaltimer stamps (post, claim, parsed, copied, cqe, seen); needs ``set_flags(trace=True)``."""
        n = nslots or self.sq_depth
        buf = (C.c_uint64 * (n * 8))()
        N.check(self.ctx._lib.rn_qp_read_trace(self._q, buf, n), "qp_read_trace")
        names = ["post", "claim", "parsed", "copied", "cqe", "seen"]
        return [{k: buf[i * 8 + j] for j, k in enumerate(names)} for i in range(n)]

    def counters(self) -> dict:
        """Engine-side counters of this QP (WQEs, CQEs, errors, bytes, RNR waits, doorbell-order violations) and its queue indices."""
        c = N.RnQpCounters()
        N.check(self.ctx._lib.rn_qp_query(self._q, C.byref(c)), "qp_query")
        d = {k: getattr(c, k) for k, _ in c._fields_ if k != "pad"}
        d["state"] = W.QP_STATE_NAMES[d["state"]]
        return d


class VerbsQueuePair(QueuePair):
    """An RC QP of a real HCA (verbs wire).  Host-posted by default (``ibv_post_send``: baselines B0 / B2);
    ``to_gpu()`` maps its mlx5 queues and doorbell register into the GPU and wraps them in the device-side
    ``QpDev`` the kernels post to (IBGDA) -- after that the host must not post to it any more."""
    def __init__(self, ctx, vq, scq, rcq, sq_depth, rq_depth, sq_mem):
        self.ctx, self._vq, self.scq, self.rcq = ctx, vq, scq, rcq
        self.sq_depth, self.rq_depth, self.sq_mem = sq_depth, rq_depth, sq_mem
        self._q = None                       # the adopted (GPU-visible) view, once to_gpu() ran
        self.qpn = ctx._lib.rn_verbs_qpn(vq)
        self.db_proxy = False
        self._peer = None

    @property
    def on_gpu(self) -> bool:
        return self._q is not None

    @property
    def dev_ptr(self) -> int:
        if self._q is None:
            raise N.NativeError("this QP is host-posted; call to_gpu() (or create it with mem=MEM_DEVICE) before launching kernels on it")
        return self.ctx._lib.rn_qp_dev(self._q)

    @property
    def state(self) -> str:
        return W.QP_STATE_NAMES[min(self.ctx._lib.rn_verbs_qp_state(self._vq), 6)]

    def modify(self, state: int):
        """Only the attribute-less transitions (RESET, ERR); ``connect`` walks INIT -> RTR -> RTS."""
        if state not in (W.QPS_RESET, W.QPS_ERR):
            raise N.NativeError("verbs wire: use connect() for INIT/RTR/RTS")
        self._vcheck(self.ctx._lib.rn_verbs_set_state(self._vq, state), "modify_qp")

    def _vcheck(self, rc, what):
        if rc:
            raise N.NativeError(f"{what} failed (rc={rc}): {self.ctx._lib.rn_verbs_why().decode(errors='replace')}")

    def address(self):
        """(qpn, lid, gid bytes): what the other side needs for its RTR transition (exchanged out of band)."""
        lid = C.c_uint16()
        gid = (C.c_uint8 * 16)()
        self.ctx._lib.rn_verbs_local_addr(self.ctx._vdev, C.byref(lid), gid)
        return self.qpn, lid.value, bytes(gid)

    def connect_to(self, qpn: int, lid: int, gid: bytes = b""):
        g = (C.c_uint8 * 16)(*gid) if gid and not lid else None
        self._vcheck(self.ctx._lib.rn_verbs_connect(self._vq, qpn, lid, g), "connect")
        return self

    def connect(self, peer: Optional["QueuePair"] = None):
        """Bring this QP and ``peer`` (default: itself -- loopback through the port) to RTS.  ``peer`` may live on
        another HCA (NIC0 -> NIC1) as long as both are reachable from this process."""
        peer = peer or self
        self.connect_to(*peer.address())
        if peer is not self:
            peer.connect_to(*self.address())
        self._peer, peer._peer = peer, self
        if self.sq_mem == W.MEM_DEVICE:
            self.to_gpu()
        if peer is not self and peer.sq_mem == W.MEM_DEVICE:
            peer.to_gpu()
        return self

    def describe(self):
        raise N.NativeError("verbs wire: peers exchange address() tuples, not softhca descriptors")

    connect_remote = describe

    def to_gpu(self):
        """mlx5dv_init_obj + cudaHostRegister: SQ / RQ / doorbell record / CQs (host memory the NIC reads) and the
        BlueFlame register (MMIO) become GPU-addressable; ``dev_ptr`` is then what ``ops.rdma_stream``,
        ``ops.pack_fp8_write`` and ``ops.gemm_send`` take.  Falls back to a CPU doorbell proxy when the UAR page
        cannot be mapped (``db_proxy`` says which)."""
        if self._q is not None:
            return self
        if self.ctx._h is None:
            raise N.NativeError("to_gpu() needs a context bound to a GPU (device=None is host-only)")
        g = N.RnGpuQp()
        N.load().rn_set_device(self.ctx.device)
        self._vcheck(self.ctx._lib.rn_verbs_map_qp_to_gpu(self._vq, C.byref(g)), "map_qp_to_gpu")
        q = C.c_void_p()
        N.check(self.ctx._lib.rn_qp_adopt(self.ctx._h, C.byref(g), C.byref(q)), "qp_adopt")
        self._q = q
        self.db_proxy = bool(g.flags & 1)
        self.raw = {k: getattr(g, k) for k, _ in g._fields_}
        return self

    def raw_queues(self) -> dict:
        """The mlx5dv view (host addresses and geometry of SQ / RQ / doorbell record / BlueFlame register / CQs)."""
        r = N.RnRawQp()
        self._vcheck(self.ctx._lib.rn_verbs_raw_qp(self._vq, C.byref(r)), "raw_qp")
        return {k: getattr(r, k) for k, _ in r._fields_ if not k.startswith("pad")}

    def _post(self, opcode, laddr, lkey, raddr, rkey, nbytes, signaled=True, imm=0) -> int:
        wr = C.c_uint64()
        self._vcheck(self.ctx._lib.rn_verbs_post_send(self._vq, opcode, laddr, lkey, raddr, rkey, nbytes, int(bool(signaled)), imm,
                                                      C.byref(wr)), "post_send")
        return wr.value

    def post_recv(self, dst: MemoryRegion, nbytes=None, off=0):
        n = dst.length - off if nbytes is None else nbytes
        self._vcheck(self.ctx._lib.rn_verbs_post_recv(self._vq, dst.addr + off, dst.lkey, n, None), "post_recv")

    def set_flags(self, sys_scope: Optional[bool] = None, trace: Optional[bool] = None):
        if self._q is not None:
            super().set_flags(sys_scope, trace)

    def read_trace(self, nslots: Optional[int] = None) -> List[dict]:
        if self._q is None:
            return []
        return super().read_trace(nslots)

    def counters(self) -> dict:
        """Poster-side indices (when on the GPU) plus, on the mock provider, the NIC's own counters
        (``n_db_order_violations`` = doorbells that arrived before the doorbell record moved)."""
        d = {"n_wqe": 0, "n_cqe": 0, "n_err": 0, "n_db_order_violations": 0, "n_bytes": 0, "n_rnr": 0}
        if self._q is not None:
            c = N.RnQpCounters()
            N.check(self.ctx._lib.rn_qp_query(self._q, C.byref(c)), "qp_query")
            d.update({k: getattr(c, k) for k in ("resv_head", "ready_head", "sq_cons")})
        st = N.RnMockQpStats()
        if self.ctx._lib.rn_verbs_mock_qp_stats(self._vq, C.byref(st)) == 0:
            d.update(n_wqe=st.n_wqe, n_cqe=st.n_cqe, n_err=st.n_err, n_bytes=st.n_bytes, n_rnr=st.n_rnr,
                     n_db_order_violations=st.n_db_no_progress, n_doorbells=st.n_doorbells, cq_overruns=st.sq_cq_overruns)
            d["nic"] = "mock"
        d["state"] = self.state
        d["db_proxy_forwarded"] = self.ctx._lib.rn_verbs_db_proxy_forwarded(self._vq)
        return d

    def destroy(self):
        if self._vq is not None:
            self.ctx._lib.rn_verbs_destroy_qp(self._vq)
            self._vq = None


class Context:
    """One software HCA bound to one GPU (one per process in multi-GPU runs)."""

    def __init__(self, device: int = 0, max_mkeys: int = 1024, max_qps: int = 256, arena_bytes: int = 64 << 20,
                 host_arena_bytes: int = 16 << 20, wire: str = "auto", nic=None, port: int = 1, gid_index: int = 0):
        """``wire``: ``softhca`` | ``verbs`` | ``auto`` (see :func:`resolve_wire`).  On the verbs wire ``nic`` names
        the HCA (``"mlx5_3"``) or gives its index (default: the GPU's index, the usual GPU i <-> NIC i pairing)."""
        self._lib = N.load()
        self.wire = resolve_wire(wire)
        self._vdev = None
        self._vqps: List["VerbsQueuePair"] = []
        self._vcqs: List[CompletionQueue] = []
        h = C.c_void_p()
        # The HCA object also backs the verbs wire: pre-created streams, the mapped result scratch, and the
        # device arena that holds the QpDev / CqDev views of adopted mlx5 queues.  ``device=None`` (verbs wire
        # only) is a host-only context: registration of host memory and host-posted verbs, no GPU needed
        # (BASELINE config 1: host-DRAM loopback between two ports).
        if device is None:
            if self.wire != "verbs":
                raise ValueError("a host-only context (device=None) needs wire='verbs'")
            h = None
        else:
            N.check(self._lib.rn_hca_open(device, max_mkeys, max_qps, arena_bytes, host_arena_bytes, C.byref(h)), "hca_open")
        self._h = h
        self.device = device
        if self.wire == "verbs":
            if self._lib.rn_verbs_available() <= 0:
                why = self._lib.rn_verbs_why().decode(errors="replace")
                if self._h:
                    self._lib.rn_hca_close(self._h)
                raise N.NativeError(f"wire='verbs' but no RDMA device is usable: {why}")
            name = nic.encode() if isinstance(nic, str) else b""
            index = nic if isinstance(nic, int) else (device or 0)
            self._vdev = self._lib.rn_verbs_open(name, index, port, gid_index)
            if not self._vdev:
                why = self._lib.rn_verbs_why().decode(errors="replace")
                if self._h:
                    self._lib.rn_hca_close(self._h)
                raise N.NativeError(f"cannot open the HCA: {why}")
            self.nic = self._lib.rn_verbs_dev_name(self._vdev).decode()
            self.nic_is_mock = bool(self._lib.rn_verbs_is_mock())
        self._mrs: List[MemoryRegion] = []
        self._closed = False
        self.last_engine_fatal = 0
        self._stream = None
        sz = C.c_uint64()
        self._scratch_ptr = self._lib.rn_hca_scratch(self._h, C.byref(sz)) if self._h else 0
        self._scratch_size = sz.value

    @property
    def aux_stream(self):
        """A second pre-created non-blocking stream (consumer kernels that must run
        concurrently with a producer on ``stream``).  Like ``stream`` it exists before any
        engine runs, because creating a stream stalls behind a resident engine."""
        if getattr(self, "_aux", None) is None:
            import torch
            self._aux = torch.cuda.ExternalStream(self._lib.rn_hca_aux_stream(self._h), device=self.device)
        return self._aux

    def streams(self, n: int):
        """The first ``n`` (<= 8) of the HCA's pre-created non-blocking streams (0 = ``stream``, 1 = ``aux_stream``)."""
        import torch
        if not 1 <= n <= 8:
            raise ValueError("1..8 streams are pre-created per context")
        if not hasattr(self, "_pool"):
            self._pool = {}
        out = []
        for i in range(n):
            if i == 0:
                out.append(self.stream)
            elif i == 1:
                out.append(self.aux_stream)
            else:
                if i not in self._pool:
                    self._pool[i] = torch.cuda.ExternalStream(self._lib.rn_hca_stream(self._h, i), device=self.device)
                out.append(self._pool[i])
        return out

    def dev_scratch(self, nbytes: int, offset: int = 0) -> int:
        """Address inside the HCA's zero-initialised device scratch (kernel counters; every
        kernel that uses it leaves it zeroed again)."""
        sz = C.c_uint64()
        base = self._lib.rn_hca_dev_scratch(self._h, C.byref(sz))
        if offset + nbytes > sz.value:
            raise ValueError("device scratch request too large")
        return base + offset

    def scratch(self, nbytes: int, offset: int = 0):
        """(address, ctypes view) of the HCA's mapped pinned result area.  Kernels write
        their status/timing words here and the host reads them after a stream sync, so the
        hot path performs no CUDA allocation or memcpy (either would stall behind the
        running engine kernel)."""
        if offset + nbytes > self._scratch_size:
            raise ValueError("scratch request too large")
        addr = self._scratch_ptr + offset
        return addr, (C.c_uint8 * nbytes).from_address(addr)

    @property
    def stream(self):
        """The context's non-blocking work stream (a ``torch.cuda.Stream``).

        Kernels that post to, or wait on, the engine MUST run on a non-blocking stream:
        a kernel launched on the legacy default stream is serialised behind the
        persistent engine kernel by the driver (observed with driver 580: the poster
        started 95 us after the engine's watchdog exit).  ``ops.*`` default to this
        stream; wrap torch work that must overlap the engine in
        ``with torch.cuda.stream(ctx.stream):``.
        """
        if self._stream is None:
            import torch
            # Created natively in rn_hca_open (before any engine runs): creating a stream
            # while the engine kernel is resident stalls until the engine exits.
            self._stream = torch.cuda.ExternalStream(self._lib.rn_hca_work_stream(self._h), device=self.device)
        return self._stream

    # ---- registration
    def classify(self, buf) -> str:
        """Where a buffer lives as the HCA sees it: device / pinned host / pageable host / managed."""
        ptr, _ = _ptr_len(buf, 1)
        dev = C.c_int(-1)
        return ["host", "device", "pinned_host", "managed"][self._lib.rn_classify_ptr(ptr, C.byref(dev))]

    def reg_mr(self, buf, nbytes=None, access: int = W.ACC_ALL, offset: int = 0, mode: str = "direct") -> MemoryRegion:
        """Register ``buf`` for RDMA.  ``mode="dmabuf"`` additionally exports the range as a dma-buf
        fd through the CUDA driver (``MemoryRegion.dmabuf_fd``) -- the handle an HCA takes in
        ``ibv_reg_dmabuf_mr`` -- which pins the GPU pages for as long as the region lives."""
        ptr, n = _ptr_len(buf, nbytes)
        if self.wire == "verbs":
            return self._verbs_reg_mr(buf, ptr + offset, n, access, mode)
        key = C.c_uint32()
        fd = C.c_int(-1)
        m = {"direct": 0, "dmabuf": 1, "peermem": 0, "auto": 0}[mode]
        N.check(self._lib.rn_reg_mr_mode(self._h, ptr + offset, n, access, m, C.byref(key), C.byref(fd)), "reg_mr")
        mr = MemoryRegion(self, ptr + offset, n, key.value, access, keepalive=buf)
        mr.dmabuf_fd = fd.value
        mr.mode = mode
        self._mrs.append(mr)
        return mr

    def _verbs_reg_mr(self, buf, ptr: int, n: int, access: int, mode: str) -> MemoryRegion:
        """``ibv_reg_dmabuf_mr`` on a dma-buf exported by the CUDA driver (``dmabuf``), or ``ibv_reg_mr`` on the pointer
        itself (``peermem`` / ``direct``: host memory, or HBM through a peer-memory client -- nvidia-peermem or
        ``kmod/b200p2p.ko``; the reference's whole purpose, amdp2p.c:363-371).  ``auto`` tries dma-buf first for device
        memory and falls back to the peer-memory path."""
        lk, rk = C.c_uint32(), C.c_uint32()
        is_dev = self.classify((ptr, 1)) == "device"
        order = {"auto": (["dmabuf", "peermem"] if is_dev else ["peermem"]), "dmabuf": ["dmabuf"], "peermem": ["peermem"],
                 "direct": ["peermem"]}[mode]
        errs = []
        for how in order:
            fd = -1
            if how == "dmabuf":
                lo, hi = ptr & ~4095, (ptr + n + 4095) & ~4095
                cu = C.c_int(0)
                self._lib.rn_set_device(self.device)
                fd = self._lib.rn_dmabuf_export(lo, hi - lo, C.byref(cu))
                if fd < 0:
                    errs.append(f"dmabuf: export failed (CUresult {cu.value})")
                    continue
                h = self._lib.rn_verbs_reg_mr(self._vdev, ptr, n, 1, fd, ptr - lo, access, C.byref(lk), C.byref(rk))
            else:
                h = self._lib.rn_verbs_reg_mr(self._vdev, ptr, n, 0, -1, 0, access, C.byref(lk), C.byref(rk))
            if h:
                mr = MemoryRegion(self, ptr, n, lk.value, access, keepalive=buf, rkey=rk.value, vmr=h)
                mr.dmabuf_fd, mr.mode = fd, how
                self._mrs.append(mr)
                return mr
            if fd >= 0:
                self._lib.rn_dmabuf_close(fd)
            errs.append(f"{how}: {self._lib.rn_verbs_why().decode(errors='replace')}")
        raise N.NativeError("reg_mr failed: " + "; ".join(errs))

    def sweep_revoked(self) -> int:
        """Driver-originated revocation: ask the CUDA driver whether the allocation behind every device-memory
        registration still exists (allocation id recorded at ``reg_mr``); registrations whose memory was freed --
        ``cudaFree``, ``torch.cuda.empty_cache()`` of the segment, or the address re-used by a new allocation -- are
        revoked (their MKey stops translating: a WQE that names it completes with a protection error instead of
        touching the address).  Returns how many were revoked now.  ``reg_mr(tensor)`` keeps a reference to the tensor,
        so this only ever fires for raw ``(ptr, nbytes)`` registrations or storage resized under the MR.
        The kernel-side counterpart is the free callback of ``kmod/b200p2p.c`` (reference: amdp2p.c:88-109)."""
        if self.wire != "softhca" or not self._h:
            return 0
        n = self._lib.rn_hca_sweep_revoked(self._h)
        if n < 0:
            raise N.NativeError(f"sweep_revoked failed ({n})")
        return n

    def watch_revocations(self, period_s: float = 0.05):
        """Start a daemon thread that calls :meth:`sweep_revoked` every ``period_s`` (the stand-in for an asynchronous
        free callback when nobody on the host touches the context between a free and the next GPU-posted WQE)."""
        import threading
        if getattr(self, "_watch", None):
            return
        stop = threading.Event()

        def run():
            while not stop.wait(period_s):
                if self._closed:
                    return
                try:
                    self.sweep_revoked()
                except Exception:
                    return
        t = threading.Thread(target=run, daemon=True)
        self._watch = (t, stop)
        t.start()

    def enable_peer(self, peer_device: int):
        """Allow this context's GPU to reach ``peer_device``'s memory over NVLink (needed before
        connecting a QP to a QP of a context that lives on that GPU)."""
        N.check(self._lib.rn_hca_enable_peer(self._h, peer_device), "enable_peer")

    # ---- queues
    def create_cq(self, depth: int = 1024, mem: int = W.MEM_DEVICE) -> CompletionQueue:
        """``ibv_create_cq``; ``mem`` = ``wire.MEM_DEVICE`` (GPU pollers) or ``wire.MEM_HOST_PINNED`` (CPU pollers)."""
        if self.wire == "verbs":
            vc = self._lib.rn_verbs_create_cq(self._vdev, depth)
            if not vc:
                raise N.NativeError("ibv_create_cq failed: " + self._lib.rn_verbs_why().decode(errors="replace"))
            cq = CompletionQueue(self, None, depth, mem, vcq=vc)
            self._vcqs.append(cq)
            return cq
        c = C.c_void_p()
        N.check(self._lib.rn_create_cq(self._h, depth, mem, C.byref(c)), "create_cq")
        return CompletionQueue(self, c, depth, mem)

    def create_qp(self, scq: CompletionQueue, rcq: Optional[CompletionQueue] = None, sq_depth: int = 256,
                  rq_depth: int = 256, sq_mem: int = W.MEM_DEVICE, chunk_bytes: int = 512 << 10) -> QueuePair:
        """``ibv_create_qp`` (RC).  ``sq_mem`` places the rings and doorbells in device memory (posted by kernels) or pinned host memory (posted by the CPU); ``chunk_bytes`` is the engine's minimum work granule for this QP."""
        q = C.c_void_p()
        rcq = rcq or scq
        if self.wire == "verbs":
            vq = self._lib.rn_verbs_create_qp(self._vdev, scq._vcq, rcq._vcq, sq_depth, rq_depth)
            if not vq:
                raise N.NativeError("ibv_create_qp failed: " + self._lib.rn_verbs_why().decode(errors="replace"))
            qp = VerbsQueuePair(self, vq, scq, rcq, sq_depth, rq_depth, sq_mem)
            self._vqps.append(qp)
            return qp
        N.check(self._lib.rn_create_qp(self._h, scq._c, rcq._c, sq_depth, rq_depth, sq_mem, chunk_bytes, C.byref(q)),
                "create_qp")
        return QueuePair(self, q, scq, rcq, sq_depth, rq_depth, sq_mem)

    def loopback_qp(self, depth: int = 256, mem: int = W.MEM_DEVICE, chunk_bytes: int = 512 << 10,
                    cq_depth: Optional[int] = None, shared_cq: bool = False) -> QueuePair:
        """A QP connected to itself: the single-GPU wire of configs 2, 3 and 5.  ``mem=MEM_DEVICE`` makes it a
        GPU-posted QP (on the verbs wire: the mlx5 queues are handed to the GPU), ``MEM_HOST_PINNED`` a
        host-posted one.  Send and receive completions get separate CQs unless ``shared_cq`` (a shared CQ needs
        both of its consumers running: each leaves the other's CQEs at the head)."""
        n = cq_depth or max(2 * depth, 64)
        scq = self.create_cq(n, mem)
        rcq = scq if shared_cq else self.create_cq(n, mem)
        return self.create_qp(scq, rcq, depth, depth, mem, chunk_bytes).connect()

    # ---- engine
    def engine_start(self, ctas: int = 32, idle_timeout_ms: int = 5000, rnr_timeout_ms: int = 500):
        """Launch the persistent DMA engine on ``ctas`` SMs.  Allocate and register everything first: cudaMalloc, stream creation and first-time kernel loads all wait for a resident kernel (DESIGN.md 3.2).  It leaves by itself after ``idle_timeout_ms`` without work."""
        if self.wire == "verbs":
            return                      # the NIC is the engine
        N.check(self._lib.rn_engine_start(self._h, ctas, idle_timeout_ms, rnr_timeout_ms), "engine_start")

    def engine_run_oneshot(self, ctas: int = 32):
        """Launch the engine, let it execute everything already posted, return when it has
        drained and exited.  For profilers (ncu serialises kernels, so a resident engine and a
        poster can never overlap there) and for host-posted batch transfers."""
        if self.wire == "verbs":
            return
        self._lib.rn_engine_set_oneshot(self._h, 1)
        try:
            N.check(self._lib.rn_engine_start(self._h, ctas, 2000, 500), "engine_start")
            N.check(self._lib.rn_engine_wait(self._h), "engine_wait")
            self._report_engine_fault()
        finally:
            self._lib.rn_engine_set_oneshot(self._h, 0)

    def engine_stop(self):
        """Ask the engine to leave and wait for it; reports an engine fault as a RuntimeWarning."""
        if self.wire == "verbs":
            return
        N.check(self._lib.rn_engine_stop(self._h), "engine_stop")
        self._report_engine_fault()

    def _report_engine_fault(self):
        """Failure detection: the engine bails out (instead of wedging an SM) when a bulk copy never completes
        (1) or a CTA that held the commit turn died (2); the host learns it here."""
        try:
            fatal = self.engine_stats()["fatal"]
        except Exception:
            return
        self.last_engine_fatal = fatal
        if fatal:
            import warnings
            warnings.warn(f"rocnrdma_b200: the DMA engine stopped after a fatal fault (code {fatal}: "
                          f"{'a TMA bulk copy never completed (bad mapping?)' if fatal == 1 else 'ordered-commit predecessor lost'}); "
                          "outstanding work requests were not completed", RuntimeWarning, stacklevel=3)

    @property
    def engine_running(self) -> bool:
        """True while the engine kernel is resident."""
        return bool(self._lib.rn_engine_running(self._h))

    def engine_stats(self) -> dict:
        """Engine-wide counters: bulk chunks moved, start / exit %globaltimer, CTAs, idle-exit and fatal flags."""
        s = N.RnEngineStats()
        N.check(self._lib.rn_engine_stats(self._h, C.byref(s)), "engine_stats")
        return {k: getattr(s, k) for k, _ in s._fields_}

    def mkey_table_ptr(self) -> int:
        """Device address of this HCA's MKey table (what a peer's engine translates rkeys with)."""
        return self._lib.rn_hca_mkey_table(self._h)

    def close(self):
        """Stop the engine and free the HCA (queues, CQs, control arenas).  Registered tensors are untouched."""
        if not self._closed:
            self._closed = True
            if getattr(self, "_watch", None):
                self._watch[1].set()
            if self._vdev:
                for q in self._vqps:
                    q.destroy()
                for mr in list(self._mrs):
                    try:
                        mr.dereg()
                    except Exception:
                        pass
                for cq in self._vcqs:
                    if cq._vcq:
                        self._lib.rn_verbs_destroy_cq(cq._vcq)
                        cq._vcq = None
                self._lib.rn_verbs_close(self._vdev)
                self._vdev = None
            if self._h:
                self._lib.rn_hca_close(self._h)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
