"""Connect a local QP to a QP that lives in another process / on another GPU of the same node.

What two nodes exchange out of band to bring up an RC connection -- QP number, rkeys, buffer addresses --
is exchanged here through ``torch.distributed`` (any backend), plus CUDA IPC handles so that the requester's
DMA engine can reach the responder's HCA state (MKey table, receive ring, receive CQ) and its registered
buffers over NVLink.  After ``connect_to`` the remote side is described to the local engine exactly like a
loopback peer: already-translated pointers in a ``RemoteView``.

There is no counterpart in the reference (it has no connection management: SURVEY.md section 2.2).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional

from .. import _native as N
from .. import wire as W


@dataclass
class PeerInfo:
    """Everything a rank publishes about one of its QPs (picklable)."""
    rank: int
    device: int
    arena_handle: bytes
    arena_base: int
    arena_size: int
    qpn: int
    rq: int
    rq_dbr: int
    rq_log: int
    rcq: int
    rcq_buf: int
    n_mkeys: int
    mrs: List[dict] = field(default_factory=list)     # key, addr, length, access, ipc handle, alloc_base, alloc_size


@dataclass
class RemoteMR:
    """A peer's memory region as seen by a requester: put ``addr``/``rkey`` into WQEs."""
    addr: int
    length: int
    rkey: int
    lkey: int = 0
    key: int = 0

    def __post_init__(self):
        self.key = self.rkey


def _export(ptr: int):
    lib = N.load()
    h = (C.c_uint8 * 64)()
    base, size = C.c_uint64(), C.c_uint64()
    N.check(lib.rn_ipc_export(ptr, h, C.byref(base), C.byref(size)), "ipc_export")
    return bytes(h), base.value, size.value


def describe_local(ctx, qp, mrs, rank: int = 0) -> PeerInfo:
    """Publishable description of ``qp`` and of the regions peers may target."""
    lib = N.load()
    lib.rn_set_device(ctx.device)
    asz = C.c_uint64()
    abase = lib.rn_hca_arena(ctx._h, C.byref(asz))
    ah, ab, _ = _export(abase)
    d = qp.describe()
    info = PeerInfo(rank=rank, device=ctx.device, arena_handle=ah, arena_base=ab, arena_size=asz.value, qpn=d.qpn, rq=d.rq,
                    rq_dbr=d.rq_dbr, rq_log=d.rq_log, rcq=d.rcq, rcq_buf=d.rcq_buf, n_mkeys=d.n_rkeys)
    for mr in mrs:
        h, b, s = _export(mr.addr)
        info.mrs.append(dict(key=mr.key, addr=mr.addr, length=mr.length, access=mr.access, handle=h, alloc_base=b, alloc_size=s))
    return info


def connect_to(ctx, qp, peer: PeerInfo) -> Dict[int, RemoteMR]:
    """Map the peer's HCA arena and buffers, build the translated remote view, bring ``qp`` to RTS.
    Returns the peer's regions keyed by their rkey."""
    lib = N.load()
    lib.rn_set_device(ctx.device)
    mapped = C.c_uint64()
    N.check(lib.rn_ipc_open(ctx._h, (C.c_uint8 * 64)(*peer.arena_handle), C.byref(mapped)), "ipc_open(arena)")
    delta = mapped.value - peer.arena_base

    def tr(p):
        if not (peer.arena_base <= p < peer.arena_base + peer.arena_size):
            raise ValueError("peer pointer outside its exported arena (host-resident rings cannot be shared across processes)")
        return p + delta

    n = max([m["key"] >> 8 for m in peer.mrs] + [0]) + 1
    table = lib.rn_hca_alloc_remote_table(ctx._h, n)
    if not table:
        raise N.NativeError("control arena exhausted (remote MKey table)")
    out: Dict[int, RemoteMR] = {}
    opened: Dict[bytes, int] = {}
    for m in peer.mrs:
        if m["handle"] not in opened:
            mb = C.c_uint64()
            N.check(lib.rn_ipc_open(ctx._h, (C.c_uint8 * 64)(*m["handle"]), C.byref(mb)), "ipc_open(mr)")
            opened[m["handle"]] = mb.value
        map_base = opened[m["handle"]] + (m["addr"] - m["alloc_base"])
        N.check(lib.rn_hca_set_remote_mkey(ctx._h, table, m["key"] >> 8, m["addr"], m["length"], map_base, m["key"], m["access"]),
                "set_remote_mkey")
        out[m["key"]] = RemoteMR(addr=m["addr"], length=m["length"], rkey=m["key"])
    r = N.RnRemote(rkeys=table, n_rkeys=n, qpn=peer.qpn, rq=tr(peer.rq), rq_dbr=tr(peer.rq_dbr), rq_log=peer.rq_log, pad=0,
                   rcq=tr(peer.rcq), rcq_buf=tr(peer.rcq_buf))
    qp.modify(W.QPS_INIT)
    qp.connect_remote(r)
    qp.modify(W.QPS_RTR)
    qp.modify(W.QPS_RTS)
    qp.set_flags(sys_scope=True)          # the responder is another GPU
    qp._peer_maps = (mapped.value, opened)
    return out


def connect_ring(ctx, qp, mrs, group=None, describe=None, connect=None):
    """All ranks call this: rank r's QP is connected to rank (r+1) % world's QP.  Returns
    (next_rank, {rkey: RemoteMR}) describing what this rank may write to / read from.
    ``describe`` / ``connect`` default to ``describe_local`` / ``connect_to``; the CPU test of the rendezvous
    (gloo, two processes) substitutes GPU-free stand-ins."""
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    me = (describe or describe_local)(ctx, qp, mrs, rank)
    infos: List[Optional[PeerInfo]] = [None] * world
    dist.all_gather_object(infos, me, group=group)
    nxt = (rank + 1) % world
    if infos[nxt] is None or infos[nxt].rank != nxt:
        raise RuntimeError(f"rank {rank}: rendezvous returned no description for rank {nxt}")
    remote = (connect or connect_to)(ctx, qp, infos[nxt])
    dist.barrier(group=group)           # everybody is mapped before anybody starts writing
    return nxt, remote


def connect_mesh(ctx, send_qps, recv_qps, mrs, group=None, describe=None, connect=None):
    """All ranks call this: the full mesh of an all-to-all.  ``send_qps[d]`` and ``recv_qps[s]`` are this rank's queue
    pairs to rank d and from rank s (entry ``rank`` of each is ignored).  Every rank publishes one description per
    receive QP, with ``mrs``, and connects its send QP for rank d to rank d's receive QP for this rank.  Returns ``{d:
    {rkey: RemoteMR}}``: what this rank may write to on each peer.  ``describe`` / ``connect`` as in
    :func:`connect_ring`."""
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if len(send_qps) != world or len(recv_qps) != world:
        raise ValueError(f"send_qps and recv_qps: one entry per rank ({world})")
    mine = {s: (describe or describe_local)(ctx, recv_qps[s], mrs, rank) for s in range(world) if s != rank}
    infos: List[Optional[Dict[int, PeerInfo]]] = [None] * world
    dist.all_gather_object(infos, mine, group=group)
    remote: Dict[int, Dict[int, RemoteMR]] = {}
    for d in range(world):
        if d == rank:
            continue
        info = (infos[d] or {}).get(rank)
        if info is None or info.rank != d:
            raise RuntimeError(f"rank {rank}: rendezvous returned no description of rank {d}'s receive queue pair for it")
        remote[d] = (connect or connect_to)(ctx, send_qps[d], info)
    dist.barrier(group=group)           # everybody is mapped before anybody starts writing
    return remote
