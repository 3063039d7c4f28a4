"""The all-to-all's out-of-band exchange (``parallel.peer.connect_mesh``) over a real process group: gloo, 3 processes,
no GPU.  The CUDA-IPC parts are replaced by stand-ins, as in test_peer_rendezvous.py; what is tested is who connects to
whom: rank q's send queue pair for rank d must be connected to rank d's receive queue pair for q, with rank d's regions,
and to nothing else."""
import json
import os
import socket
import subprocess
import sys
import textwrap

import pytest

WORKER = textwrap.dedent('''
    import os, sys, json
    import torch.distributed as dist
    sys.path.insert(0, os.environ["RN_REPO"])
    from rocnrdma_b200.parallel import peer

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{os.environ['MASTER_PORT']}", rank=rank, world_size=world)

    # queue pairs are plain labels here: ("send", owner, peer) / ("recv", owner, peer); the qpn names the receive QP
    def describe(ctx, qp, mrs, r):
        kind, owner, src = qp
        assert kind == "recv" and owner == r == rank
        info = peer.PeerInfo(rank=r, device=r, arena_handle=bytes([r]) * 64, arena_base=0x7000_0000_0000 + (r << 32),
                             arena_size=1 << 24, qpn=1000 * r + src, rq=0, rq_dbr=0, rq_log=8, rcq=0, rcq_buf=0, n_mkeys=64)
        for k, (addr, length) in enumerate(mrs):
            info.mrs.append(dict(key=((k + 1) << 8) | r, addr=addr, length=length, access=0xf, handle=bytes([0x80 | r]) * 64,
                                 alloc_base=addr & ~0xfffff, alloc_size=1 << 21))
        return info

    links = []
    def connect(ctx, qp, info):
        links.append(dict(qp=list(qp), peer_rank=info.rank, qpn=info.qpn, arena_ok=info.arena_handle == bytes([info.rank]) * 64))
        return {m["key"]: peer.RemoteMR(addr=m["addr"], length=m["length"], rkey=m["key"]) for m in info.mrs}

    send = [None if d == rank else ("send", rank, d) for d in range(world)]
    recv = [None if s == rank else ("recv", rank, s) for s in range(world)]
    mrs = [(0x7f00_0000_0000 + (rank << 30), 1 << 20)]
    remote = peer.connect_mesh(None, send, recv, mrs, describe=describe, connect=connect)
    out = dict(rank=rank, links=links, remote={str(d): [[k, v.addr] for k, v in m.items()] for d, m in remote.items()})
    print("RESULT " + json.dumps(out), flush=True)
    dist.destroy_process_group()
''')


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_mesh_rendezvous_over_gloo_three_processes(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    world, port = 3, _free_port()
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RN_REPO=repo,
                   CUDA_VISIBLE_DEVICES="")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    results = {}
    for r, p in enumerate(procs):
        try:
            out, err = p.communicate(timeout=180)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            pytest.fail("rendezvous timed out")
        assert p.returncode == 0, err[-2000:]
        line = [l for l in out.splitlines() if l.startswith("RESULT ")][-1]
        results[r] = json.loads(line[len("RESULT "):])
    for q in range(world):
        res = results[q]
        peers = [d for d in range(world) if d != q]
        # one connection per peer, from the send QP for d to d's receive QP for q
        assert sorted(l["peer_rank"] for l in res["links"]) == peers
        for link in res["links"]:
            d = link["peer_rank"]
            assert link["qp"] == ["send", q, d] and link["qpn"] == 1000 * d + q and link["arena_ok"]
        assert sorted(int(d) for d in res["remote"]) == peers
        for d in peers:
            assert res["remote"][str(d)] == [[(1 << 8) | d, 0x7f00_0000_0000 + (d << 30)]]
