"""N0: environment probe -- which GPUs, which HCAs, how they are wired, and which data paths can run.

Replaces the reference's build-time "is OFED / KFD present?" checks (Makefile:2-8, :23-28) with a
run-time answer, because on this platform the same binary meets three different worlds: a host with
ConnectX + rdma-core (real verbs wire), a container that sees the HCAs only in sysfs (this project's GPU
box: no /dev/infiniband, no libibverbs), and a CPU-only dev box.

    python -m rocnrdma_b200.probe            # human table
    python -m rocnrdma_b200.probe --json
"""
from __future__ import annotations

import ctypes.util
import functools
import glob
import json
import os
import re
from dataclasses import asdict, dataclass, field
from typing import Dict, List, Optional

SYS = os.environ.get("ROCNRDMA_SYSFS_ROOT", "/sys")


def _read(path: str, default: str = "") -> str:
    try:
        with open(path) as f:
            return f.read().strip()
    except OSError:
        return default


@dataclass
class Hca:
    name: str
    pci: str = ""
    numa: int = -1
    node_type: str = ""
    ports: Dict[str, dict] = field(default_factory=dict)
    uverbs: str = ""
    pci_path: List[str] = field(default_factory=list)

    @property
    def active(self) -> bool:
        return any("ACTIVE" in p.get("state", "") for p in self.ports.values())

    @property
    def rate_gbps(self) -> float:
        best = 0.0
        for p in self.ports.values():
            m = re.match(r"([\d.]+)\s*Gb/sec", p.get("rate", ""))
            if m:
                best = max(best, float(m.group(1)))
        return best


@dataclass
class Gpu:
    index: int
    pci: str
    name: str = ""
    numa: int = -1
    pci_path: List[str] = field(default_factory=list)
    caps: Dict[str, bool] = field(default_factory=dict)


def _pci_path(pci: str) -> List[str]:
    """Bridge chain from the root complex down to the device (from the sysfs device symlink)."""
    try:
        real = os.path.realpath(f"{SYS}/bus/pci/devices/{pci}")
    except OSError:
        return []
    return [p for p in real.split("/") if re.match(r"^[0-9a-f]{4}:[0-9a-f]{2}:[0-9a-f]{2}\.[0-9a-f]$", p) or p.startswith("pci")]


def list_hcas() -> List[Hca]:
    out = []
    for d in sorted(glob.glob(f"{SYS}/class/infiniband/*")):
        h = Hca(name=os.path.basename(d))
        real = os.path.realpath(d)
        m = re.findall(r"[0-9a-f]{4}:[0-9a-f]{2}:[0-9a-f]{2}\.[0-9a-f]", real)
        h.pci = m[-1] if m else ""
        h.pci_path = _pci_path(h.pci) if h.pci else []
        h.numa = int(_read(f"{SYS}/bus/pci/devices/{h.pci}/numa_node", "-1") or -1) if h.pci else -1
        h.node_type = _read(f"{d}/node_type")
        for p in sorted(glob.glob(f"{d}/ports/*")):
            h.ports[os.path.basename(p)] = {"state": _read(f"{p}/state"), "rate": _read(f"{p}/rate"),
                                            "link_layer": _read(f"{p}/link_layer"), "lid": _read(f"{p}/lid")}
        for u in glob.glob(f"{SYS}/class/infiniband_verbs/uverbs*"):
            if _read(f"{u}/ibdev") == h.name:
                h.uverbs = os.path.basename(u)
        out.append(h)
    return out


def list_gpus() -> List[Gpu]:
    gpus: List[Gpu] = []
    try:
        import torch
        if not torch.cuda.is_available():
            return gpus
        from . import _native as N
        lib = N.load()
        import ctypes as C
        for i in range(torch.cuda.device_count()):
            buf = C.create_string_buffer(32)
            lib.rn_device_pci(i, buf, 32)
            pci = buf.value.decode().lower()
            pci = pci[-12:] if len(pci) > 12 else pci            # "00000000:53:00.0" -> "0000:53:00.0"
            caps = lib.rn_device_caps(i)
            g = Gpu(index=i, pci=pci, name=torch.cuda.get_device_name(i),
                    numa=int(_read(f"{SYS}/bus/pci/devices/{pci}/numa_node", "-1") or -1), pci_path=_pci_path(pci),
                    caps={"dmabuf": bool(caps & 1), "gpudirect_rdma": bool(caps & 2), "vmm": bool(caps & 4), "posix_fd": bool(caps & 8)})
            gpus.append(g)
    except Exception:
        pass
    return gpus


def pci_distance(a: List[str], b: List[str]) -> str:
    """nvidia-smi topo style relation of two PCI paths: PIX (same switch) < PXB < PHB/NODE < SYS."""
    if not a or not b:
        return "UNKNOWN"
    common = 0
    for x, y in zip(a, b):
        if x != y:
            break
        common += 1
    if common == 0:
        return "SYS"
    up_a, up_b = len(a) - common, len(b) - common
    if common >= 2 and up_a <= 2 and up_b <= 2:
        return "PIX"
    if common >= 2:
        return "PXB"
    return "NODE"


_ORDER = {"PIX": 0, "PXB": 1, "NODE": 2, "PHB": 2, "SYS": 3, "UNKNOWN": 4}


def affinity(gpus: List[Gpu], hcas: List[Hca]) -> Dict[int, Optional[str]]:
    """Closest active InfiniBand-class HCA for every GPU (the reference's one performance rule:
    GPU and HCA on the same root complex, README.md:71-72)."""
    out: Dict[int, Optional[str]] = {}
    for g in gpus:
        best, best_rank = None, 99
        for h in hcas:
            if not h.ports:
                continue
            rel = pci_distance(g.pci_path, h.pci_path)
            rank = _ORDER[rel] * 2 + (0 if h.active else 1)
            if h.numa >= 0 and g.numa >= 0 and h.numa != g.numa:
                rank += 4
            if rank < best_rank:
                best, best_rank = h.name, rank
        out[g.index] = best
    return out


def capabilities() -> dict:
    has_lib = ctypes.util.find_library("ibverbs") is not None
    dev_nodes = sorted(glob.glob("/dev/infiniband/uverbs*"))
    caps = {
        "has_hca_sysfs": bool(glob.glob(f"{SYS}/class/infiniband/*")),
        "has_uverbs_dev": bool(dev_nodes),
        "has_libibverbs": has_lib,
        "has_peermem": os.path.isdir(f"{SYS}/module/nvidia_peermem"),
        "peermem_version": _read(f"{SYS}/module/nvidia_peermem/version"),
        "has_gdrdrv": os.path.isdir(f"{SYS}/module/gdrdrv"),
        "has_b200p2p": os.path.isdir(f"{SYS}/module/b200p2p"),
        "has_b200p2ptest_dev": os.path.exists("/dev/b200p2ptest"),
        "can_load_modules": os.path.isdir("/lib/modules") and os.geteuid() == 0,
        "iommu_groups": len(glob.glob(f"{SYS}/kernel/iommu_groups/*")),
    }
    caps["has_verbs"] = caps["has_uverbs_dev"] and caps["has_libibverbs"]
    return caps


@functools.lru_cache(maxsize=None)
def dmabuf_export_works(device: int = 0) -> bool:
    """Whether the CUDA driver exports device memory as a dma-buf here (cuMemGetHandleForAddressRange).  The device
    attribute is not enough: a driver can report support and still refuse the export."""
    import ctypes as C
    import torch
    from . import _native as N
    lib = N.load()
    lib.rn_set_device(device)
    t = torch.empty(4 << 20, dtype=torch.uint8, device=f"cuda:{device}")
    cu = C.c_int(0)
    fd = lib.rn_dmabuf_export((t.data_ptr() + 65535) & ~65535, 1 << 20, C.byref(cu))
    if fd < 0:
        return False
    lib.rn_dmabuf_close(fd)
    return True


def choose_wire(caps: dict, n_gpus: int) -> dict:
    """Registration mode, post mode and wire backend the stack will use here (SURVEY.md section 7.1 branches)."""
    if caps.get("has_verbs"):
        return {"wire": "verbs", "registration": "peermem" if caps.get("has_peermem") or caps.get("has_b200p2p") else "dmabuf",
                "post": "gpu", "why": "ConnectX reachable through libibverbs"}
    why = []
    if caps.get("has_hca_sysfs") and not caps.get("has_uverbs_dev"):
        why.append("HCAs visible in sysfs but /dev/infiniband is not exposed to this container")
    if not caps.get("has_libibverbs"):
        why.append("no rdma-core userspace")
    if n_gpus == 0:
        return {"wire": "none", "registration": "none", "post": "none", "why": "; ".join(why + ["no GPU"])}
    return {"wire": "softhca", "registration": "dmabuf", "post": "gpu", "why": "; ".join(why) or "no HCA"}


def probe() -> dict:
    gpus, hcas = list_gpus(), list_hcas()
    caps = capabilities()
    aff = affinity(gpus, hcas)
    return {"gpus": [asdict(g) for g in gpus], "hcas": [dict(asdict(h), active=h.active, rate_gbps=h.rate_gbps) for h in hcas],
            "affinity": aff, "capabilities": caps, "plan": choose_wire(caps, len(gpus))}


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--json", action="store_true")
    a = ap.parse_args(argv)
    r = probe()
    if a.json:
        print(json.dumps(r, indent=1))
        return 0
    print(f"GPUs: {len(r['gpus'])}   HCAs: {len(r['hcas'])}")
    for g in r["gpus"]:
        print(f"  GPU{g['index']} {g['name']} {g['pci']} numa={g['numa']} caps={[k for k, v in g['caps'].items() if v]} -> HCA {r['affinity'].get(g['index'])}")
    for h in r["hcas"]:
        print(f"  {h['name']:8s} {h['pci']} numa={h['numa']} active={h['active']} rate={h['rate_gbps']} Gb/s uverbs={h['uverbs'] or '-'}")
    print("capabilities:", {k: v for k, v in r["capabilities"].items()})
    print("plan:", r["plan"])
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
