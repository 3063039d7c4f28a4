"""Roofline arithmetic against measured peaks (MEASURED_PEAKS.json, when a run has written one) or the H100 SXM data sheet."""
from __future__ import annotations

import json
from pathlib import Path

# NVIDIA H100 SXM data sheet (700 W board): 3.35 TB/s HBM3, 989 TFLOP/s dense bf16.  Not measured: a card run at a lower
# power limit reaches less.
FALLBACK = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "_source": "fallback"}
NIC_LINE_RATE_GBS = 50.0          # ConnectX-7, 400 Gb/s per direction
PCIE_GEN5_X16_GBS = 63.0          # raw, per direction
NVLINK_PEER_GBS = 450.0           # H100 SXM NVLink 4, per direction (data sheet: 900 GB/s total)


def measured_peaks(repo_root=None) -> dict:
    root = Path(repo_root) if repo_root else Path(__file__).resolve().parents[2]
    p = root / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        d["_source"] = "measured"
        return d
    return dict(FALLBACK)


def copy_roofline_gbps(peaks=None) -> float:
    """Payload GB/s a device-local copy can reach: the measured figure counts read+write bytes."""
    peaks = peaks or measured_peaks()
    return peaks["hbm_gbs"] / 2.0


def fused_pack_roofline_gbps(peaks=None, wire_gbs: float = None) -> float:
    """Source-bf16 GB/s bound of the fused pack + write.  HBM side: the pack's ALGORITHMIC traffic -- 2 B read and
    (1 + 1/32) B written per element -- at the measured copy peak.  (Round 1 also charged the DMA engine's re-read and
    write of the staged records to HBM, 5.09 B per 2 B of source; the 4 MiB records are L2-resident when the engine
    picks them up, ncu shows DRAM traffic equal to the algorithmic bytes, and the fraction came out above 1.)
    With a real wire the bound is min(that, wire * 2 / 1.03)."""
    peaks = peaks or measured_peaks()
    hbm = peaks["hbm_gbs"] * 2.0 / (2.0 + (1 + 1 / 32))
    if wire_gbs:
        return min(hbm, wire_gbs * 2.0 / (1 + 1 / 32))
    return hbm


def fraction(achieved: float, bound: float) -> float:
    return achieved / bound if bound else float("nan")
