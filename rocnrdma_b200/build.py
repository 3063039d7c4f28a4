"""In-tree native build: nvcc -> rocnrdma_b200/lib/librocnrdma_b200.so (sm_90a only: H100).

The shared object exports a flat C ABI (``rn_*``) that ``rocnrdma_b200._native``
loads with ctypes; keeping torch's C++ headers out of the build keeps a full
rebuild to well under a minute and the .so free of ABI coupling to the torch
wheel.  Replaces the reference's kbuild Makefiles for the userspace half
(Makefile:1-71, tests/Makefile:1-69); the kernel modules keep real kbuild
Makefiles under ``kmod/``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIBDIR = ROOT / "lib"
LIB = LIBDIR / "librocnrdma_b200.so"

CUDA_SOURCES = [
    "hca/hca_host.cu",
    "kernels/rdma_ops.cu",
    "kernels/pack_fp8.cu",
    "kernels/gemm_send.cu",
    "kernels/gemm_mxfp8.cu",
]
CXX_SOURCES = [
    "reg/registration.cc",
    "reg/p2ptest_user.cc",
    "verbs/verbs_dl.cc",
]
# The mock rdma-core provider (csrc/mockverbs): separate shared objects with the real sonames, loaded by
# verbs_dl.cc through ROCNRDMA_VERBS_LIBDIR exactly like the system libraries would be.
MOCKDIR = LIBDIR / "mock"
MOCK_VERBS = MOCKDIR / "libibverbs.so.1"
MOCK_MLX5 = MOCKDIR / "libmlx5.so.1"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _cuda_home() -> Path:
    return Path(_nvcc()).resolve().parent.parent


def _stamp(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(str(p).encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS + CXX_FLAGS).encode())
    return h.hexdigest()


def sources():
    cu = [CSRC / s for s in CUDA_SOURCES]
    cc = [CSRC / s for s in CXX_SOURCES]
    missing = [str(p) for p in cu + cc if not p.exists()]
    if missing:
        raise RuntimeError(f"native sources listed in build.py do not exist: {missing}")
    return cu, cc


def build_mock() -> Path:
    """lib/mock/libibverbs.so.1 + libmlx5.so.1: the in-tree stand-in for rdma-core (host code only)."""
    MOCKDIR.mkdir(parents=True, exist_ok=True)
    subprocess.run(["g++", *CXX_FLAGS, "-I", str(CSRC), "-shared", "-Wl,-soname,libibverbs.so.1", "-o", str(MOCK_VERBS),
                    str(CSRC / "mockverbs" / "mock_verbs.cc"), "-ldl", "-lpthread"], check=True)
    subprocess.run(["g++", *CXX_FLAGS, "-I", str(CSRC), "-shared", "-Wl,-soname,libmlx5.so.1", "-Wl,-rpath,$ORIGIN", "-o", str(MOCK_MLX5),
                    str(CSRC / "mockverbs" / "mock_mlx5.cc"), "-L", str(MOCKDIR), "-l:libibverbs.so.1"], check=True)
    return MOCKDIR


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every native source for sm_90a and link the shared object."""
    cu, cc = sources()
    headers = list(CSRC.rglob("*.h")) + list(CSRC.rglob("*.cuh"))
    mock_srcs = sorted((CSRC / "mockverbs").glob("*.cc"))
    stamp = _stamp(cu + cc + headers + mock_srcs)
    stamp_file = LIBDIR / ".build_stamp"
    if not force and LIB.exists() and MOCK_VERBS.exists() and MOCK_MLX5.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return LIB
    LIBDIR.mkdir(exist_ok=True)
    objdir = LIBDIR / "obj"
    objdir.mkdir(exist_ok=True)
    nvcc = _nvcc()
    cuda_inc = _cuda_home() / "include"
    objs = []
    procs = []
    logs = {}
    for src in cu:
        obj = objdir / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src in cc:
        obj = objdir / (src.stem + ".o")
        cmd = ["g++", *CXX_FLAGS, "-I", str(CSRC), "-I", str(cuda_inc), "-c", str(src), "-o", str(obj)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        logs[src.name] = out
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- {src} FAILED\n{out}\n")
        elif verbose:
            sys.stderr.write(f"--- {src}\n{out}\n")
    if failed:
        raise RuntimeError("native build failed")
    # register / shared-memory / spill summary per kernel (tracked: it is evidence); compile times are noise
    keep = lambda v: "\n".join(l for l in v.splitlines() if "Compile time" not in l)
    (LIBDIR / "ptxas_info.txt").write_text("\n".join(f"=== {k}\n{keep(v)}" for k, v in logs.items()))
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs),
            "-Xcompiler", "-fPIC", "-ldl", "-lpthread"]
    subprocess.run(link, check=True)
    build_mock()
    stamp_file.write_text(stamp)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
