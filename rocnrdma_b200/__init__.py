"""rocnrdma_b200 -- a Hopper-native (H100) GPU<->NIC zero-copy RDMA stack.

Capability-for-capability rebuild of AMD's ``amdp2p`` PeerDirect bridge
(rocmarchive/ROCnRDMA) for NVIDIA H100: registration of GPU HBM for RDMA
(kernel ``peer_memory_client`` on nv-p2p + userspace dma-buf exporter), the
``amdp2ptest`` harness (ioctl ABI, kernel module, userspace twin, CLI), and --
new here -- a GPU-initiated data path: sm_90a kernels build mlx5 WQEs, ring the
doorbell and poll the CQ on the device, fused with a bf16->fp8 block-scaled pack
or a wgmma/TMA GEMM that produces the send tile.
"""
from . import wire  # noqa: F401
from .wire import (ACC_ALL, ACC_LOCAL_WRITE, ACC_REMOTE_READ, ACC_REMOTE_WRITE, MEM_DEVICE,  # noqa: F401
                   MEM_HOST_PINNED, OP_RDMA_READ, OP_RDMA_WRITE, OP_SEND)

__version__ = "0.1.0"


def __getattr__(name):
    # Heavy imports (torch, the native library) are deferred so that the wire-format
    # and config layers stay importable on a machine without CUDA.
    if name in ("Context", "MemoryRegion", "QueuePair", "CompletionQueue", "WorkCompletion"):
        from . import api
        return getattr(api, name)
    if name in ("ops", "models", "parallel", "utils", "api", "config", "probe"):
        import importlib
        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
