import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# The ConnectX backend dlopen()s libibverbs once per process: point it at the in-tree mock provider before
# anything loads it (no rdma-core in the image, no /dev/infiniband in the sandbox).  `wire="auto"` never
# selects the mock, so the softhca tests are unaffected.
os.environ.setdefault("ROCNRDMA_VERBS_LIBDIR", os.path.join(ROOT, "rocnrdma_b200", "lib", "mock"))


def _private_kmod_sim():
    """The mock's peer-memory bridge gets its OWN copy of the kmod simulation: test_kmod_sim.py resets and
    reloads the shared one freely, and a dlopen of the same path would share its globals."""
    import shutil
    import tempfile
    try:
        from tools import build_kmod_sim
        src = build_kmod_sim.build()
    except Exception:
        return
    d = tempfile.mkdtemp(prefix="rn_kmod_sim_")
    dst = os.path.join(d, "libb200p2p_sim_bridge.so")
    shutil.copy(src, dst)
    os.environ.setdefault("ROCNRDMA_KMOD_SIM", dst)


_private_kmod_sim()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `-m gpu` on a GPU machine)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def ctx():
    import rocnrdma_b200 as rn
    c = rn.Context(device=0)
    yield c
    c.close()
