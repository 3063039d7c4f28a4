"""The fp8 all-to-all with one process per GPU, connected through ``parallel.peer.connect_mesh``."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_alltoall_one_process_per_gpu():
    """Two ranks, one per GPU, run by ``tools/alltoall_bench.py`` under torchrun: each connects its plan with
    ``connect()`` and checks its output against ``ref_alltoall_fp8`` bit for bit, exiting non-zero otherwise."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29583", os.path.join(root, "tools", "alltoall_bench.py"), "--reps", "1"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=root)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    rows = [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]
    assert rows and rows[-1]["world"] == 2, p.stdout[-2000:]
