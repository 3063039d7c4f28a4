"""The fp8 ring all-reduce with one process per GPU, connected through ``parallel.connect_ring``."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]


def test_ring_allreduce_one_process_per_gpu():
    """Two ranks, one per GPU, run by ``tools/allreduce_bench.py`` under torchrun.  Every rank checks its output
    against ``ref_allreduce_fp8`` bit for bit and exits non-zero otherwise."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29581", os.path.join(root, "tools", "allreduce_bench.py"), "--elems",
           str(1 << 22), "--chunk", str(1 << 20), "--reps", "1"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=root)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    rows = [json.loads(l) for l in p.stdout.splitlines() if l.startswith("{")]
    assert rows and rows[-1]["world"] == 2, p.stdout[-2000:]
