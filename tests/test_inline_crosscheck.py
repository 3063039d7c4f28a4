"""The inline WQE layout against an independent source: DOCA GPUNetIO's definitions in the NCCL wheel
(tests/native/inline_crosscheck.cc; every layout assertion is a static_assert, and the program checks the ds the encoder
writes for 12- and 28-byte payloads)."""
import shutil
import subprocess
from pathlib import Path

import pytest

from test_wire_crosscheck import _doca_header

ROOT = Path(__file__).resolve().parent.parent
SRC = ROOT / "tests" / "native" / "inline_crosscheck.cc"


def _compile(tmp_path, include_dir, hdr):
    exe = tmp_path / "inline_crosscheck"
    cmd = ["g++", "-std=c++17", "-fpermissive", "-w", f"-I{include_dir}", f'-DDOCA_VERBS_DEF_H="{hdr}"', str(SRC), "-o", str(exe)]
    return exe, subprocess.run(cmd, capture_output=True, text=True, timeout=120)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host compiler")
def test_inline_limit_segment_and_segment_counts_agree_with_doca_gpunetio(tmp_path):
    hdr = _doca_header()
    if hdr is None:
        pytest.skip("the NCCL wheel in this image does not ship doca_gpunetio_verbs_def.h")
    exe, r = _compile(tmp_path, ROOT / "rocnrdma_b200" / "csrc", hdr)
    assert r.returncode == 0, r.stderr[-3000:]
    assert subprocess.run([str(exe)], timeout=60).returncode == 0


def test_the_inline_crosscheck_can_fail(tmp_path):
    """Negative control: raise our inline limit by one byte and the same translation unit must stop compiling."""
    hdr = _doca_header()
    if hdr is None or shutil.which("g++") is None:
        pytest.skip("no independent header / compiler")
    src = (ROOT / "rocnrdma_b200" / "csrc" / "wire" / "mlx5_wire.h").read_text()
    old = "  MAX_INLINE = 28,"
    assert old in src
    (tmp_path / "wire").mkdir()
    (tmp_path / "wire" / "mlx5_wire.h").write_text(src.replace(old, "  MAX_INLINE = 29,", 1))
    _, r = _compile(tmp_path, tmp_path, hdr)
    assert r.returncode != 0 and "largest inline payload" in r.stderr
