#!/bin/bash
# Everything that can be checked without a GPU, in the order a CI job would run it (≈ 3 minutes):
#   1. build the sm_90a library, the mock rdma-core provider and the kernel-module simulation (nvcc / g++ / gcc, no GPU needed)
#   2. python tests that need no GPU (wire format + cross-check against DOCA's header, protocol models, mock-NIC verbs wire,
#      kernel-module simulation, probe / config, ABI signatures)
#   3. both kernel modules against the vendored kernel-API declarations (`make -C kmod check`), the simulation under UBSan / ASan,
#      the multi-threaded stress under ASan and TSan
#   4. SASS listings: the Hopper instructions (wgmma, TMA, multicast) every kernel is expected to contain
# GPU tier (on an H100): python -m pytest tests -m gpu ; bash tools/run_sanitizers.sh ; python bench.py --gpus 1
set -euo pipefail
cd "$(dirname "$0")/.."
python -c "import __graft_entry__ as g; g.build(); print('build ok')"
python -m pytest tests -q -m "not gpu" -p no:cacheprovider
make -C kmod check
make -C kmod check-sanitize check-stress check-tsan
python tools/dump_sass.py > /dev/null
python - <<'PY'
import json
s = json.load(open("profiles/sass/summary.json"))
need = {"gemm_send2_kernel": ["HGMMA", "UTMALDG.2D.MULTICAST", "UTMASTG.2D", "UTMASTG.3D"],
        "gemm_send_kernel": ["HGMMA", "UTMALDG.2D", "UTMASTG.2D"], "gemm_mxfp8_pair_kernel": ["QGMMA", "UTMALDG.3D.MULTICAST"],
        "gemm_mxfp8_kernel": ["QGMMA", "UTMALDG.3D"], "engine_kernel": ["UBLKCP.S.G"]}
for k, ops in need.items():
    have = s[k]["hopper"]
    missing = [o for o in ops if not any(h.startswith(o) for h in have)]
    assert not missing, (k, missing)
print("sass ok:", ", ".join(need))
PY
echo "CI (CPU tier) passed"
