"""Regenerate profiles/sass/*.sass and summary.json from the built library (CPU only: cuobjdump)."""
import collections, json, os, re, subprocess
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(root, "rocnrdma_b200", "lib", "librocnrdma_b200.so")
out = os.path.join(root, "profiles", "sass")
os.makedirs(out, exist_ok=True)
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
want = ["engine_kernel", "gemm_mxfp8_pair_kernel", "gemm_mxfp8_ordered_kernel", "gemm_mxfp8_kernel", "gemm_send2_kernel", "gemm_send_kernel", "gemm_reduce_send_kernel", "pack_fp8_write_kernel", "pack_fp8_scatter_kernel", "unpack_fp8_kernelILb0", "unpack_fp8_kernelILb1", "reduce_fp8_kernel", "relay_records_kernel",
        "rdma_stream_kernel", "shared_post_stress_kernel", "recv_consume_kernel", "recv_consume_qps_kernel"]
summary = {}
for m in re.finditer(r"\t\tFunction : (\S+)\n(.*?)(?=\n\t\tFunction : |\Z)", txt, re.S):
    mangled, body = m.group(1), m.group(2)
    name = next((w for w in want if re.search(r"\d+" + w + r"(?![a-z_])", mangled) or mangled == w), None)
    if not name:
        continue
    # the first instance of a kernel keeps its plain key; every instance of a template is also keyed by its arguments,
    # e.g. reduce_fp8_kernel<4,1,false,false>, so that each one is listed
    base = re.match(r"[a-z0-9_]+", name).group(0)
    targs = re.search(r"\d+" + base + r"I((?:L[ib]\d+E)+)E", mangled)
    keys = [] if name in summary else [name]
    if targs:
        args = [v if t == "i" else ("true" if v == "1" else "false") for t, v in re.findall(r"L([ib])(\d+)E", targs.group(1))]
        keys.append(base + "<" + ",".join(args) + ">")
    if not keys:
        continue
    for key in keys:
        open(os.path.join(out, re.sub(r"[<>,]", "_", key).rstrip("_") + ".sass"), "w").write("Function : " + mangled + "\n" + body + "\n")
    ops = collections.Counter()
    full = collections.Counter()
    for line in body.splitlines():
        mm = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)", line)
        if mm:
            ops[mm.group(1)] += 1
            full[mm.group(1) + mm.group(2)] += 1
    hopper = {k: v for k, v in full.items() if k.split(".")[0] in ("HGMMA", "QGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "UTMACMDFLUSH", "F2FP")}
    for key in keys:
        summary[key] = {"mangled": mangled, "instructions": sum(ops.values()), "hopper": dict(sorted(hopper.items())), "mnemonics": dict(ops.most_common())}
json.dump(summary, open(os.path.join(out, "summary.json"), "w"), indent=1)
for k, v in summary.items():
    print(k, v["instructions"], v["hopper"])

# the register / spill / shared-memory report of the same build, next to the listings (the build writes it into the
# git-ignored lib directory)
import shutil
_src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rocnrdma_b200", "lib", "ptxas_info.txt")
if os.path.exists(_src):
    shutil.copy(_src, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles", "ptxas_info.txt"))
