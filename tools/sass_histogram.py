"""SASS opcode histogram of the shipped library (no GPU needed): proves which hardware paths the kernels use
(HGMMA = wgmma, UBLKCP = TMA bulk copy, SYNCS = mbarrier, REDUX = warp reductions, LDGSTS = cp.async).  usage: python tools/sass_histogram.py [lib.so] > sass_histogram.txt"""
import collections
import re
import subprocess
import sys

lib = sys.argv[1] if len(sys.argv) > 1 else "rl4co_b200/libcorollout.so"
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
per_kernel, total, cur = {}, collections.Counter(), None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        per_kernel[cur] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and cur:
        op = m.group(1)
        per_kernel[cur][op] += 1
        total[op] += 1
KEY = ["HGMMA", "WARPGROUP", "UBLKCP", "UTMALDG", "UTMASTG", "LDGSTS", "SYNCS", "REDUX", "MUFU", "SHFL", "LDS", "STS", "BAR", "FFMA", "HMMA", "ATOMS", "LDL", "STL"]
print(f"# {lib}: {sum(total.values())} SASS instructions in {len(per_kernel)} kernels (sm_90a)")
print("## whole library, selected opcodes")
for k in KEY:
    print(f"  {k:10s} {total.get(k, 0)}")
print("## per kernel (kernels with tensor-core / bulk-copy / async-copy / warp-reduction instructions)")
for name, c in sorted(per_kernel.items()):
    sel = {k: c[k] for k in KEY if c.get(k)}
    if any(k in sel for k in ("HGMMA", "UBLKCP", "UTMALDG", "LDGSTS", "REDUX")):
        print(f"  {name[:100]}")
        print("     " + "  ".join(f"{k}={v}" for k, v in sel.items()))
