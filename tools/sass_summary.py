"""Opcode histogram per kernel of the shipped library (cuobjdump -sass), written as a small markdown table: the evidence
that the wgmma / TMA paths are what the .so contains (HGMMA = wgmma.mma_async, UTMALDG = TMA tensor load, SYNCS = mbarrier,
HMMA = mma.sync).  Runs on CPU (no GPU needed).
    python tools/sass_summary.py [other/libaqlm_b200.so] > sass_summary.md"""
import collections
import os
import re
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "aqlm_b200", "csrc", "libaqlm_b200.so")
KEY = ["HGMMA", "UTMALDG", "UTMAPF", "SYNCS", "HMMA", "LDG", "LDS", "STS", "LDGSTS", "SHFL", "FFMA",
       "FADD", "PRMT", "ATOMG", "MEMBAR", "ACQBULK", "UCGABAR_ARV", "BAR"]


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else LIB
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    demangle = {}
    kernels = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    names = list(kernels)
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
        demangle = dict(zip(names, out))
    except Exception:
        demangle = {n: n for n in names}
    agg = collections.OrderedDict()
    for n, c in kernels.items():
        d = demangle.get(n, n)
        short = re.sub(r"^void aqlm_b200::", "", d)
        short = re.sub(r"\(.*$", "", short)
        agg[short] = c
    print(f"# SASS opcode summary of {os.path.relpath(lib, REPO)} (sm_90a)\n")
    print("`python tools/sass_summary.py` (cuobjdump -sass; counts are static instruction counts per kernel instantiation).\n")
    total = collections.Counter()
    for c in agg.values():
        total.update(c)
    print("Library totals: " + ", ".join(f"{k} {total[k]}" for k in KEY if total[k]) + "\n")
    cols = [k for k in KEY if total[k]]
    print("| kernel | instrs | " + " | ".join(cols) + " |")
    print("|---|---|" + "---|" * len(cols))
    for n, c in agg.items():
        if sum(c.values()) == 0:
            continue
        print(f"| `{n}` | {sum(c.values())} | " + " | ".join(str(c[k]) if c[k] else "" for k in cols) + " |")


if __name__ == "__main__":
    sys.exit(main())
