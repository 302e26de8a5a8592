"""Register / spill report of every kernel in the library (`nvcc -Xptxas -v`, CPU only; output to a scratch .so):
    python tools/ptxas_report.py > ptxas_report.md
Lists registers, stack frame and spill bytes per kernel family; kernels with spills are listed one by one."""
import collections
import os
import re
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from aqlm_b200 import _cabi  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = ["nvcc", *_cabi.NVCC_FLAGS, "-Xptxas", "-v", "-o", os.path.join(tmp, "lib.so"),
               *[os.path.join(_cabi.CSRC, s) for s in _cabi.SOURCES]]
        log = subprocess.run(cmd, cwd=_cabi.CSRC, capture_output=True, text=True, check=True).stderr
    ents = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'\nptxas info\s+: Function properties for \S+\n\s+(\d+) bytes stack frame, "
                      r"(\d+) bytes spill stores, (\d+) bytes spill loads\nptxas info\s+: Used (\d+) registers", log)
    names = subprocess.run(["c++filt"] + [e[0] for e in ents], capture_output=True, text=True).stdout.splitlines()
    rows = [(n.replace("void aqlm_b200::", "").split("(")[0], int(e[1]), int(e[2]), int(e[3]), int(e[4])) for n, e in zip(names, ents)]
    fam = collections.defaultdict(list)
    for r in rows:
        fam[r[0].split("<")[0]].append(r)
    print("# ptxas resource report of `libaqlm_b200.so` (sm_90a, `-O3`)\n")
    print(f"{len(rows)} kernel instantiations; {sum(1 for r in rows if r[2] or r[3])} of them spill.\n")
    print("| kernel family | instantiations | registers (min-max) | with spills | worst spill (store / load bytes) |")
    print("|---|---|---|---|---|")
    for k, v in sorted(fam.items()):
        sp = [r for r in v if r[2] or r[3]]
        worst = max(v, key=lambda r: r[2] + r[3])
        print(f"| `{k}` | {len(v)} | {min(r[4] for r in v)}-{max(r[4] for r in v)} | {len(sp)} | {worst[2]} / {worst[3]} |")
    print("\n## Kernels with spills\n")
    print("| kernel | registers | stack frame | spill stores | spill loads |")
    print("|---|---|---|---|---|")
    for r in sorted(rows, key=lambda r: -(r[2] + r[3])):
        if r[2] or r[3]:
            print(f"| `{r[0]}` | {r[4]} | {r[1]} | {r[2]} | {r[3]} |")


if __name__ == "__main__":
    main()
