"""Time the UNMODIFIED reference CUDA kernels (pip-installed into the git-ignored oracle/_ref) on this GPU with the
same protocol as tools/probe_gemv.py (CUDA-graph replay over rotating weight copies, CUDA events).

Run in its OWN process (the reference and aqlm_b200 both register `aqlm::` torch.library ops):
    TORCH_CUDA_ARCH_LIST=9.0 python tools/compare_reference_gpu.py [--out FILE]
The reference JIT-builds its extension on first import (cuda_kernel.py:8-11); ~1 minute.
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "_ref"))
os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")

import torch  # noqa: E402

L2_BYTES = 50 * 2**20  # H100 SXM


def time_graph(fn_list, iters=20):
    for f in fn_list:
        f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for f in fn_list:
            f()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters / len(fn_list)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--cases", default="all", choices=["all", "quick"], help="quick: the subset bench.py reports in `secondary`")
    args = ap.parse_args()
    import aqlm  # the reference
    assert "oracle/_ref" in aqlm.__file__, aqlm.__file__
    from aqlm.inference_kernels.cuda_kernel import CUDA_KERNEL  # JIT build

    dev = "cuda:0"
    rows = []
    cases = [("1x16", 1, 16, (4096, 4096), 1), ("1x16", 1, 16, (4096, 14336), 1), ("1x16", 1, 16, (14336, 4096), 1),
             ("2x8", 2, 8, (4096, 4096), 1), ("2x8", 2, 8, (4096, 11008), 1),
             ("1x16", 1, 16, (4096, 14336), 256), ("1x16", 1, 16, (4096, 14336), 64), ("1x16", 1, 16, (4096, 4096), 256)]
    if args.cases == "quick":
        cases = [("1x16", 1, 16, (4096, 4096), 1), ("1x16", 1, 16, (4096, 14336), 1), ("2x8", 2, 8, (4096, 11008), 1),
                 ("1x16", 1, 16, (4096, 14336), 256), ("1x16", 1, 16, (4096, 4096), 256)]
    for scheme, K, nbits, (fin, fout), bs in cases:
        cbytes = fout * (fin // 8) * K * ((nbits + 7) // 8)
        copies = max(2, min(64, (2 * L2_BYTES + cbytes - 1) // cbytes + 1))
        ws = []
        for _ in range(copies):
            lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
            codes = torch.randint(lo, hi, (fout, fin // 8, K), dtype=torch.int8 if nbits <= 8 else torch.int16, device=dev)
            cb = torch.randn((K, 2**nbits, 1, 8), dtype=torch.float16, device=dev)
            sc = (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=dev)).half()
            ws.append((codes, cb, sc))
        x = torch.randn((bs, fin), dtype=torch.float16, device=dev)
        if bs <= 6:
            op = CUDA_KERNEL.code1x16_matmat if scheme == "1x16" else CUDA_KERNEL.code2x8_matmat
            name = f"code{scheme}_matmat"
        else:
            op = CUDA_KERNEL.code1x16_matmat_dequant if scheme == "1x16" else CUDA_KERNEL.code2x8_matmat_dequant
            name = f"code{scheme}_matmat_dequant"
        try:
            us = time_graph([(lambda w=w: op(x, w[0], w[1], w[2], None)) for w in ws])
            mode = "cuda_graph"
        except Exception as e:  # the reference's host wrapper is not capturable on every path: fall back to eager timing
            torch.cuda.synchronize()
            for w in ws[:3]:
                op(x, w[0], w[1], w[2], None)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for w in ws:
                op(x, w[0], w[1], w[2], None)
            b.record()
            torch.cuda.synchronize()
            us = a.elapsed_time(b) * 1e3 / len(ws)
            mode = f"eager ({type(e).__name__})"
        row = dict(impl="reference (oracle/_ref, unmodified, JIT sm_90)", op=name, scheme=scheme, in_features=fin,
                   out_features=fout, batch=bs, us=round(us, 2), code_GBps=round(cbytes / us / 1e3, 1),
                   tflops=round(2.0 * bs * fin * fout / us / 1e6, 1), timing=mode)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del ws
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
