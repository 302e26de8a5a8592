"""Per-shape timing probe of the fused GEMV (and large-batch op): CUDA-graph replay over rotating weight copies
(so codes come from HBM, not L2), CUDA events, reported as us and code-bytes GB/s vs the measured HBM peak.

    python tools/probe_gemv.py [--schemes 1x16,2x8,8x8] [--batches 1,2,4,8] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aqlm_b200 import _cabi  # noqa: E402
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402

L2_BYTES = 50 * 2**20  # H100 SXM


def peak_gbs():
    try:
        with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
            return json.load(f)["hbm_gbs"], "measured"
    except Exception:
        return 6650.0, "fallback"


def make_weights(fin, fout, K, nbits, g, copies, dev):
    ws = []
    for _ in range(copies):
        lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
        codes = torch.randint(lo, hi, (fout, fin // g, K), dtype=torch.int8 if nbits <= 8 else torch.int16, device=dev)
        cb = torch.randn((K, 2**nbits, 1, g), dtype=torch.float16, device=dev)
        sc = (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=dev)).half()
        ws.append((codes, cb, sc))
    return ws


def time_graph(fn_list, iters=20):
    """fn_list: callables launched back to back inside ONE graph; returns us per callable."""
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
    ap.add_argument("--schemes", default="1x16,2x8,8x8")
    ap.add_argument("--batches", default="1")
    ap.add_argument("--ctas", default="8")
    ap.add_argument("--op", default="matmat")
    ap.add_argument("--shapes", default="4096x4096,4096x1024,4096x14336,14336x4096,4096x11008,8192x8192,8192x28672")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = "cuda:0"
    peak, peak_kind = peak_gbs()
    rows = []
    op = getattr(cuda_kernel, args.op)
    for scheme in args.schemes.split(","):
        K, nbits = (int(v) for v in scheme.split("x"))
        for shape in args.shapes.split(","):
            fin, fout = (int(v) for v in shape.split("x"))
            cbytes = fout * (fin // 8) * K * ((nbits + 7) // 8)
            copies = max(2, min(64, (2 * L2_BYTES + cbytes - 1) // cbytes + 1))
            ws = make_weights(fin, fout, K, nbits, 8, copies, dev)
            for batch in (int(b) for b in args.batches.split(",")):
                x = torch.randn((batch, fin), dtype=torch.float16, device=dev)
                for ctas in args.ctas.split(","):
                    os.environ["AQLM_B200_GEMV_CTAS_PER_SM"] = ctas
                    _cabi.reload_tunables()
                    fns = [(lambda w=w: op(x, w[0], w[1], w[2], None)) for w in ws]
                    us = time_graph(fns)
                    gbs = cbytes / us / 1e3
                    tflops = 2.0 * batch * fin * fout / us / 1e6
                    row = dict(scheme=scheme, in_features=fin, out_features=fout, batch=batch, tflops=round(tflops, 1),
                               ctas_per_sm=int(ctas), op=args.op, us=round(us, 3), code_GBps=round(gbs, 1),
                               frac_of_hbm_peak=round(gbs / peak, 4), peak=peak_kind, rotating_copies=copies)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
            del ws
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
