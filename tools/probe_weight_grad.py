"""Weight gradient of a quantized linear: the fused wgmma kernel against the dense formulation it replaces.
    python tools/probe_weight_grad.py [--tokens 64,256,1024,4096,8192] [--only NAME[,NAME]] [--json FILE]

Both paths compute grad_codebooks and grad_scales of one linear from its input x [tokens, in] and output gradient
g [tokens, out]:
  fused  zero grad_codebooks, then ONE `aqlm_b200_matmat_weight_grad` launch (csrc/gemm_wgrad.cuh);
  dense  what a training layer that materialises W does (the reference project's): Wu = dequant (our kernel), the
         dense dW = g^T x through cuBLAS in the activation dtype, then grad_codebooks with index_add_ of s * dW over the
         codes (indices precomputed, not timed) and grad_scales as the row dot of dW and Wu, in fp32.
Shapes: Llama-3-8B 1x16 (4096 -> 4096, 4096 -> 14336, 14336 -> 4096) and Llama-2-7B 2x8 (4096 -> 11008), fp16 and bf16.
Protocol of probe_gemm.py: each path runs from a CUDA graph over rotating copies of the codes (so codes come from HBM),
timed with CUDA events; the two paths' outputs are compared at every timed size before timing.  TFLOP/s counts the
main loop's 2 * tokens * out * in; `epilogue share` is the fused time at 64 tokens over the fused time (the epilogue's cost
does not depend on the token count, and at 64 tokens the main loop is one k-block).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from aqlm_b200 import _cabi  # noqa: E402
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402

# name -> (in_features, out_features, K, nbits)
SHAPES = {
    "llama3-8b 1x16 q/o": (4096, 4096, 1, 16),
    "llama3-8b 1x16 gate/up": (4096, 14336, 1, 16),
    "llama3-8b 1x16 down": (14336, 4096, 1, 16),
    "llama2-7b 2x8 gate/up": (4096, 11008, 2, 8),
}
REL_TOL = {torch.float16: 5e-3, torch.bfloat16: 3e-2}  # the dense path rounds dW to the activation dtype


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def graph_time_us(fns, iters):
    """Mean time of one call, from CUDA events around `iters` replays of a graph that holds every fn once."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for f in fns:
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
    t = a.elapsed_time(b) * 1e3 / iters / len(fns)
    del g
    return t


class Linear:
    """One copy of the weight, its C descriptor and the unsigned code indices of the dense path."""

    def __init__(self, codes, codebooks, scales):
        self.codes, self.codebooks, self.scales = codes, codebooks, scales
        self.w = cuda_kernel.make_weight(codes, codebooks, scales, None)
        n = codebooks.shape[1]
        self.idx = [(codes[:, :, k].long() % n).reshape(-1) for k in range(codes.shape[2])]


def run_fused(lin, x, g, gcb, gs, ws):
    st = torch.cuda.current_stream().cuda_stream
    gcb.zero_()
    _cabi.check(_cabi.lib().aqlm_b200_matmat_weight_grad(ctypes.byref(lin.w), x.data_ptr(), g.data_ptr(), x.shape[0],
                                                         gcb.data_ptr(), gs.data_ptr(), ws.data_ptr(), ws.numel(), st))


def run_dense(lin, x, g, gcb, gs):
    Wu = cuda_kernel.dequant(lin.codes, lin.codebooks, None)
    dW = (g.t() @ x).float()
    torch.sum(dW * Wu.float(), dim=1, out=gs)
    sD = (dW * lin.scales.float()[:, None]).reshape(-1, 8)
    gcb.zero_()
    for k, idx in enumerate(lin.idx):
        gcb[k].index_add_(0, idx, sD)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def probe(name, fin, fout, K, nbits, dtype, tokens, rows):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(fin + fout + K)
    lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
    cdt = torch.int8 if nbits <= 8 else torch.int16
    codebooks = (torch.randn((K, 2 ** nbits, 1, 8), device=dev, generator=gen) * 0.5 / K ** 0.5).to(dtype)
    scales = (0.75 + 0.5 * torch.rand(fout, device=dev, generator=gen)).to(dtype)
    cbytes = fout * (fin // 8) * K * (2 if nbits > 8 else 1)
    copies = max(2, min(8, 400 * 2 ** 20 // cbytes))
    lins = [Linear(torch.randint(lo, hi, (fout, fin // 8, K), dtype=cdt, device=dev, generator=gen), codebooks, scales)
            for _ in range(copies)]
    gcb = torch.zeros((K, 2 ** nbits, 8), dtype=torch.float32, device=dev)
    gs = torch.zeros(fout, dtype=torch.float32, device=dev)
    ref_cb, ref_s = torch.zeros_like(gcb), torch.zeros_like(gs)
    t64 = None
    for bs in tokens:
        x = torch.randn((bs, fin), dtype=dtype, device=dev, generator=gen)
        g = torch.randn((bs, fout), dtype=dtype, device=dev, generator=gen)
        ws = cuda_kernel._workspace(dev, _cabi.lib().aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(lins[0].w), bs))
        run_fused(lins[0], x, g, gcb, gs, ws)
        run_dense(lins[0], x, g, ref_cb, ref_s)
        torch.cuda.synchronize()
        row = dict(shape=name, dtype=str(dtype).replace("torch.", ""), tokens=bs, rel_cb=rel(gcb, ref_cb),
                   rel_s=rel(gs, ref_s))
        iters = max(3, min(50, int(3e4 / (bs * fin * fout / 1e9 + 20))))
        row["fused_us"] = round(graph_time_us([(lambda li=li: run_fused(li, x, g, gcb, gs, ws)) for li in lins], iters), 1)
        row["dense_us"] = round(graph_time_us([(lambda li=li: run_dense(li, x, g, ref_cb, ref_s)) for li in lins], iters), 1)
        if bs == 64:
            t64 = row["fused_us"]
        row["fused_tflops"] = round(2.0 * bs * fin * fout / row["fused_us"] / 1e6, 1)
        row["dense_over_fused"] = round(row["dense_us"] / row["fused_us"], 2)
        row["epilogue_share"] = round(t64 / row["fused_us"], 2) if t64 else None
        row["ok"] = row["rel_cb"] < REL_TOL[dtype] and row["rel_s"] < REL_TOL[dtype]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, g
        torch.cuda.empty_cache()
    del lins
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="64,256,1024,4096,8192")
    ap.add_argument("--only", default="", help="comma-separated substrings of shape names")
    ap.add_argument("--dtypes", default="float16,bfloat16")
    ap.add_argument("--json", default="", help="also write every row to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels: it needs a GPU"
    tokens = [int(v) for v in args.tokens.split(",")]
    c = card()
    print(f"# card (name, power limit, max SM clock): {c}", flush=True)
    rows = []
    for name, (fin, fout, K, nbits) in SHAPES.items():
        if args.only and not any(s in name for s in args.only.split(",")):
            continue
        for dt in args.dtypes.split(","):
            probe(name, fin, fout, K, nbits, getattr(torch, dt), tokens, rows)
    print(f"\n{c}\n")
    print("| shape | dtype | tokens | fused (us) | fused TFLOP/s | dense (us) | dense / fused | epilogue share |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        share = "" if r["epilogue_share"] is None else f"{r['epilogue_share']:.2f}"
        print(f"| {r['shape']} | {r['dtype']} | {r['tokens']} | {r['fused_us']} | {r['fused_tflops']} | {r['dense_us']} | "
              f"{r['dense_over_fused']}x | {share} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=c, rows=rows), f, indent=1)
    bad = [r for r in rows if not r["ok"]]
    if bad:
        raise SystemExit(f"{len(bad)} cases: fused and dense outputs differ by more than the tolerance")


if __name__ == "__main__":
    main()
