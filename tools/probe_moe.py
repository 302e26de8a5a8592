"""Mixtral expert block on the routed wgmma GEMM against the per-expert loop over the same `QuantizedLinear`s.
    python tools/probe_moe.py [--tokens 1,4,16,64,256,1024,4096] [--only 1x16|2x8] [--json FILE]

Shape: Mixtral-8x7B, hidden 4096, intermediate 14336, 8 experts, top-2; schemes 1x16 and 2x8; fp16 and bf16.
Routing: `uniform` (seeded router logits) and `skewed` (most tokens send their first slot to expert 0).
Per case:
  routed_us   `QuantizedMixtralExperts.forward` (sort, gathers, two routed GEMMs, act, combine), from a CUDA graph;
  loop_us     transformers' MixtralExperts algorithm over the same members, eager (it syncs with the host: no graph);
  kernels_us  the two routed GEMM launches alone (w1|w3 and w2) on pre-sorted rows, from a CUDA graph;
  backward_us the block's backward (two routed transposed GEMMs + autograd plumbing), eager, from CUDA events.
Rates: code GB/s = code bytes of the experts that received tokens / kernels_us; TFLOP/s = 2 * pairs * (2 I H + I H)
/ kernels_us.  The routed and the loop outputs are compared before timing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402
from aqlm_b200.moe import QuantizedMixtralExperts, route  # noqa: E402

HIDDEN, INTER, EXPERTS, TOP_K = 4096, 14336, 8, 2
SCHEMES = {"1x16": (1, 16), "2x8": (2, 8)}
REL_TOL = {torch.float16: 5e-3, torch.bfloat16: 3e-2}  # mean |routed - loop| / mean |loop|: other summation orders


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def graph_time_us(fn, iters):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    del g
    return a.elapsed_time(b) * 1e3 / iters


def host_time_us(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e6 / iters


def make_block(K, nbits, dtype, seed):
    dev = torch.device("cuda:0")
    act = torch.nn.SiLU()
    blk = QuantizedMixtralExperts(EXPERTS, HIDDEN, INTER, act, 8, 1, K, nbits, device="meta", dtype=dtype)
    gen = torch.Generator(device=dev).manual_seed(seed)
    lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
    with torch.no_grad():
        blk = blk.to_empty(device=dev)
        for m in blk.modules():
            if m.__class__.__name__ == "QuantizedLinear":
                m.codes.copy_(torch.randint(lo, hi, m.codes.shape, dtype=torch.int32, device=dev, generator=gen)
                              .to(m.codes.dtype))
                m.codebooks.copy_((torch.randn(m.codebooks.shape, device=dev, generator=gen) * 0.5 / K ** 0.5).to(dtype))
                m.scales.copy_((0.02 + 0.01 * torch.rand(m.scales.shape, device=dev, generator=gen)).to(dtype))
    return blk


def routing(T, kind, seed):
    gen = torch.Generator(device="cuda:0").manual_seed(seed)
    logits = torch.randn((T, EXPERTS), device="cuda:0", generator=gen)
    if kind == "skewed":
        logits[:, 0] += 8.0  # the first slot of almost every token goes to expert 0
    w, idx = torch.topk(torch.softmax(logits, -1), TOP_K, dim=-1)
    return idx, w / w.sum(-1, keepdim=True)


def probe(blk, scheme, dtype, tokens, rows):
    K, nbits = SCHEMES[scheme]
    code_bytes_w = (2 * INTER * HIDDEN + HIDDEN * INTER) // 8 * K * (2 if nbits > 8 else 1)  # per expert
    for T in tokens:
        for kind in ("uniform", "skewed"):
            idx, w = routing(T, kind, T)
            x = torch.randn((T, HIDDEN), dtype=dtype, device="cuda:0", generator=torch.Generator("cuda:0").manual_seed(T))
            with torch.no_grad():
                y = blk(x, idx, w)
                ref = blk._forward_loop(x, idx, w)
            err = float((y.float() - ref.float()).abs().mean() / ref.float().abs().mean())
            iters = max(5, min(50, int(2e4 / T) + 5))
            row = dict(scheme=scheme, dtype=str(dtype).replace("torch.", ""), tokens=T, routing=kind, rel_diff=err,
                       ok=err < REL_TOL[dtype])
            with torch.no_grad():
                row["routed_us"] = round(graph_time_us(lambda: blk(x, idx, w), iters), 1)
                row["loop_us"] = round(host_time_us(lambda: blk._forward_loop(x, idx, w), iters), 1)
                order, off, _ = route(idx, EXPERTS)
                xs = x.index_select(0, order // TOP_K)
                hs = torch.randn((T * TOP_K, INTER), dtype=dtype, device="cuda:0")
                c13, b13, s13, seg13 = blk._w13
                c2, b2, s2, _ = blk._w2

                def kernels():
                    cuda_kernel.matmat_dequant_routed(xs, c13, b13, s13, off, seg13)
                    cuda_kernel.matmat_dequant_routed(hs, c2, b2, s2, off)

                row["kernels_us"] = round(graph_time_us(kernels, iters), 1)
            xg = x.clone().requires_grad_(True)
            gy = torch.randn_like(x)
            times = []
            for i in range(max(3, iters // 2) + 1):
                yy = blk(xg, idx, w)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                yy.backward(gy)
                b.record()
                torch.cuda.synchronize()
                if i:
                    times.append(a.elapsed_time(b) * 1e3)
                xg.grad = None
            row["backward_us"] = round(sorted(times)[len(times) // 2], 1)
            hit = int(torch.unique(idx).numel())
            pairs = T * TOP_K
            row["experts_hit"] = hit
            row["code_GBps"] = round(hit * code_bytes_w / row["kernels_us"] / 1e3, 1)
            row["TFLOPs"] = round(2.0 * pairs * 3 * INTER * HIDDEN / row["kernels_us"] / 1e6, 1)
            rows.append(row)
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="1,4,16,64,256,1024,4096")
    ap.add_argument("--only", default="", help="1x16 or 2x8")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels: it needs a GPU"
    tokens = [int(v) for v in args.tokens.split(",")]
    c = card()
    print(f"# card (name, power limit, max SM clock): {c}", flush=True)
    rows = []
    for scheme, (K, nbits) in SCHEMES.items():
        if args.only and args.only != scheme:
            continue
        for dtype in (torch.float16, torch.bfloat16):
            blk = make_block(K, nbits, dtype, seed=K * 100 + nbits)
            probe(blk, scheme, dtype, tokens, rows)
            del blk
            torch.cuda.empty_cache()
    print(f"\n{c}\n")
    print("| scheme | dtype | tokens | routing | routed block, graph (us) | per-expert loop, eager (us) | routed / loop |"
          " routed kernels (us) | code GB/s | TFLOP/s | backward (us) |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['scheme']} | {r['dtype']} | {r['tokens']} | {r['routing']} | {r['routed_us']} | {r['loop_us']} | "
              f"{r['routed_us'] / r['loop_us']:.2f} | {r['kernels_us']} | {r['code_GBps']} | {r['TFLOPs']} | "
              f"{r['backward_us']} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=c, rows=rows), f, indent=1)
    bad = [r for r in rows if not r["ok"]]
    if bad:
        raise SystemExit(f"{len(bad)} cases: routed and loop outputs differ by more than the tolerance")


if __name__ == "__main__":
    main()
