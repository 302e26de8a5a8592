"""Trainable codebooks and scales in Mixtral expert blocks and grouped linears: one routed / grouped weight-gradient
launch per projection against the member-by-member path.
    python tools/probe_routed_weight_grad.py [--tokens 64,256,1024,4096] [--only moe|group] [--json FILE]

Mixtral-8x7B block (hidden 4096, intermediate 14336, 8 experts, top-2), 1x16 and 2x8, fp16, `uniform` and `skewed`
routing (most tokens send their first slot to expert 0), codebooks and scales trainable, input not:
  routed_us   forward + backward of `QuantizedMixtralExperts` (two routed GEMMs, w2's routed transposed GEMM, two routed
              weight-gradient launches and the plumbing), from a CUDA graph;
  loop_us     the same forward + backward through transformers' loop over the members (each member's forward, transposed
              and weight-gradient launches; it syncs with the host: eager, wall clock);
  wgrad_us    the two routed weight-gradient launches alone (w1|w3 and w2) on pre-sorted rows, from a CUDA graph.
Llama-3-8B q/k/v (4096 -> 4096 | 1024 | 1024) and gate/up (4096 -> 14336 | 14336), 1x16, fp16:
  grouped_us  one grouped weight-gradient launch;  members_us  one weight-gradient launch per member; both from a graph.
The routed and loop gradients (and the grouped and member ones) are compared before timing.  Prints the card's name,
power limit and max SM clock, read in the same run.
"""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from probe_moe import EXPERTS, HIDDEN, INTER, SCHEMES, TOP_K, card, graph_time_us, make_block, routing  # noqa: E402

from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402
from aqlm_b200.moe import route  # noqa: E402

DEV = "cuda:0"
REL_TOL = 2e-2  # ||routed - loop|| / ||loop|| of the weight gradients: other summation orders, fp16 intermediates


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def members(blk):
    return [getattr(blk.expert(e), n) for e in range(EXPERTS) for n in ("w1", "w2", "w3")]


def grads(blk):
    return torch.cat([torch.cat([m.codebooks.grad.reshape(-1), m.scales.grad.reshape(-1)]).float() for m in members(blk)
                      if m.codebooks.grad is not None])


def median_event_us(fn, iters):
    times = []
    for i in range(iters + 1):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if i:
            times.append((time.perf_counter() - t0) * 1e6)
    return sorted(times)[len(times) // 2]


def probe_moe(tokens, rows):
    for scheme, (K, nbits) in SCHEMES.items():
        blk = make_block(K, nbits, torch.float16, seed=K * 100 + nbits)
        for m in members(blk):
            m.codebooks.requires_grad_(True)
            m.scales.requires_grad_(True)
        for T in tokens:
            for kind in ("uniform", "skewed"):
                idx, w = routing(T, kind, T)
                gen = torch.Generator(DEV).manual_seed(T)
                x = torch.randn((T, HIDDEN), dtype=torch.float16, device=DEV, generator=gen)
                gy = torch.randn((T, HIDDEN), dtype=torch.float16, device=DEV, generator=gen) * 1e-2
                iters = max(5, min(30, int(2e4 / T) + 5))

                def routed():
                    blk(x, idx, w).backward(gy)

                def loop():
                    blk._forward_loop(x, idx, w).backward(gy)
                blk.zero_grad(set_to_none=True)
                routed()
                g_routed = grads(blk)
                blk.zero_grad(set_to_none=True)
                loop()
                g_loop = grads(blk)  # experts without tokens have no gradient in the loop: compare where both do
                err = rel(g_routed, g_loop) if g_routed.numel() == g_loop.numel() else float("nan")
                row = dict(scheme=scheme, tokens=T, routing=kind, rel_diff=err, ok=err < REL_TOL or err != err)
                blk.zero_grad(set_to_none=True)
                row["routed_us"] = round(graph_time_us(routed, iters), 1)
                blk.zero_grad(set_to_none=True)
                row["loop_us"] = round(median_event_us(loop, max(3, iters // 3)), 1)
                order, off, _ = route(idx, EXPERTS)
                xs = x.index_select(0, order // TOP_K)
                hs = torch.randn((T * TOP_K, INTER), dtype=torch.float16, device=DEV, generator=gen)
                g13 = torch.randn((T * TOP_K, 2 * INTER), dtype=torch.float16, device=DEV, generator=gen)
                g2 = torch.randn((T * TOP_K, HIDDEN), dtype=torch.float16, device=DEV, generator=gen)
                c13, b13, s13, seg13 = blk._w13
                c2, b2, s2, _ = blk._w2

                def wgrads():
                    cuda_kernel.matmat_weight_grad_routed(xs, g13, c13, b13, s13, off, seg13)
                    cuda_kernel.matmat_weight_grad_routed(hs, g2, c2, b2, s2, off)
                row["wgrad_us"] = round(graph_time_us(wgrads, iters), 1)
                row["wgrad_TFLOPs"] = round(2.0 * T * TOP_K * 3 * INTER * HIDDEN / row["wgrad_us"] / 1e6, 1)
                rows.append(row)
                print(json.dumps(row), flush=True)
        del blk
        torch.cuda.empty_cache()


def random_linear_stack(outs, fin, seed):
    gen = torch.Generator(DEV).manual_seed(seed)
    out = sum(outs)
    codes = torch.randint(-32768, 32768, (out, fin // 8, 1), dtype=torch.int16, device=DEV, generator=gen)
    cbs = (torch.randn((len(outs), 1, 65536, 1, 8), device=DEV, generator=gen) * 0.5).half()
    scales = (0.02 + 0.01 * torch.rand((out, 1, 1, 1), device=DEV, generator=gen)).half()
    return codes, cbs, scales


def probe_group(tokens, rows):
    for name, outs in (("q/k/v", [4096, 1024, 1024]), ("gate/up", [14336, 14336])):
        codes, cbs, scales = random_linear_stack(outs, 4096, len(outs))
        for T in tokens:
            gen = torch.Generator(DEV).manual_seed(T)
            x = torch.randn((T, 4096), dtype=torch.float16, device=DEV, generator=gen)
            gy = torch.randn((T, sum(outs)), dtype=torch.float16, device=DEV, generator=gen)
            gys = [g.contiguous() for g in gy.split(outs, -1)]
            offs = [sum(outs[:i]) for i in range(len(outs))]
            iters = max(5, min(50, int(2e4 / T) + 5))

            def grouped():
                return cuda_kernel.matmat_weight_grad_grouped(x, gy, codes, cbs, scales, outs)

            def member_calls():
                return [cuda_kernel.matmat_weight_grad(x, g, codes[o:o + n], cbs[i], scales[o:o + n])
                        for i, (o, n, g) in enumerate(zip(offs, outs, gys))]
            gcb, gs = grouped()
            ms = member_calls()
            err = max(rel(gcb.float(), torch.stack([m[0] for m in ms]).float()),
                      rel(gs.float(), torch.cat([m[1] for m in ms]).float()))
            row = dict(group=name, tokens=T, rel_diff=err, ok=err < 1e-2)
            row["grouped_us"] = round(graph_time_us(grouped, iters), 1)
            row["members_us"] = round(graph_time_us(member_calls, iters), 1)
            rows.append(row)
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="64,256,1024,4096")
    ap.add_argument("--only", default="", help="moe or group")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels: it needs a GPU"
    tokens = [int(v) for v in args.tokens.split(",")]
    c = card()
    print(f"# card (name, power limit, max SM clock): {c}", flush=True)
    moe_rows, group_rows = [], []
    if args.only in ("", "moe"):
        probe_moe(tokens, moe_rows)
    if args.only in ("", "group"):
        probe_group(tokens, group_rows)
    print(f"\n{c}\n")
    if moe_rows:
        print("| scheme | tokens | routing | routed fwd+bwd, graph (us) | member loop fwd+bwd, eager (us) | loop / routed |"
              " routed weight-gradient launches (us) | their TFLOP/s |")
        print("|---|---|---|---|---|---|---|---|")
        for r in moe_rows:
            print(f"| {r['scheme']} | {r['tokens']} | {r['routing']} | {r['routed_us']} | {r['loop_us']} | "
                  f"{r['loop_us'] / r['routed_us']:.2f} | {r['wgrad_us']} | {r['wgrad_TFLOPs']} |")
    if group_rows:
        print("\n| group | tokens | grouped launch (us) | member launches (us) | members / grouped |")
        print("|---|---|---|---|---|")
        for r in group_rows:
            print(f"| {r['group']} | {r['tokens']} | {r['grouped_us']} | {r['members_us']} | "
                  f"{r['members_us'] / r['grouped_us']:.2f} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=c, moe=moe_rows, group=group_rows), f, indent=1)
    bad = [r for r in moe_rows + group_rows if not r["ok"]]
    if bad:
        raise SystemExit(f"{len(bad)} cases: the one-launch and member gradients differ by more than the tolerance")


if __name__ == "__main__":
    main()
