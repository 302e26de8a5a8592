"""Grouped wgmma GEMM against its members: linears that share their input (q/k/v, gate/up) as ONE launch over the
row-concatenated weight, or one launch per member (the form before grouping reached prefill and the backward).
    python tools/probe_grouped_gemm.py [--batches 16,64,256,1024,4096] [--only NAME[,NAME]] [--json FILE]

Shapes (in -> out of each member):
  llama3-8b 1x16   q/k/v 4096 -> 4096|1024|1024, gate/up 4096 -> 14336|14336        fp16 and bf16
  llama2-7b 2x8    q/k/v 4096 -> 3 x 4096,       gate/up 4096 -> 2 x 11008          fp16
  70b shard W=8    q/k/v 1024 -> 8192|1024|1024, fp32 partials (AQLM_B200_FLAG_PARTIAL_F32), forward only
For each shape and batch: the forward (`aqlm_b200_matmat_dequant_grouped` against one `aqlm_b200_matmat_dequant_ex`
per member) and the transposed GEMM (`aqlm_b200_matmat_dequant_transposed_grouped` against one
`aqlm_b200_matmat_dequant_transposed` per member plus the adds autograd makes to sum the members' input gradients).
Protocol of probe_gemm.py: every variant runs from a CUDA graph over rotating copies of the codes (so codes come from
HBM), times from CUDA events; the grouped and the members' outputs are compared before timing.
Last, the grouped transposed kernel against the plain one on the same weight for the 8-codebook schemes (see OVERHEAD).
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

# name -> (in_features, member out_features, K, nbits, dtypes, partial)
SHAPES = {
    "llama3-8b 1x16 q/k/v": (4096, [4096, 1024, 1024], 1, 16, (torch.float16, torch.bfloat16), False),
    "llama3-8b 1x16 gate/up": (4096, [14336, 14336], 1, 16, (torch.float16, torch.bfloat16), False),
    "llama2-7b 2x8 q/k/v": (4096, [4096, 4096, 4096], 2, 8, (torch.float16,), False),
    "llama2-7b 2x8 gate/up": (4096, [11008, 11008], 2, 8, (torch.float16,), False),
    "70b W=8 shard q/k/v partials": (1024, [8192, 1024, 1024], 1, 16, (torch.float16,), True),
}
REL_TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}  # |grouped - members| / max|members|: another summation order


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


class Group:
    """One copy of a group: fused codes, the members' views of them, and C descriptors of both."""

    def __init__(self, codes, codebooks, scales, segs, partial):
        self.segs, self.partial = segs, partial
        sc = None if partial else scales
        self.w = cuda_kernel.make_weight(codes, codebooks[0], sc, None)
        self.w_t = cuda_kernel.make_weight(codes, codebooks[0], scales, None)
        self.seg = (ctypes.c_int64 * len(segs))(*segs)
        self.members, off = [], 0
        for i, n in enumerate(segs):
            self.members.append(cuda_kernel.make_weight(codes[off:off + n], codebooks[i], scales[off:off + n], None))
            off += n


def _ws(dev, need):
    return cuda_kernel._workspace(dev, need) if need else None


def _ptr(ws):
    return (ws.data_ptr(), ws.numel()) if ws is not None else (None, 0)


def run_forward(grp, x, y, ys, grouped):
    L = _cabi.lib()
    st = torch.cuda.current_stream().cuda_stream
    flags = _cabi.FLAG_PARTIAL_F32 if grp.partial else 0
    bs = x.shape[0]
    if grouped:
        ws, n = _ptr(_ws(x.device, L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(grp.w), bs)))
        _cabi.check(L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(grp.w), grp.seg, len(grp.segs), x.data_ptr(),
                                                       y.data_ptr(), bs, flags, ws, n, st))
        return
    for w, ym in zip(grp.members, ys):
        ws, n = _ptr(_ws(x.device, L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), bs)))
        _cabi.check(L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), x.data_ptr(), ym.data_ptr(), bs, flags, ws, n, st))


def run_transposed(grp, go, gx, gos, gxs, grouped):
    L = _cabi.lib()
    st = torch.cuda.current_stream().cuda_stream
    bs = go.shape[0]
    if grouped:
        ws, n = _ptr(_ws(go.device, L.aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(grp.w_t), bs)))
        _cabi.check(L.aqlm_b200_matmat_dequant_transposed_grouped(ctypes.byref(grp.w_t), grp.seg, len(grp.segs),
                                                                  go.data_ptr(), gx.data_ptr(), bs, ws, n, st))
        return
    for w, gom, gxm in zip(grp.members, gos, gxs):
        ws, n = _ptr(_ws(go.device, L.aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(w), bs)))
        _cabi.check(L.aqlm_b200_matmat_dequant_transposed(ctypes.byref(w), gom.data_ptr(), gxm.data_ptr(), bs, ws, n, st))
    torch.add(gxs[0], gxs[1], out=gx)  # autograd sums the members' input gradients
    for g in gxs[2:]:
        gx.add_(g)


def rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30))


def probe(name, fin, segs, K, nbits, dtype, partial, batches, rows):
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(fin + sum(segs) + K)
    fout = sum(segs)
    lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
    cdt = torch.int8 if nbits <= 8 else torch.int16
    codebooks = (torch.randn((len(segs), K, 2 ** nbits, 1, 8), device=dev, generator=gen) * 0.5 / K ** 0.5).to(dtype)
    scales = (0.75 + 0.5 * torch.rand(fout, device=dev, generator=gen)).to(dtype)
    cbytes = fout * (fin // 8) * K * (2 if nbits > 8 else 1)
    copies = max(2, min(24, 400 * 2 ** 20 // cbytes))
    codes = [torch.randint(lo, hi, (fout, fin // 8, K), dtype=cdt, device=dev, generator=gen) for _ in range(copies)]
    groups = [Group(c, codebooks, scales, segs, partial) for c in codes]
    odt = torch.float32 if partial else dtype
    for bs in batches:
        x = torch.randn((bs, fin), dtype=dtype, device=dev, generator=gen)
        y = torch.empty((bs, fout), dtype=odt, device=dev)
        ys = [torch.empty((bs, n), dtype=odt, device=dev) for n in segs]
        iters = max(3, min(50, int(2e5 / (bs * cbytes / 1e6 + 1))))
        run_forward(groups[0], x, y, ys, True)
        run_forward(groups[0], x, y, ys, False)
        torch.cuda.synchronize()
        row = dict(shape=name, dtype=str(dtype).replace("torch.", ""), dir="forward", batch=bs,
                   rel_diff=rel(y, torch.cat(ys, dim=1)))
        for grouped, key in ((False, "members_us"), (True, "grouped_us")):
            row[key] = round(graph_time_us([(lambda g=g, gr=grouped: run_forward(g, x, y, ys, gr)) for g in groups],
                                           iters), 2)
        row["speedup"] = round(row["members_us"] / row["grouped_us"], 3)
        row["ok"] = row["rel_diff"] < REL_TOL[dtype]
        rows.append(row)
        print(json.dumps(row), flush=True)
        del y, ys
        if not partial:
            go = torch.randn((bs, fout), dtype=dtype, device=dev, generator=gen)
            gos, off = [], 0
            for n in segs:
                gos.append(go[:, off:off + n].contiguous())
                off += n
            gx = torch.empty((bs, fin), dtype=dtype, device=dev)
            gxs = [torch.empty((bs, fin), dtype=dtype, device=dev) for _ in segs]
            ref = torch.empty_like(gx)
            run_transposed(groups[0], go, ref, gos, gxs, False)
            run_transposed(groups[0], go, gx, gos, gxs, True)
            torch.cuda.synchronize()
            row = dict(shape=name, dtype=str(dtype).replace("torch.", ""), dir="transposed", batch=bs,
                       rel_diff=rel(gx, ref))
            for grouped, key in ((False, "members_us"), (True, "grouped_us")):
                row[key] = round(graph_time_us(
                    [(lambda g=g, gr=grouped: run_transposed(g, go, gx, gos, gxs, gr)) for g in groups], iters), 2)
            row["speedup"] = round(row["members_us"] / row["grouped_us"], 3)
            row["ok"] = row["rel_diff"] < REL_TOL[dtype]
            rows.append(row)
            print(json.dumps(row), flush=True)
            del go, gos, gx, gxs, ref
        del x
        torch.cuda.empty_cache()
    del codes, groups
    torch.cuda.empty_cache()


# The grouped transposed kernels of the 8-codebook schemes run at the register limit and some instantiations spill a few
# bytes (N = 16 / 32 / 64).  This measures the grouped kernel against the plain one on the SAME concatenated weight,
# with a second segment of one k-block so that the extra codebook set adds almost no L2 traffic: what is left is the cost of
# the segment lookup and of the spills.
OVERHEAD = [(8, 8), (8, 16)]
OVERHEAD_SHAPE = (4096, 12288)


def probe_kernel_overhead(batches, rows):
    dev = torch.device("cuda:0")
    fin, fout = OVERHEAD_SHAPE
    segs = [fout - 64, 64]
    L = _cabi.lib()
    for K, nbits in OVERHEAD:
        for dtype in (torch.float16, torch.bfloat16):
            gen = torch.Generator(device=dev).manual_seed(K * 100 + nbits)
            lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
            cdt = torch.int8 if nbits <= 8 else torch.int16
            cbs = (torch.randn((2, K, 2 ** nbits, 1, 8), device=dev, generator=gen) * 0.5 / K ** 0.5).to(dtype)
            scales = (0.75 + 0.5 * torch.rand(fout, device=dev, generator=gen)).to(dtype)
            cbytes = fout * (fin // 8) * K * (2 if nbits > 8 else 1)
            copies = max(2, min(24, 400 * 2 ** 20 // cbytes))
            codes = [torch.randint(lo, hi, (fout, fin // 8, K), dtype=cdt, device=dev, generator=gen)
                     for _ in range(copies)]
            ws_ = [cuda_kernel.make_weight(c, cbs[0], scales, None) for c in codes]
            seg = (ctypes.c_int64 * 2)(*segs)
            for bs in batches:
                go = torch.randn((bs, fout), dtype=dtype, device=dev, generator=gen)
                gx = torch.empty((bs, fin), dtype=dtype, device=dev)

                def call(w, grouped):
                    st = torch.cuda.current_stream().cuda_stream  # the capture stream inside a graph capture
                    ws, n = _ptr(_ws(dev, L.aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(w), bs)))
                    if grouped:
                        _cabi.check(L.aqlm_b200_matmat_dequant_transposed_grouped(
                            ctypes.byref(w), seg, 2, go.data_ptr(), gx.data_ptr(), bs, ws, n, st))
                    else:
                        _cabi.check(L.aqlm_b200_matmat_dequant_transposed(ctypes.byref(w), go.data_ptr(), gx.data_ptr(),
                                                                          bs, ws, n, st))
                iters = max(3, min(50, int(2e5 / (bs * cbytes / 1e6 + 1))))
                row = dict(scheme=f"{K}x{nbits}", dtype=str(dtype).replace("torch.", ""), batch=bs)
                for grouped, key in ((False, "plain_us"), (True, "grouped_us")):
                    row[key] = round(graph_time_us([(lambda w=w, gr=grouped: call(w, gr)) for w in ws_], iters), 2)
                row["grouped_over_plain"] = round(row["grouped_us"] / row["plain_us"], 4)
                rows.append(row)
                print(json.dumps(row), flush=True)
            del codes, ws_
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="16,64,256,1024,4096")
    ap.add_argument("--only", default="", help="comma-separated substrings of shape names")
    ap.add_argument("--json", default="", help="also write every row to this file")
    ap.add_argument("--overhead-batches", default="16,32,64,128",
                    help="batches of the grouped-against-plain transposed kernel comparison (empty: skip it)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels: it needs a GPU"
    batches = [int(v) for v in args.batches.split(",")]
    c = card()
    print(f"# card (name, power limit, max SM clock): {c}", flush=True)
    rows = []
    for name, (fin, segs, K, nbits, dtypes, partial) in SHAPES.items():
        if args.only and not any(s in name for s in args.only.split(",")):
            continue
        for dtype in dtypes:
            probe(name, fin, segs, K, nbits, dtype, partial, batches, rows)
    over = []
    if args.overhead_batches:
        probe_kernel_overhead([int(v) for v in args.overhead_batches.split(",")], over)
    print(f"\n{c}\n")
    print("| shape | dtype | direction | batch | members (us) | grouped (us) | members / grouped |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['dtype']} | {r['dir']} | {r['batch']} | {r['members_us']} | {r['grouped_us']} | "
              f"{r['speedup']}x |")
    if over:
        print(f"\ntransposed {OVERHEAD_SHAPE[0]} -> {OVERHEAD_SHAPE[1]}: grouped kernel (2 segments) against the plain "
              "kernel on the same weight\n")
        print("| scheme | dtype | batch | plain (us) | grouped (us) | grouped / plain |")
        print("|---|---|---|---|---|---|")
        for r in over:
            print(f"| {r['scheme']} | {r['dtype']} | {r['batch']} | {r['plain_us']} | {r['grouped_us']} | "
                  f"{r['grouped_over_plain']} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=c, rows=rows, kernel_overhead=over), f, indent=1)
    bad = [r for r in rows if not r["ok"]]
    if bad:
        raise SystemExit(f"{len(bad)} cases: grouped and members' outputs differ by more than the tolerance")


if __name__ == "__main__":
    main()
