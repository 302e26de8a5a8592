"""Prefill on the in_features-sharded path: the partial product and the exchange at prompt-sized batches.
    python tools/probe_sharded_prefill.py [--worlds 2,4,8] [--batches 16,64,256,1024] [--scheme 1x16] [--json]

1. On one GPU, for every Llama-3-70B shard shape (in_features / W) and batch: the UNSCALED fp32 partials as GEMV passes
   of at most 8 rows (`aqlm_b200_matmat_ex` + AQLM_B200_FLAG_PARTIAL_F32, the form before prefill had its own path)
   against one wgmma GEMM (`aqlm_b200_matmat_dequant_ex` + the same flag).  Both run from a CUDA graph over rotating
   copies of the codes, so codes come from HBM; times from CUDA events.  The two outputs must agree up to fp32
   summation order.
2. With two or more GPUs (one process each): the peer-memory exchange + epilogue (`PeerComm.allreduce_scale_bias`,
   chunked when batch * out_features exceeds the communicator's default max_elems) against NCCL `all_reduce` +
   `scale_bias`, at the same batches and output widths.  With fewer GPUs those figures are reported as not measured.
"""
import argparse
import ctypes
import json
import os
import socket
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
from aqlm_b200 import _cabi  # noqa: E402
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402

# Llama-3-70B linears (in_features, out_features); a shard holds in_features / W
LINEARS = {"q/o": (8192, 8192), "k/v": (8192, 1024), "gate/up": (8192, 28672), "down": (28672, 8192)}
REL_TOL = 1e-4  # |GEMM - GEMV| / max|GEMV|: fp32 sums in another order (1x16: the same fp16 weights on both sides)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
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
    return a.elapsed_time(b) * 1e3 / iters / len(fns)


def partial_call(entry, w, x, y, ws):
    L = _cabi.lib()
    st = torch.cuda.current_stream().cuda_stream
    if entry == "gemv":
        rc = L.aqlm_b200_matmat_ex(ctypes.byref(w), x.data_ptr(), y.data_ptr(), x.shape[0], _cabi.FLAG_PARTIAL_F32, st)
    else:
        rc = L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), x.data_ptr(), y.data_ptr(), x.shape[0], _cabi.FLAG_PARTIAL_F32,
                                           ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0, st)
    _cabi.check(rc)


def probe_partials(worlds, batches, K, nbits, out_rows):
    from helpers import gpu_case

    dev = torch.device("cuda:0")
    for W in worlds:
        for name, (fin_full, fout) in LINEARS.items():
            fin = fin_full // W
            t = gpu_case(fin, fout, K, nbits, 1, seed=fin + fout)
            cbytes = fout * (fin // 8) * K * (2 if nbits > 8 else 1)
            copies = max(2, min(24, 400 * 2**20 // cbytes))
            lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
            codes = [t["codes"]] + [torch.randint(lo, hi, t["codes"].shape, dtype=t["codes"].dtype, device=dev)
                                    for _ in range(copies - 1)]
            weights = [cuda_kernel.make_weight(c, t["codebooks"], None, None) for c in codes]
            for bs in batches:
                x = torch.randn((bs, fin), dtype=t["codebooks"].dtype, device=dev)
                need = _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(weights[0]), bs)
                ws = cuda_kernel._workspace(dev, need) if need else None
                ys = {e: torch.empty((bs, fout), dtype=torch.float32, device=dev) for e in ("gemv", "gemm")}
                for e, y in ys.items():
                    partial_call(e, weights[0], x, y, ws)
                torch.cuda.synchronize()
                diff = float((ys["gemm"] - ys["gemv"]).abs().max() / ys["gemv"].abs().max())
                row = dict(W=W, linear=name, shape=f"{fin}x{fout}", batch=bs, rel_diff=diff)
                iters = max(3, min(50, int(2e5 / (bs * cbytes / 1e6 + 1))))
                for e in ("gemv", "gemm"):
                    row[f"{e}_us"] = round(graph_time_us(
                        [(lambda w=w, e=e, y=ys[e]: partial_call(e, w, x, y, ws)) for w in weights], iters), 2)
                row["speedup"] = round(row["gemv_us"] / row["gemm_us"], 2)
                row["gemm_tflops"] = round(2.0 * bs * fin * fout / row["gemm_us"] / 1e6, 1)
                row["ok"] = diff < REL_TOL
                out_rows.append(row)
                print(json.dumps(row), flush=True)
            del codes, weights
            torch.cuda.empty_cache()


def _exchange_worker(rank, world, port, batches, q):
    import torch.distributed as dist

    from aqlm_b200.peer import PeerComm

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        comm = PeerComm()
        dev = torch.device("cuda", rank)
        for fout in sorted({o for _, o in LINEARS.values()}):
            scales = torch.rand(fout, dtype=torch.float16, device=dev) + 0.5
            for bs in batches:
                part = torch.randn((bs, fout), dtype=torch.float32, device=dev)
                work = part.clone()

                def nccl():
                    work.copy_(part)
                    dist.all_reduce(work)
                    return cuda_kernel.scale_bias(work, scales, None, torch.float16)

                def peer():
                    return comm.allreduce_scale_bias(part, scales, None, torch.float16)

                a = peer()
                b = nccl()
                torch.cuda.synchronize()
                diff = float((a.float() - b.float()).abs().max() / b.float().abs().max())
                times = {}
                for nm, fn in (("peer", peer), ("nccl", nccl)):
                    for _ in range(3):
                        fn()
                    torch.cuda.synchronize()
                    dist.barrier()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(20):
                        fn()
                    e1.record()
                    torch.cuda.synchronize()
                    times[nm] = round(e0.elapsed_time(e1) * 1e3 / 20, 2)
                chunks = -(-bs // (comm.max_elems // fout))
                if rank == 0:
                    q.put(dict(world=world, out=fout, batch=bs, chunks=chunks, peer_us=times["peer"],
                               nccl_us=times["nccl"], rel_diff=diff))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def probe_exchange(batches, out_rows):
    import torch.multiprocessing as mp

    world = min(torch.cuda.device_count(), 8)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    q = mp.get_context("spawn").Manager().Queue()
    mp.spawn(_exchange_worker, args=(world, port, batches, q), nprocs=world, join=True)
    while not q.empty():
        row = q.get()
        out_rows.append(row)
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--batches", default="16,64,256,1024")
    ap.add_argument("--scheme", default="1x16")
    ap.add_argument("--json", default="", help="also write every row to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels: it needs a GPU"
    K, nbits = (int(v) for v in args.scheme.split("x"))
    worlds = [int(v) for v in args.worlds.split(",")]
    batches = [int(v) for v in args.batches.split(",")]
    print(f"# card: {card()}; scheme {args.scheme}, fp16", flush=True)
    rows = []
    probe_partials(worlds, batches, K, nbits, rows)
    if torch.cuda.device_count() >= 2:
        probe_exchange(batches, rows)
    else:
        print("# exchange (peer vs NCCL): not measured -- needs two or more GPUs", flush=True)
    print("\n| W | linear | shard (in x out) | batch | GEMV passes (us) | wgmma GEMM (us) | speedup | GEMM TFLOP/s |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        if "linear" in r:
            print(f"| {r['W']} | {r['linear']} | {r['shape']} | {r['batch']} | {r['gemv_us']} | {r['gemm_us']} | "
                  f"{r['speedup']}x | {r['gemm_tflops']} |")
    bad = [r for r in rows if "linear" in r and not r["ok"]]
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)
    if bad:
        raise SystemExit(f"{len(bad)} shapes: GEMM and GEMV partials differ by more than {REL_TOL} (relative)")


if __name__ == "__main__":
    main()
