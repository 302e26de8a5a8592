"""A/B of two builds of the library on the fused dequant + wgmma GEMMs: same results bit for bit, same speed?
    python tools/ab_builds.py OLD/libaqlm_b200.so NEW/libaqlm_b200.so [--out DIR] [--rounds 3]
Each round runs the cases below once per library, alternating, each run in a fresh process with AQLM_B200_LIB set
(aqlm_b200/_cabi.py loads that file).  A run computes every case on seeded inputs, stores the output's bytes, and times
it with the protocol of probe_gemm.py (CUDA-graph replay over rotating weight copies, CUDA events, warm-up first).
Reports per case whether the outputs of all runs of both libraries are byte-identical (the split-K fix-up adds in a
fixed order, so they must be) and every run's time, so one library's run-to-run spread sits next to the difference
between the two.  Needs a GPU; there is no fallback."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, op, scheme, dtype, in_features, out_features, batch): the GEMM sizes README.md reports
CASES = [(f"fwd 1x16 {dt} bs{bs}", "forward", "1x16", dt, 4096, 14336, bs) for dt in ("f16", "bf16") for bs in (16, 64, 256)] + [
    ("fwd 2x8 f16 bs256", "forward", "2x8", "f16", 4096, 11008, 256),
    ("fwd 8x8 f16 bs256", "forward", "8x8", "f16", 4096, 11008, 256),
    ("transposed 1x16 f16 bs256", "transposed", "1x16", "f16", 4096, 14336, 256),
    ("partial_f32 1x16 f16 bs256", "partial", "1x16", "f16", 3584, 8192, 256),
]


def child(out_dir):
    import torch

    sys.path.insert(0, REPO)
    sys.path.insert(0, os.path.join(REPO, "tests"))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from helpers import gpu_case
    from probe_gemm import timed

    from aqlm_b200.inference_kernels import cuda_kernel

    assert torch.cuda.is_available(), "ab_builds.py needs a GPU"
    rows = {}
    for name, op, scheme, dtype, fin, fout, bs in CASES:
        K, nbits = (int(v) for v in scheme.split("x"))
        dt = torch.float16 if dtype == "f16" else torch.bfloat16
        t = gpu_case(fin, fout, K, nbits, bs, dtype=dt, seed=fin + fout + bs)
        if op == "forward":
            x, fn = t["x"], lambda c: cuda_kernel.matmat_dequant(x, c, t["codebooks"], t["scales"], None)
        elif op == "transposed":
            x = torch.randn((bs, fout), dtype=dt, device="cuda:0", generator=torch.Generator(device="cuda:0").manual_seed(bs))
            fn = lambda c: cuda_kernel.matmat_dequant_transposed(x, c, t["codebooks"], t["scales"], None)  # noqa: E731
        else:
            x, fn = t["x"], lambda c: cuda_kernel.matmat_partial(x, c, t["codebooks"])
        y = fn(t["codes"])
        torch.cuda.synchronize()
        raw = y.contiguous().view(torch.uint8).cpu().numpy().tobytes()
        with open(os.path.join(out_dir, name.replace(" ", "_") + ".bin"), "wb") as f:
            f.write(raw)
        cbytes = t["codes"].numel() * t["codes"].element_size()
        copies = max(2, min(24, 300 * 2**20 // cbytes))
        lo, hi = (-128, 128) if nbits <= 8 else (-32768, 32768)
        gen = torch.Generator(device="cuda:0").manual_seed(1)
        ws = [t["codes"]] + [torch.randint(lo, hi, t["codes"].shape, dtype=t["codes"].dtype, device="cuda:0", generator=gen)
                             for _ in range(copies - 1)]
        us = timed([(lambda c=c: fn(c)) for c in ws], iters=20)
        rows[name] = dict(sha256=hashlib.sha256(raw).hexdigest(), us=round(us, 2))
        del ws, t
        torch.cuda.empty_cache()
    with open(os.path.join(out_dir, "result.json"), "w") as f:
        json.dump(rows, f, indent=1)


def main():
    if len(sys.argv) == 3 and sys.argv[1] == "--child":
        return child(sys.argv[2])
    ap = argparse.ArgumentParser()
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--out", default=None, help="output directory (default: a new temporary directory)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="ab_builds_")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    print("GPU (name, power limit, max SM clock):", gpu, flush=True)
    runs = {"old": [], "new": []}
    for r in range(args.rounds):
        for which, lib in (("old", args.old), ("new", args.new)):
            d = os.path.join(out, f"{which}_{r}")
            os.makedirs(d, exist_ok=True)
            env = dict(os.environ, AQLM_B200_LIB=os.path.abspath(lib))
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", d], env=env, check=True)
            with open(os.path.join(d, "result.json")) as f:
                runs[which].append(json.load(f))
            print(f"round {r} {which}: done", flush=True)
    all_same, within = True, True
    print("\n| case | outputs identical | old us (each run) | new us (each run) | new median / old median |")
    print("|---|---|---|---|---|")
    for name, *_ in CASES:
        o = [run[name] for run in runs["old"]]
        n = [run[name] for run in runs["new"]]
        same = len({x["sha256"] for x in o + n}) == 1
        all_same &= same
        ou, nu = sorted(x["us"] for x in o), sorted(x["us"] for x in n)
        within &= nu[len(nu) // 2] <= ou[-1]
        print(f"| {name} | {'yes' if same else 'NO'} | {' '.join(str(x['us']) for x in o)} | {' '.join(str(x['us']) for x in n)} | "
              f"{nu[len(nu) // 2] / ou[len(ou) // 2]:.4f} |")
    summary = dict(gpu=gpu, old=args.old, new=args.new, runs=runs, outputs_identical=all_same,
                   new_median_within_old_range=within)
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(f"\noutputs byte-identical in every case: {all_same}; new median <= slowest old run in every case: {within}")
    print("written to", out)
    return 0 if all_same else 1


if __name__ == "__main__":
    sys.exit(main())
