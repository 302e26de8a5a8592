"""Diagnose wgmma GEMM mismatches: per-M-tile / per-column error map, repeated runs, env overrides."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402

DEV = "cuda:0"


def run(fin, fout, batch, reps=3, label=""):
    g = torch.Generator(device=DEV).manual_seed(fin + fout + batch)
    codes = torch.randint(-32768, 32768, (fout, fin // 8, 1), dtype=torch.int16, device=DEV, generator=g)
    codebooks = torch.randn((1, 65536, 1, 8), dtype=torch.float16, device=DEV, generator=g)
    scales = (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=DEV, generator=g)).half()
    x = torch.randn((batch, fin), dtype=torch.float16, device=DEV, generator=g)
    W = cuda_kernel.dequant(codes, codebooks, scales).float()
    ref = x.float() @ W.t()
    for r in range(reps):
        y = cuda_kernel.matmat_dequant(x, codes, codebooks, scales, None).float()
        torch.cuda.synchronize()
        err = (y - ref).abs()
        rel = (err.mean() / ref.abs().mean()).item()
        tile_err = err.reshape(batch, -1, 128).mean(dim=(0, 2)) / ref.abs().mean()
        bad_tiles = (tile_err > 2e-3).nonzero().flatten().tolist()
        col_err = err.mean(dim=1) / ref.abs().mean()
        bad_cols = (col_err > 2e-3).nonzero().flatten().tolist()
        print(f"{label} {fin}x{fout} bs={batch} rep{r}: rel={rel:.3e} bad_tiles={bad_tiles[:20]} (n={len(bad_tiles)}) "
              f"bad_batch_rows={bad_cols[:8]}..(n={len(bad_cols)})", flush=True)
        if bad_tiles:
            t = bad_tiles[0]
            e = err[:, t * 128:(t + 1) * 128]
            rows_bad = (e.mean(dim=0) / ref.abs().mean() > 2e-3).nonzero().flatten().tolist()
            print(f"   tile {t}: bad rows in tile {rows_bad[:16]} (n={len(rows_bad)}); nan={torch.isnan(y).sum().item()}", flush=True)


if __name__ == "__main__":
    for env in ({}, {"AQLM_B200_GEMM_KSPLIT": "1"}, {"AQLM_B200_GEMM_KSPLIT": "2"}, {"AQLM_B200_GEMM_KSPLIT": "5"}):
        for k in ("AQLM_B200_GEMM_STAGES", "AQLM_B200_GEMM_KSPLIT"):
            os.environ.pop(k, None)
        os.environ.update(env)
        from aqlm_b200 import _cabi
        _cabi.reload_tunables()
        run(4096, 14336, 16, reps=3, label=str(env))
        run(4096, 4096, 16, reps=2, label=str(env))
