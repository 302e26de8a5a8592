"""Cluster LUT GEMV, first vs second form (AQLM_B200_LUT_CLUSTER=1|2|3, AQLM_B200_LUT_C2_RB=0|16|32): time per launch
(CUDA-graph replay over rotating weight copies, CUDA events) and a parity check of every variant against the fp32
dequantized matvec computed by torch on the same tensors."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from aqlm_b200 import _cabi  # noqa: E402
from aqlm_b200.inference_kernels import cuda_kernel  # noqa: E402

sys.path.insert(0, os.path.join(REPO, "tools"))
from probe_gemm import timed  # noqa: E402


def dense_ref(x, codes, codebooks, scales):
    K = codes.shape[2]
    idx = codes.to(torch.int64) % 256
    W = sum(codebooks[k, :, 0, :].float()[idx[:, :, k]] for k in range(K))  # [out, in/8, 8]
    W = W.reshape(codes.shape[0], -1) * scales.float().reshape(-1, 1)
    return x.float() @ W.t()


def main():
    dev = "cuda:0"
    shapes = ((2, (4096, 11008)), (2, (4096, 4096)), (1, (4096, 11008)), (2, (4096, 22016)), (2, (4096, 12288)), (2, (1024, 4096)), (1, (4096, 4096)))
    variants = (("shipped default (second form, 16-row warp batches)", {}),
                ("first form", {"AQLM_B200_LUT_CLUSTER": "1"}),
                ("second form", {"AQLM_B200_LUT_CLUSTER": "2"}),
                ("second form, RB16", {"AQLM_B200_LUT_CLUSTER": "2", "AQLM_B200_LUT_C2_RB": "16"}),
                ("second form, RB32", {"AQLM_B200_LUT_CLUSTER": "2", "AQLM_B200_LUT_C2_RB": "32"}))
    for K, (fin, fout) in shapes:
        cb = fout * (fin // 8) * K
        copies = max(2, min(40, 300 * 2**20 // cb))
        ws = [(torch.randint(-128, 128, (fout, fin // 8, K), dtype=torch.int8, device=dev),
               torch.randn((K, 256, 1, 8), dtype=torch.float16, device=dev),
               (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=dev)).half()) for _ in range(copies)]
        x = torch.randn((1, fin), dtype=torch.float16, device=dev)
        ref = dense_ref(x, *ws[0])
        for label, env in variants:
            os.environ.update(env)
            _cabi.reload_tunables()
            y = cuda_kernel.matmat(x, ws[0][0], ws[0][1], ws[0][2], None).float()
            rel = float((y - ref).abs().mean() / ref.abs().mean())
            us = timed([(lambda w=w: cuda_kernel.matmat(x, w[0], w[1], w[2], None)) for w in ws])
            print(json.dumps(dict(scheme=f"{K}x8", shape=f"{fin}x{fout}", variant=label, us=round(us, 2),
                                  code_GBps=round(cb / us / 1e3, 1), rel_err=rel)), flush=True)
            for k in env:
                os.environ.pop(k)
        _cabi.reload_tunables()
        del ws
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
