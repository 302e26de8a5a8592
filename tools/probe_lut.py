"""Batch-1 Kx8 LUT GEMV against its alternatives: the shipped plan, one LUT CTA per SM, the gather kernel (no LUT), and at
batch 2 / 4 the gather kernel against one LUT launch per row -- CUDA-graph replay over rotating weight copies, CUDA events."""
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


def main():
    dev = "cuda:0"
    for K, (fin, fout) in ((2, (4096, 11008)), (2, (4096, 4096)), (8, (4096, 11008)), (1, (4096, 11008)), (2, (11008, 4096))):
        cb = fout * (fin // 8) * K
        copies = max(2, min(40, 300 * 2**20 // cb))
        ws = [(torch.randint(-128, 128, (fout, fin // 8, K), dtype=torch.int8, device=dev),
               torch.randn((K, 256, 1, 8), dtype=torch.float16, device=dev),
               (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=dev)).half()) for _ in range(copies)]
        x = torch.randn((1, fin), dtype=torch.float16, device=dev)
        # the shipped plan, the ctas-per-SM knob and the plain gather kernel
        for env, label in (({}, "shipped"), ({"AQLM_B200_LUT_CTAS_PER_SM": "1"}, "1 CTA/SM"),
                           ({"AQLM_B200_DISABLE_LUT": "1"}, "gather kernel (no LUT)")):
            os.environ.update(env)
            _cabi.reload_tunables()
            us = timed([(lambda w=w: cuda_kernel.matmat(x, w[0], w[1], w[2], None)) for w in ws])
            print(json.dumps(dict(scheme=f"{K}x8", shape=f"{fin}x{fout}", variant=label, us=round(us, 2),
                                  code_GBps=round(cb / us / 1e3, 1))), flush=True)
            for k in env:
                os.environ.pop(k)
            _cabi.reload_tunables()
        # batch 2 / 4: gather kernel (current path) vs looping the LUT kernel per row
        for bs in (2, 4):
            xb = torch.randn((bs, fin), dtype=torch.float16, device=dev)
            us = timed([(lambda w=w: cuda_kernel.matmat(xb, w[0], w[1], w[2], None)) for w in ws])
            us_loop = timed([(lambda w=w: [cuda_kernel.matmat(xb[i:i + 1], w[0], w[1], w[2], None) for i in range(bs)]) for w in ws])
            print(json.dumps(dict(scheme=f"{K}x8", shape=f"{fin}x{fout}", batch=bs, us_gather_kernel=round(us, 2),
                                  us_lut_per_row_loop=round(us_loop, 2))), flush=True)
        del ws
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
