"""LoRA adapters on quantized linears: the fused path against the base op plus PEFT's formulation, and the cost of the
adapter term in the kernels' epilogue.
    python tools/probe_lora.py [--out results.jsonl] [--tokens 1,4,16,256,1024,4096] [--ranks 8,16,64]

For each shape, token count T and rank r (fp16 base, fp32 adapter as PEFT creates it):
  * forward: `LoraQuantizedLinear.forward` (U = x A^T in torch, then ONE fused launch) against `peft_forward` (the base
    op, then lora_A, lora_B, cast, scale and add in torch), both under no_grad;
  * forward + backward (x, A and B trainable, dropout 0): the same two formulations through autograd;
  * epilogue: the LoRA-flagged kernel alone with B = 0 against the plain kernel (GEMV at T <= 6, wgmma GEMM above; and
    the transposed GEMM), which isolates what the adapter term costs inside the kernel.
Times are CUDA-graph replays (CUDA events, mean per call), so launch gaps are not counted for either side.  Outputs of
the two formulations are compared (max relative difference).  The card, its power limit and its max SM clock are
printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import aqlm_b200  # noqa: E402
from aqlm_b200.inference_kernels import cuda_kernel as ck  # noqa: E402

DEV = "cuda:0"
# (name, in, out, K, nbits, fused GEMV at T <= 6)
SHAPES = [("llama3-8b q_proj/o_proj 1x16", 4096, 4096, 1, 16, True),
          ("llama2-7b gate_proj 2x8 (wgmma only)", 4096, 11008, 2, 8, False)]


def timed(fn, iters=20):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
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
    return a.elapsed_time(b) * 1e3 / iters


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def make(fin, fout, K, nbits, r, gemv):
    torch.manual_seed(fin + fout + r)
    base = aqlm_b200.QuantizedLinear(fin, fout, 8, 1, K, nbits, bias=False, device=DEV, dtype=torch.float16)
    with torch.no_grad():
        base.codes.copy_(torch.randint(-2 ** (nbits - 1), 2 ** (nbits - 1), base.codes.shape, device=DEV))
        base.codebooks.copy_(torch.randn(base.codebooks.shape, device=DEV) * 0.05)
        base.scales.copy_(torch.rand(base.scales.shape, device=DEV) + 0.5)
    m = aqlm_b200.LoraQuantizedLinear(base, r, 2 * r)
    with torch.no_grad():
        m.lora_B.weight.normal_(0, 0.02)
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the rows, unrounded, as JSON lines to this file")
    ap.add_argument("--tokens", default="1,4,16,256,1024,4096")
    ap.add_argument("--ranks", default="8,16,64")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "probe_lora needs a GPU"
    info = card()
    print("card, power limit, max SM clock:", info, flush=True)
    rows = []
    for name, fin, fout, K, nbits, gemv in SHAPES:
        for r in (int(v) for v in args.ranks.split(",")):
            m = make(fin, fout, K, nbits, r, gemv)
            base = m.base_layer
            for T in (int(v) for v in args.tokens.split(",")):
                if T <= 6 and not gemv:
                    continue  # no fused 2x8 GEMV: at these T the module runs PEFT's formulation itself
                x = torch.randn(T, fin, device=DEV, dtype=torch.float16)
                go = torch.randn(T, fout, device=DEV, dtype=torch.float16)
                with torch.no_grad():
                    y_f, y_p = m(x), m.peft_forward(x)
                    diff = ((y_f.float() - y_p.float()).abs().max() / y_p.float().abs().max()).item()
                    t_fwd_fused = timed(lambda: m(x))
                    t_fwd_peft = timed(lambda: m.peft_forward(x))
                xg = x.clone().requires_grad_(True)

                def step(fwd):
                    def run():
                        fwd(xg).backward(go)
                    return run

                t_bwd_fused = timed(step(m))
                t_bwd_peft = timed(step(m.peft_forward))
                # the epilogue alone: the LoRA-flagged kernel with B = 0 against the plain kernel
                zero_b = torch.zeros_like(m.lora_B.weight)
                zero_a = torch.zeros_like(m.lora_A.weight)
                u = torch.zeros(T, r, device=DEV)
                small = T <= 6 and gemv
                plain = (lambda: ck.matmat(x, base.codes, base.codebooks, base.scales)) if small else \
                    (lambda: ck.matmat_dequant(x, base.codes, base.codebooks, base.scales))
                fused_op = ck.matmat_lora if small else ck.matmat_dequant_lora
                flagged = lambda: fused_op(x, base.codes, base.codebooks, base.scales, None, u, zero_b, 1.0)  # noqa: E731
                t_plain, t_flag = timed(plain), timed(flagged)
                t_tplain = timed(lambda: ck.matmat_dequant_transposed(go, base.codes, base.codebooks, base.scales))
                t_tflag = timed(lambda: ck.matmat_dequant_transposed_lora(go, base.codes, base.codebooks, base.scales,
                                                                          u, zero_a, 1.0))
                row = dict(shape=name, T=T, r=r, fwd_fused_us=t_fwd_fused, fwd_peft_us=t_fwd_peft,
                           fwd_bwd_fused_us=t_bwd_fused, fwd_bwd_peft_us=t_bwd_peft, kernel_plain_us=t_plain,
                           kernel_lora_b0_us=t_flag, transposed_plain_us=t_tplain, transposed_lora_b0_us=t_tflag,
                           max_rel_diff_vs_peft=diff, card=info)
                rows.append(row)
                print(json.dumps({k: (float(f"{v:.4g}") if isinstance(v, float) else v) for k, v in row.items() if k != "card"}),
                      flush=True)
                del x, go, xg
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
