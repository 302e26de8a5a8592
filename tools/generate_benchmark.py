"""End-to-end decode benchmark through Hugging Face (SURVEY §8 f1), the counterpart of the reference's
benchmark/generate_benchmark.py:67-106: a Llama-architecture model whose ONE decoder layer is replicated to full depth
(shared parameters, exactly the reference's `load_shared_model`), random AQLM weights, tokens/s of

  * `hf_generate`              -- `model.generate(prompt, min_new_tokens=max_new_tokens=N)`, timed as the reference does
                                  (perf_counter around the benchmark iterations, after warm-up);
  * `static_cache_cuda_graph`  -- one decode step (StaticCache, greedy token fed back on the device) captured in a CUDA
                                  graph and replayed N times, CUDA-event timed (the notebook recipe the reference ships
                                  as notebooks/aqlm_cuda_graph.ipynb, without torch.compile).

`--impl ours` uses aqlm_b200 aliased as `aqlm` (optionally with q/k/v and gate/up grouped launches, `--fuse`);
`--impl reference` imports the UNMODIFIED reference from oracle/_ref (its CUDA kernels are JIT-built for sm_90);
`--impl dense` is the fp16 nn.Linear model.  Run each impl in its own process (both packages register `aqlm::` ops).
One JSON line per mode on stdout.
"""
import argparse
import json
import os
import sys
import time
import warnings

warnings.filterwarnings("ignore")
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MODELS = {
    "llama3-8b": dict(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                      num_key_value_heads=8, vocab_size=128256),
    "llama2-7b": dict(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                      num_key_value_heads=32, vocab_size=32000),
    "tiny": dict(hidden_size=256, intermediate_size=512, num_hidden_layers=4, num_attention_heads=4,
                 num_key_value_heads=2, vocab_size=512),
}


def build_shared_model(args, device):
    import torch
    from transformers import AqlmConfig, LlamaConfig, LlamaForCausalLM

    K, nbits = (int(v) for v in args.scheme.split("x"))
    kw = dict(MODELS[args.model])
    num_layers = kw.pop("num_hidden_layers")
    cfg = LlamaConfig(num_hidden_layers=1, max_position_embeddings=4096, tie_word_embeddings=False, **kw)
    torch.manual_seed(0)
    model = LlamaForCausalLM(cfg).half()
    if args.impl != "dense":
        from transformers.integrations.aqlm import replace_with_aqlm_linear

        qcfg = AqlmConfig(in_group_size=8, out_group_size=1, num_codebooks=K, nbits_per_codebook=nbits)
        model = replace_with_aqlm_linear(model, modules_to_not_convert=["lm_head"], quantization_config=qcfg)
        gen = torch.Generator().manual_seed(1)
        for name, mod in model.named_modules():
            if type(mod).__name__ != "QuantizedLinear":
                continue
            lo, hi = (-128, 128) if nbits <= 8 else (-(2 ** (nbits - 1)), 2 ** (nbits - 1))
            mod.to_empty(device="cpu")
            mod.codes.data = torch.randint(lo, hi, mod.codes.shape, dtype=mod.codes.dtype, generator=gen)
            mod.codebooks.data = (torch.randn(mod.codebooks.shape, generator=gen) * (0.02 / K**0.5)).half()
            mod.scales.data = (0.75 + 0.5 * torch.rand(mod.scales.shape, generator=gen)).half()
    model = model.to(device)
    layer = model.model.layers[0]
    for i in range(1, num_layers):  # reference generate_benchmark.py:70-77: new layer objects, shared parameter storage
        new_layer = type(layer)(model.config, i)
        if args.impl != "dense":
            from transformers.integrations.aqlm import replace_with_aqlm_linear

            new_layer = replace_with_aqlm_linear(new_layer, quantization_config=qcfg)
        new_layer = new_layer.to_empty(device=device) if any(p.is_meta for p in new_layer.parameters()) else new_layer.to(device)
        for new_p, p in zip(new_layer.parameters(), layer.parameters()):
            new_p.data = p.data
        new_layer.self_attn.layer_idx = i
        model.model.layers.append(new_layer)
    model.config.num_hidden_layers = num_layers
    model.eval()
    fused = 0
    if args.impl == "ours" and args.fuse:
        import aqlm_b200

        fused = aqlm_b200.fuse_shared_input_linears(model)
    return model, fused


def bench_hf_generate(model, prompt, args):
    import torch

    for i in range(args.warmup_iters + args.benchmark_iters):
        model.generate(prompt, min_new_tokens=args.output_length, max_new_tokens=args.output_length, do_sample=False)
        if i == args.warmup_iters - 1:
            torch.cuda.synchronize()
            t_s = time.perf_counter()
    torch.cuda.synchronize()
    return args.benchmark_iters * args.output_length / (time.perf_counter() - t_s)


def bench_static_graph(model, prompt, args):
    import torch
    from transformers import StaticCache

    n = args.output_length
    cache = StaticCache(config=model.config, max_cache_len=prompt.shape[1] + n * (args.benchmark_iters + 1) + 16)
    tok = torch.zeros((1, 1), dtype=torch.long, device=prompt.device)
    with torch.no_grad():
        out = model(input_ids=prompt, past_key_values=cache, use_cache=True)  # prefill (eager)
        tok.copy_(out.logits[:, -1].argmax(-1, keepdim=True))

        def step():
            logits = model(input_ids=tok, past_key_values=cache, use_cache=True).logits
            tok.copy_(logits[:, -1].argmax(-1, keepdim=True))

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        for _ in range(n):  # warm-up replays
            graph.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n * args.benchmark_iters):
            graph.replay()
        b.record()
        torch.cuda.synchronize()
    return n * args.benchmark_iters / (a.elapsed_time(b) * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "dense"])
    ap.add_argument("--model", default="llama3-8b", choices=list(MODELS))
    ap.add_argument("--scheme", default="1x16")
    ap.add_argument("--warmup_iters", type=int, default=1)
    ap.add_argument("--benchmark_iters", type=int, default=3)
    ap.add_argument("--input_length", type=int, default=1)
    ap.add_argument("--output_length", type=int, default=128)
    ap.add_argument("--fuse", action="store_true", help="ours: grouped q/k/v and gate/up launches")
    ap.add_argument("--modes", default="hf_generate,static_cache_cuda_graph")
    args = ap.parse_args()

    if args.impl == "reference":
        sys.path.insert(0, os.path.join(REPO, "oracle", "_ref"))
        os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
        import aqlm

        assert "oracle/_ref" in aqlm.__file__, aqlm.__file__
    elif args.impl == "ours":
        sys.path.insert(0, REPO)
        import aqlm_b200

        aqlm_b200.install_as_aqlm()
    import torch

    assert torch.cuda.is_available()
    device = torch.device("cuda:0")
    model, fused = build_shared_model(args, device)
    prompt = torch.randint(0, model.config.vocab_size, (1, args.input_length), device=device)
    base = dict(impl=args.impl, model=args.model, scheme=args.scheme if args.impl != "dense" else "fp16", fused_groups=fused,
                input_length=args.input_length, output_length=args.output_length, iters=args.benchmark_iters,
                layers=model.config.num_hidden_layers, shared_layer=True)
    for mode in args.modes.split(","):
        row = dict(base, mode=mode)
        try:
            with torch.no_grad():
                fn = bench_hf_generate if mode == "hf_generate" else bench_static_graph
                row["tok_s"] = round(fn(model, prompt, args), 2)
        except Exception as e:  # keep the other mode's number
            row["error"] = f"{type(e).__name__}: {str(e)[:300]}"
            torch.cuda.synchronize()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
