"""LoRA adapters fused into the 1x16 GEMV and the wgmma GEMMs (forward and input gradient), on an H100.

Kernel tests are bit-exact on an integer lattice (as in test_zz_gemm_exact.py): small-integer activations, codebooks,
adapter operands U / V and A / B, power-of-two scales and scaling, integer biases.  Every product is exact and every
partial sum is a multiple of 2^-e well inside fp32's significand, so the kernels' result is the exact float64 result
rounded once to the output type, whatever the summation order, split or tile.  The module tests compare against a
dense float64 autograd model within a stated tolerance, PEFT's own formulation bit for bit where no fused kernel
applies, and a Llama model with adapters on q/k/o end to end.
"""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

import aqlm_b200
from aqlm_b200 import _cabi
from aqlm_b200.inference_kernels import cuda_kernel as ck

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
DT_ID = {torch.float16: "f16", torch.bfloat16: "bf16"}


@contextlib.contextmanager
def switches(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    _cabi.reload_tunables()
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        _cabi.reload_tunables()


def lattice(seed, fin, fout, K, nbits, batch, rank, dtype, adt, bias=True):
    """Lattice operands on the device, and the float64 dense weight W (unscaled) and scales on the CPU."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda lo, hi, shape: torch.randint(lo, hi + 1, shape, generator=g)  # noqa: E731
    codes = ri(0, 2 ** nbits - 1, (fout, fin // 8, K))
    cb = ri(-2, 2, (K, 2 ** nbits, 1, 8)).double()
    W = cb[torch.arange(K), codes].sum(dim=2).reshape(fout, fin)  # [out, in], codes[o, gi, k] -> cb[k, code]
    e = ri(0, 3, (fout,))
    scales = (2.0 ** -e.double()).reshape(fout, 1, 1, 1)
    b = ri(-8, 8, (fout,)).double() if bias else None
    x = ri(-2, 2, (batch, fin)).double()
    u = ri(-3, 3, (batch, rank)).double()   # U forward, V transposed
    up = ri(-2, 2, (fout, rank)).double()   # B [out, rank]
    down = ri(-2, 2, (rank, fin)).double()  # A [rank, in]
    go = ri(-2, 2, (batch, fout)).double()
    signed = torch.int16 if nbits == 16 else torch.int8
    codes_dev = (codes - (codes >= 2 ** (nbits - 1)).long() * 2 ** nbits).to(signed).to(DEV).contiguous()
    d = lambda t, dt=dtype: None if t is None else t.to(dt).to(DEV).contiguous()  # noqa: E731
    dev = dict(codes=codes_dev, codebooks=d(cb), scales=d(scales), bias=d(b), x=d(x), u=d(u, adt), up=d(up, adt),
               down=d(down, adt), go=d(go))
    host = dict(W=W, scales=scales.reshape(-1), bias=b, x=x, u=u, up=up, down=down, go=go)
    return dev, host


def exact_forward(h, scaling, dtype):
    y = h["x"] @ h["W"].t() * h["scales"] + (h["bias"] if h["bias"] is not None else 0) + scaling * (h["u"] @ h["up"].t())
    return y.float().to(dtype)


def exact_transposed(h, scaling, dtype):
    gx = (h["go"] * h["scales"]) @ h["W"] + scaling * (h["u"] @ h["down"])
    return gx.float().to(dtype)


def assert_exact(y, ref, what):
    y = y.cpu()
    bad = (y.float() != ref.float()).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.shape[0]} of {y.numel()} elements differ, first at {bad[:4].tolist()}"


def one_launch(fn):
    before = _cabi.launch_count()
    out = fn()
    assert out is not None, "the fused op refused the call"
    assert _cabi.launch_count() - before == 1, "a fused call is one library launch"
    return out


RANKS = [8, 16, 64]
ADT = {"f32": lambda dt: torch.float32, "T": lambda dt: dt}


@pytest.mark.parametrize("adt", ["f32", "T"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("batch", [1, 2, 3, 4, 5, 6])
def test_gemv_lora_exact(batch, dtype, adt):
    rank = RANKS[batch % 3]
    dev, h = lattice(batch * 7 + rank, 1024, 768, 1, 16, batch, rank, dtype, ADT[adt](dtype))
    y = one_launch(lambda: ck.matmat_lora(dev["x"], dev["codes"], dev["codebooks"], dev["scales"], dev["bias"], dev["u"],
                                          dev["up"], 0.5))
    torch.cuda.synchronize()
    assert_exact(y, exact_forward(h, 0.5, dtype), f"GEMV batch {batch}")


GEMM_BATCHES = [7, 16, 17, 64, 300, 4096]
SCHEMES = [(1, 16), (2, 8), (8, 8)]


@pytest.mark.parametrize("adt", ["f32", "T"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("scheme", SCHEMES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("batch", GEMM_BATCHES)
def test_gemm_lora_exact(batch, scheme, dtype, adt):
    K, nbits = scheme
    rank = RANKS[(batch + K) % 3]
    dev, h = lattice(batch + 13 * K + rank, 512, 384, K, nbits, batch, rank, dtype, ADT[adt](dtype))
    y = one_launch(lambda: ck.matmat_dequant_lora(dev["x"], dev["codes"], dev["codebooks"], dev["scales"], dev["bias"],
                                                  dev["u"], dev["up"], 2.0))
    torch.cuda.synchronize()
    assert_exact(y, exact_forward(h, 2.0, dtype), f"GEMM batch {batch}")


@pytest.mark.parametrize("adt", ["f32", "T"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("scheme", SCHEMES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("batch", GEMM_BATCHES)
def test_transposed_lora_exact(batch, scheme, dtype, adt):
    K, nbits = scheme
    rank = RANKS[(batch + 2 * K) % 3]
    dev, h = lattice(batch + 17 * K + rank, 512, 384, K, nbits, batch, rank, dtype, ADT[adt](dtype), bias=False)
    gx = one_launch(lambda: ck.matmat_dequant_transposed_lora(dev["go"], dev["codes"], dev["codebooks"], dev["scales"],
                                                              dev["u"], dev["down"], 0.5))
    torch.cuda.synchronize()
    assert_exact(gx, exact_transposed(h, 0.5, dtype), f"transposed batch {batch}")


@pytest.mark.parametrize("forced", [dict(AQLM_B200_GEMM_KSPLIT=3), dict(AQLM_B200_GEMM_KSPLIT=5, AQLM_B200_GEMM_TILE_M=72),
                                    dict(AQLM_B200_GEMM_TILE_M=40), dict(AQLM_B200_GEMM_STAGES=2, AQLM_B200_GEMM_KSPLIT=2)],
                         ids=["ks3", "ks5-tm72", "tm40", "s2-ks2"])
@pytest.mark.parametrize("batch", [17, 300])
def test_forced_plans_exact(forced, batch):
    dtype = torch.bfloat16
    for K, nbits in [(1, 16), (2, 8)]:
        dev, h = lattice(batch + K, 1024, 520, K, nbits, batch, 64, dtype, torch.float32)
        with switches(**forced):
            y = one_launch(lambda: ck.matmat_dequant_lora(dev["x"], dev["codes"], dev["codebooks"], dev["scales"],
                                                          dev["bias"], dev["u"], dev["up"], 0.25))
            gx = one_launch(lambda: ck.matmat_dequant_transposed_lora(dev["go"], dev["codes"], dev["codebooks"],
                                                                      dev["scales"], dev["u"], dev["down"], 0.25))
            torch.cuda.synchronize()
        assert_exact(y, exact_forward(h, 0.25, dtype), f"forward {forced}")
        assert_exact(gx, exact_transposed(h, 0.25, dtype), f"transposed {forced}")


@pytest.mark.parametrize("pdl", [0, 1])
def test_adapter_rewritten_by_the_previous_kernel(pdl):
    """B (forward) and A (transposed) rewritten in place by the kernel right before the fused launch: the launch sees the
    new values, PDL on and off."""
    dtype = torch.float16
    with switches(AQLM_B200_PDL=pdl):
        for batch, op in [(3, ck.matmat_lora), (64, ck.matmat_dequant_lora)]:
            dev, h = lattice(batch + pdl, 1024, 512, 1, 16, batch, 16, dtype, torch.float32)
            torch.cuda.synchronize()
            dev["up"].neg_()  # the previous kernel of the stream
            y = op(dev["x"], dev["codes"], dev["codebooks"], dev["scales"], dev["bias"], dev["u"], dev["up"], 1.0)
            torch.cuda.synchronize()
            h["up"] = -h["up"]
            assert_exact(y, exact_forward(h, 1.0, dtype), f"B rewritten, batch {batch}")
        dev, h = lattice(5 + pdl, 1024, 512, 1, 16, 64, 16, dtype, torch.float32, bias=False)
        torch.cuda.synchronize()
        dev["down"].mul_(2.0)
        dev["u"].neg_()
        gx = ck.matmat_dequant_transposed_lora(dev["go"], dev["codes"], dev["codebooks"], dev["scales"], dev["u"],
                                               dev["down"], 1.0)
        torch.cuda.synchronize()
        h["down"], h["u"] = h["down"] * 2, -h["u"]
        assert_exact(gx, exact_transposed(h, 1.0, dtype), "A and V rewritten")


# ---- the module ------------------------------------------------------------------------------------------------------
def quantized_linear(seed, fin, fout, K, nbits, dtype, bias=True):
    dev, h = lattice(seed, fin, fout, K, nbits, 1, 8, dtype, torch.float32, bias)
    m = aqlm_b200.QuantizedLinear(fin, fout, 8, 1, K, nbits, bias=bias, device=DEV, dtype=dtype)
    with torch.no_grad():
        m.codes.copy_(dev["codes"])
        m.codebooks.copy_(dev["codebooks"])
        m.scales.copy_(dev["scales"])
        if bias:
            m.bias.copy_(dev["bias"])
    return m, h


def lora_module(seed, fin=512, fout=384, K=1, nbits=16, dtype=torch.float16, r=16, alpha=32.0, p=0.0, adt=torch.float32):
    base, h = quantized_linear(seed, fin, fout, K, nbits, dtype)
    m = aqlm_b200.LoraQuantizedLinear(base, r, alpha, p)
    torch.manual_seed(seed)
    with torch.no_grad():
        m.lora_B.weight.normal_(0, 0.05)  # PEFT starts B at zero; a trained adapter does not
    return m.to(adt) if adt != torch.float32 else m, h


def peft_reference(m, x):
    """PEFT's AQLM LoRA linear written out: base(x) + (lora_B(lora_A(dropout(x))) cast to the result's dtype) * scaling."""
    result = m.base_layer(x)
    out = torch.nn.functional.linear(torch.nn.functional.linear(m.lora_dropout(x.to(m.lora_A.weight.dtype)),
                                                                m.lora_A.weight), m.lora_B.weight)
    return result + out.to(result.dtype) * m.scaling


@pytest.mark.parametrize("case", ["rank4", "2x8-decode", "unaligned-u"])
def test_fallback_is_peft_formulation_bit_for_bit(case):
    kw = dict(rank4=dict(r=4), **{"2x8-decode": dict(K=2, nbits=8), "unaligned-u": dict(r=12)})[case]
    m, _ = lora_module(3, **kw)
    x = torch.randn(4, 512, device=DEV, dtype=torch.float16)
    with torch.no_grad():
        assert ck.matmat_lora(x, m.base_layer.codes, m.base_layer.codebooks, m.base_layer.scales, m.base_layer.bias,
                              m.lora_A(x.float()), m.lora_B.weight, m.scaling) is None
        y, ref = m(x), peft_reference(m, x)
    assert torch.equal(y, ref)


def dense_reference(m, h, x, seed, p):
    """float64 autograd model of the module: dequantized W, the same dropout mask (same seed, same RNG call)."""
    W = (h["W"] * h["scales"].reshape(-1, 1)).to(DEV)
    x64 = x.detach().double().requires_grad_(True)
    A = m.lora_A.weight.detach().double().requires_grad_(True)
    B = m.lora_B.weight.detach().double().requires_grad_(True)
    torch.manual_seed(seed)
    mask = torch.nn.functional.dropout(torch.ones_like(x, dtype=m.lora_A.weight.dtype), p, training=p > 0).double()
    y = x64 @ W.t() + h["bias"].to(DEV) + m.scaling * ((x64 * mask) @ A.t()) @ B.t()
    return y, x64, A, B


@pytest.mark.parametrize("p", [0.0, 0.2])
@pytest.mark.parametrize("rows", [4, 200])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_module_gradients_match_a_dense_float64_model(p, rows, dtype):
    m, h = lora_module(11, dtype=dtype, p=p)
    m.train()
    x = (torch.randn(rows, 512, device=DEV) * 0.5).to(dtype).requires_grad_(True)
    go = torch.randn(rows, 384, device=DEV).to(dtype)
    torch.manual_seed(99)
    y = m(x)
    y.backward(go)
    yr, x64, A, B = dense_reference(m, h, x, 99, p)
    yr.backward(go.double())
    # tolerance: T's rounding of y and grad_x (2^-8 relative for bf16) and fp32 sums of the adapter gradients
    tol = 1e-2 if dtype == torch.bfloat16 else 2e-3
    for name, got, ref in (("y", y, yr), ("grad_x", x.grad, x64.grad), ("grad_A", m.lora_A.weight.grad, A.grad),
                           ("grad_B", m.lora_B.weight.grad, B.grad)):
        err = (got.double() - ref).norm() / ref.norm().clamp_min(1e-30)
        assert err < tol, f"{name}: relative error {err:.2e} >= {tol}"


def test_cuda_graph_training_and_decode_steps_replay_after_an_optimizer_update():
    m, h = lora_module(21)
    opt = torch.optim.SGD([m.lora_A.weight, m.lora_B.weight], lr=0.1)
    x_train = torch.randn(64, 512, device=DEV, dtype=torch.float16).requires_grad_(True)
    x_dec = torch.randn(1, 512, device=DEV, dtype=torch.float16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):  # warm-up (workspace sizing) outside the capture
            opt.zero_grad(set_to_none=False)
            m(x_train).float().sum().backward()
            with torch.no_grad():
                m(x_dec)
    torch.cuda.current_stream().wait_stream(s)
    g_train, g_dec = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=False)
    with torch.cuda.graph(g_train):
        y_train = m(x_train)
        y_train.float().sum().backward()
    with torch.no_grad(), torch.cuda.graph(g_dec):
        y_dec = m(x_dec)
    for step in range(2):
        with torch.no_grad():
            m.lora_B.weight.add_(0.01 * (step + 1))  # an optimizer-like update between replays
        opt.zero_grad(set_to_none=False)
        g_train.replay()
        g_dec.replay()
        torch.cuda.synchronize()
        with torch.no_grad():
            ref_dec = peft_reference(m, x_dec)
            ref_train = m(x_train.detach())
        assert torch.equal(y_train, ref_train)
        assert (y_dec.float() - ref_dec.float()).abs().max() <= 2e-3 * ref_dec.float().abs().max()
        # the captured backward's grad_B matches an eager backward of the same step
        got = m.lora_B.weight.grad.clone()
        opt.zero_grad(set_to_none=False)
        m(x_train).float().sum().backward()
        torch.testing.assert_close(got, m.lora_B.weight.grad, rtol=1e-5, atol=1e-6)
        opt.step()


def test_llama_with_adapters_on_q_k_o_end_to_end(tmp_path):
    transformers = pytest.importorskip("transformers")  # noqa: F841
    import sys

    import transformers.quantizers.quantizer_aqlm as QA
    from test_checkpoint import write_synthetic_checkpoint
    from transformers import AutoModelForCausalLM, LlamaForCausalLM

    saved = {k: v for k, v in sys.modules.items() if k == "aqlm" or k.startswith("aqlm.")}
    aqlm_b200.install_as_aqlm()
    old = QA.is_accelerate_available
    QA.is_accelerate_available = lambda: True
    try:
        cfg, dense_sd, _ = write_synthetic_checkpoint(str(tmp_path / "m"), 1, 16)
        load = lambda: AutoModelForCausalLM.from_pretrained(str(tmp_path / "m"), dtype=torch.float16).to(DEV).eval()  # noqa: E731
        model = load()
        names = aqlm_b200.add_lora(model, ["q_proj", "k_proj", "o_proj"], r=8, lora_alpha=16)
        assert len(names) == 3 * cfg.num_hidden_layers
        torch.manual_seed(5)
        with torch.no_grad():
            for n in names:
                model.get_submodule(n).lora_B.weight.normal_(0, 0.02)
        dense = LlamaForCausalLM(cfg).half()
        dense.load_state_dict(dense_sd)
        dense = dense.to(DEV).eval()
        with torch.no_grad():
            for n in names:
                lm, dl = model.get_submodule(n), dense.get_submodule(n)
                delta = (lm.lora_B.weight @ lm.lora_A.weight) * lm.scaling
                dl.weight.copy_((dl.weight.float() + delta).half())
        ids = torch.randint(0, cfg.vocab_size, (2, 12), device=DEV)
        with torch.no_grad():
            for t in (ids, ids[:1, :3]):  # prefill (GEMM) and few rows (GEMV)
                got, ref = model(t).logits.float(), dense(t).logits.float()
                err = (got - ref).norm() / ref.norm()
                assert err < 2e-2, f"logits vs dense + torch LoRA: relative error {err:.2e}"
        aqlm_b200.save_lora_adapter(model, str(tmp_path / "adapter"))
        fresh = load()
        aqlm_b200.load_lora_adapter(fresh, str(tmp_path / "adapter"))
        with torch.no_grad():
            assert torch.equal(model(ids).logits, fresh(ids).logits)
    finally:
        QA.is_accelerate_available = old
        for k in [k for k in sys.modules if k == "aqlm" or k.startswith("aqlm.")]:
            del sys.modules[k]
        sys.modules.update(saved)
