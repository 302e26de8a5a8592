"""Checkpoint-format path (SURVEY §8 f2): a synthetic Llama checkpoint written in the reference converter's format
(convert_to_hf.py:50-100: config.json `quantization_config` block, `<linear>.codes` packed ints, `.codebooks`/`.scales`
fp16, everything else fp16) must load through `AutoModelForCausalLM.from_pretrained` -- Hugging Face's own AQLM
integration -- into OUR `QuantizedLinear` modules, report a version through `importlib.metadata`, and on an H100 produce
the logits of a dense model holding the dequantized weights.

Environment notes: (1) the image has no `accelerate`; HF's AQLM quantizer only CHECKS for it (`validate_environment`),
so the tests patch that one check. (2) transformers >= 5 matches `linear_weights_not_to_quantize` against MODULE names
(`should_convert_module`), while the reference converter writes PARAMETER names (`lm_head.weight`); the synthetic
checkpoint lists both, as a real checkpoint has to for this transformers version.
"""
import sys

import numpy as np
import pytest
import torch

from oracle import aqlm_oracle as O

transformers = pytest.importorskip("transformers")


@pytest.fixture
def aqlm_alias(monkeypatch):
    import aqlm_b200

    saved = {k: v for k, v in sys.modules.items() if k == "aqlm" or k.startswith("aqlm.")}
    aqlm_b200.install_as_aqlm()
    import transformers.quantizers.quantizer_aqlm as QA

    monkeypatch.setattr(QA, "is_accelerate_available", lambda: True)
    yield aqlm_b200
    for k in [k for k in sys.modules if k == "aqlm" or k.startswith("aqlm.")]:
        del sys.modules[k]
    sys.modules.update(saved)


def write_synthetic_checkpoint(path, K, nbits, seed=0, hidden=128, inter=256, layers=2, heads=4, kv_heads=2, vocab=96):
    """Returns (LlamaConfig, dense state dict with the dequantized weights, the checkpoint's state dict)."""
    from transformers import LlamaConfig, LlamaForCausalLM

    from aqlm_b200 import hf

    cfg = LlamaConfig(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=heads,
                      num_key_value_heads=kv_heads, vocab_size=vocab, max_position_embeddings=64, tie_word_embeddings=False)
    torch.manual_seed(seed)
    dense = LlamaForCausalLM(cfg).half()
    rng = np.random.default_rng(seed)
    ckpt, dense_sd, not_quantized = {}, {}, []
    for name, p in dense.state_dict().items():
        if name.endswith("_proj.weight"):
            out_f, in_f = p.shape
            codes = rng.integers(0, 2**nbits, size=(out_f, in_f // 8, K))
            cb = (rng.standard_normal((K, 2**nbits, 1, 8)) * (0.08 / K**0.5)).astype(np.float16)
            sc = (0.75 + 0.5 * rng.random((out_f, 1, 1, 1))).astype(np.float16)
            ckpt.update(hf.quantized_state_entries(name[: -len(".weight")], torch.from_numpy(codes), torch.from_numpy(cb),
                                                   torch.from_numpy(sc), nbits))
            W = O.dequantize_weight(codes, cb.astype(np.float32), sc.astype(np.float32))
            dense_sd[name] = torch.from_numpy(W).half()
        else:
            ckpt[name] = p.half()
            dense_sd[name] = p.half()
            not_quantized.append(name)
    if "lm_head.weight" not in not_quantized:
        not_quantized.append("lm_head.weight")
    not_quantized.append("lm_head")  # module-name form for transformers >= 5 (see the module docstring)
    hf.save_quantized_checkpoint(path, cfg.to_dict(), ckpt,
                                 hf.quantization_config_dict(K, nbits, linear_weights_not_to_quantize=not_quantized))
    return cfg, dense_sd, ckpt


@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_from_pretrained_builds_our_modules_and_reports_a_version(tmp_path, aqlm_alias, K, nbits):
    from importlib import metadata

    from packaging import version
    from transformers import AutoModelForCausalLM

    cfg, _, ckpt = write_synthetic_checkpoint(str(tmp_path / "m"), K, nbits)
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "m"), dtype=torch.float16)
    n = 0
    for name, mod in model.named_modules():
        if name.endswith("_proj"):
            assert type(mod) is aqlm_alias.QuantizedLinear, (name, type(mod))
            assert torch.equal(mod.codes, ckpt[f"{name}.codes"]) and mod.codes.dtype == (torch.int8 if nbits <= 8 else torch.int16)
            assert torch.equal(mod.codebooks, ckpt[f"{name}.codebooks"]) and torch.equal(mod.scales, ckpt[f"{name}.scales"])
            n += 1
    assert n == 7 * cfg.num_hidden_layers
    assert isinstance(model.lm_head, torch.nn.Linear)
    # HF's AqlmHfQuantizer.is_trainable reads the distribution version (quantizer_aqlm.py:65)
    assert version.parse(metadata.version("aqlm")) >= version.parse("1.1.6")
    assert model.hf_quantizer.is_trainable is True
    # round trip: the loaded model's state dict has the checkpoint's names/shapes/dtypes
    sd = model.state_dict()
    for k, v in ckpt.items():
        assert k in sd and sd[k].shape == v.shape and sd[k].dtype == v.dtype, k


@pytest.mark.gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8), (1, 8)])
def test_checkpoint_logits_match_dense_dequantized_model(tmp_path, aqlm_alias, K, nbits):
    from transformers import AutoModelForCausalLM, LlamaForCausalLM

    cfg, dense_sd, _ = write_synthetic_checkpoint(str(tmp_path / "m"), K, nbits, seed=3)
    model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "m"), dtype=torch.float16).to("cuda:0").eval()
    dense = LlamaForCausalLM(cfg).half()
    dense.load_state_dict(dense_sd)
    dense = dense.to("cuda:0").eval()
    ids = torch.randint(0, cfg.vocab_size, (1, 5), device="cuda:0")
    from aqlm_b200 import _cabi

    before = _cabi.launch_count()
    with torch.no_grad():
        lq = model(ids).logits.float()          # 5 rows: GEMV op
        ld = dense(ids).logits.float()
        lq_big = model(ids.repeat(4, 1)).logits.float()  # 20 rows: tensor-core op
    assert _cabi.launch_count() > before
    rel = ((lq - ld).abs().mean() / ld.abs().mean()).item()
    assert rel < 5e-3, rel
    assert ((lq_big[0] - ld[0]).abs().mean() / ld.abs().mean()).item() < 5e-3
    if (K, nbits) == (1, 16):
        # grouped q/k/v and gate/up launches wired into the loaded model: same logits, fewer launches, names unchanged
        import aqlm_b200

        names = sorted(model.state_dict().keys())
        one = ids[:, :1]
        with torch.no_grad():
            ref1 = model(one).logits
            c0 = _cabi.launch_count()
            model(one)
            plain_launches = _cabi.launch_count() - c0
            n_groups = aqlm_b200.fuse_shared_input_linears(model)
            assert n_groups == 2 * cfg.num_hidden_layers
            c0 = _cabi.launch_count()
            fused1 = model(one).logits
            fused_launches = _cabi.launch_count() - c0
            out = model.generate(one, max_new_tokens=4, min_new_tokens=4, do_sample=False)
        assert torch.equal(ref1, fused1)
        assert fused_launches == plain_launches - 3 * cfg.num_hidden_layers
        assert sorted(model.state_dict().keys()) == names
        assert out.shape == (1, 5)
