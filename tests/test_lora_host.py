"""CPU tests of the LoRA surface: argument checks of the three adapter entry points (no device is queried before them),
the module on the meta device, PEFT's on-disk format both ways, and every refusal of add_lora / load_lora_adapter."""
import ctypes
import json
import os

import pytest
import torch
from torch import nn

import aqlm_b200
from aqlm_b200 import LoraQuantizedLinear, QuantizedLinear, _cabi, add_lora, load_lora_adapter, save_lora_adapter

safetensors_torch = pytest.importorskip("safetensors.torch")


def _weight(K=1, nbits=16, g=8, in_f=256, out_f=128):
    w = _cabi.Weight()
    w.codes, w.codebooks, w.scales = 256, 256, 256  # dummy aligned pointers (never dereferenced)
    w.in_features, w.out_features = in_f, out_f
    w.num_codebooks, w.nbits_per_codebook, w.in_group_size, w.out_group_size = K, nbits, g, 1
    w.dtype = _cabi.F16
    return w


def _lora(rank=16, dtype=_cabi.F32):
    d = _cabi.Lora()
    d.down, d.up, d.rank, d.dtype, d.scaling = 512, 512, rank, dtype, 2.0
    return d


def _calls(L, w, d, lin=1024, a=2048, y=4096, batch=16):
    ws = (None, 0, None)
    return {
        "gemv": L.aqlm_b200_matmat_lora(ctypes.byref(w), d, a, lin, y, min(batch, 8), None),
        "gemm": L.aqlm_b200_matmat_dequant_lora(ctypes.byref(w), d, a, lin, y, batch, *ws),
        "transposed": L.aqlm_b200_matmat_dequant_transposed_lora(ctypes.byref(w), d, a, lin, y, batch, *ws),
    }


def test_lora_struct_matches_header_layout():
    assert ctypes.sizeof(_cabi.Lora) == 2 * 8 + 3 * 4 + 4  # two pointers, rank, dtype, scaling, tail padding
    assert _cabi.Lora.rank.offset == 16 and _cabi.Lora.scaling.offset == 24


def test_adapter_entry_points_check_arguments_without_a_device():
    L = _cabi.lib()
    w, d = _weight(), _lora()
    for name, rc in _calls(L, w, None).items():
        assert rc == _cabi.ERR_SHAPE, name  # NULL adapter descriptor
    for rank in (0, 4, 12, 72, 128):
        for name, rc in _calls(L, w, ctypes.byref(_lora(rank))).items():
            assert rc == _cabi.ERR_UNSUPPORTED, (name, rank)
            assert b"rank" in L.aqlm_b200_last_error()
    for name, rc in _calls(L, w, ctypes.byref(_lora(16, _cabi.BF16))).items():
        assert rc == _cabi.ERR_DTYPE, name  # neither fp32 nor the weight's dtype
    for name, rc in _calls(L, w, ctypes.byref(d), lin=None).items():
        assert rc == _cabi.ERR_SHAPE, name
    for name, rc in _calls(L, w, ctypes.byref(d), lin=1032).items():
        assert rc == _cabi.ERR_UNSUPPORTED, name  # U / V not 16-byte aligned
    for name, rc in _calls(L, w, ctypes.byref(d), batch=-1).items():
        assert rc == _cabi.ERR_SHAPE, name
    up_null = _lora()
    up_null.up = None
    rcs = _calls(L, w, ctypes.byref(up_null))
    assert rcs["gemv"] == rcs["gemm"] == _cabi.ERR_SHAPE and rcs["transposed"] != _cabi.ERR_SHAPE
    # layouts without a fused kernel: ERR_UNSUPPORTED, never another rounding
    assert _calls(L, _weight(K=2, nbits=8), ctypes.byref(d))["gemv"] == _cabi.ERR_UNSUPPORTED
    assert L.aqlm_b200_matmat_lora(ctypes.byref(w), ctypes.byref(d), 2048, 1024, 4096, 9, None) == _cabi.ERR_UNSUPPORTED
    g16 = _calls(L, _weight(g=16), ctypes.byref(d))
    assert g16["gemv"] == g16["gemm"] == g16["transposed"] == _cabi.ERR_UNSUPPORTED
    odd = _calls(L, _weight(in_f=200), ctypes.byref(d))
    assert odd["gemm"] == _cabi.ERR_UNSUPPORTED  # in_features % 64 != 0
    assert _calls(L, _weight(out_f=100), ctypes.byref(d))["transposed"] == _cabi.ERR_UNSUPPORTED  # out % 8 != 0
    # batch 0 of a valid call: no launch, no device needed
    assert set(_calls(L, w, ctypes.byref(d), batch=0).values()) == {_cabi.OK}


def _base(device="meta", out_f=128, in_f=256):
    return QuantizedLinear(in_f, out_f, 8, 1, 1, 16, bias=False, device=device, dtype=torch.float16)


def test_module_on_meta_has_peft_names_shapes_and_init():
    m = LoraQuantizedLinear(_base(), r=8, lora_alpha=16, lora_dropout=0.1)
    assert [k for k in m.state_dict()] == ["base_layer.codebooks", "base_layer.codes", "base_layer.scales",
                                           "lora_A.weight", "lora_B.weight"]
    assert m.lora_A.weight.shape == (8, 256) and m.lora_B.weight.shape == (128, 8)
    assert m.lora_A.weight.dtype == m.lora_B.weight.dtype == torch.float32
    assert isinstance(m.lora_A, nn.Linear) and m.lora_A.bias is None and m.lora_B.bias is None
    assert m.scaling == 2.0 and isinstance(m.lora_dropout, nn.Dropout) and m.lora_dropout.p == 0.1
    assert LoraQuantizedLinear(_base(), r=16, lora_alpha=16, use_rslora=True).scaling == 4.0
    assert not isinstance(m, QuantizedLinear)
    assert not any(p.requires_grad for p in m.base_layer.parameters())
    cpu = LoraQuantizedLinear(_base("cpu"), r=8, lora_alpha=8)
    assert torch.count_nonzero(cpu.lora_B.weight) == 0
    bound = 1 / 256 ** 0.5  # kaiming_uniform(a=sqrt(5)) on [8, 256]: U(-1/sqrt(in), 1/sqrt(in))
    assert cpu.lora_A.weight.abs().max() <= bound and cpu.lora_A.weight.std() > bound / 4


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.q_proj, self.k_proj, self.o_proj = _base("cpu"), _base("cpu"), _base("cpu", out_f=256, in_f=128)
        self.norm = nn.LayerNorm(256)


class _Model(nn.Module):
    def __init__(self, n=2):
        super().__init__()
        self.layers = nn.ModuleList(_Block() for _ in range(n))


def test_targets_match_as_peft_matches_them():
    m = _Model()
    assert add_lora(m, ["q_proj", "o_proj"], 8, 16) == ["layers.0.q_proj", "layers.0.o_proj", "layers.1.q_proj",
                                                        "layers.1.o_proj"]
    assert isinstance(m.layers[1].q_proj, LoraQuantizedLinear) and type(m.layers[1].k_proj) is QuantizedLinear
    m = _Model()
    assert add_lora(m, r"layers\.1\.(q|k)_proj", 8, 16) == ["layers.1.q_proj", "layers.1.k_proj"]
    with pytest.raises(ValueError, match="match no QuantizedLinear"):
        add_lora(_Model(), r"q_proj", 8, 16)  # a string is a full-name regex, not a suffix
    with pytest.raises(ValueError, match="already has an adapter"):
        add_lora(m, ["q_proj"], 8, 16)


def _write_peft_dir(path, names, r=8, alpha=16, **cfg_overrides):
    cfg = {"peft_type": "LORA", "task_type": "CAUSAL_LM", "r": r, "lora_alpha": alpha, "lora_dropout": 0.05,
           "target_modules": ["q_proj", "o_proj"], "bias": "none", "fan_in_fan_out": False, "modules_to_save": None,
           "use_dora": False, "use_rslora": False, "rank_pattern": {}, "alpha_pattern": {}}
    cfg.update(cfg_overrides)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "adapter_config.json"), "w") as f:
        json.dump(cfg, f)
    g = torch.Generator().manual_seed(0)
    tensors = {}
    for n, (i, o) in names.items():
        tensors[f"base_model.model.{n}.lora_A.weight"] = torch.randn(r, i, generator=g)
        tensors[f"base_model.model.{n}.lora_B.weight"] = torch.randn(o, r, generator=g)
    safetensors_torch.save_file(tensors, os.path.join(path, "adapter_model.safetensors"))
    return tensors


def test_a_peft_directory_loads_and_saves_back_with_the_same_keys_and_config(tmp_path):
    names = {f"layers.{i}.{p}": (256, 128) if p == "q_proj" else (128, 256) for i in range(2) for p in ("q_proj", "o_proj")}
    tensors = _write_peft_dir(str(tmp_path / "peft"), names)
    m = _Model()
    assert load_lora_adapter(m, str(tmp_path / "peft")) == sorted(names)
    lq = m.layers[1].o_proj
    assert isinstance(lq, LoraQuantizedLinear) and lq.scaling == 2.0 and lq.lora_dropout.p == 0.05
    assert torch.equal(lq.lora_B.weight, tensors["base_model.model.layers.1.o_proj.lora_B.weight"])
    save_lora_adapter(m, str(tmp_path / "ours"))
    back = safetensors_torch.load_file(str(tmp_path / "ours" / "adapter_model.safetensors"))
    assert sorted(back) == sorted(tensors)
    for k in tensors:
        assert torch.equal(back[k], tensors[k]) and back[k].dtype == torch.float32
    with open(tmp_path / "ours" / "adapter_config.json") as f:
        cfg = json.load(f)
    assert (cfg["peft_type"], cfg["r"], cfg["lora_alpha"], cfg["lora_dropout"], cfg["bias"], cfg["use_dora"],
            cfg["use_rslora"], cfg["target_modules"]) == ("LORA", 8, 16, 0.05, "none", False, False, ["q_proj", "o_proj"])
    # and our directory loads into a fresh model with equal weights
    fresh = _Model()
    load_lora_adapter(fresh, str(tmp_path / "ours"))
    adapters = {k: v for k, v in fresh.state_dict().items() if ".lora_" in k}
    assert len(adapters) == 8
    for k, v in adapters.items():
        assert torch.equal(v, m.state_dict()[k]), k


@pytest.mark.parametrize("override,match", [
    ({"use_dora": True}, "DoRA"), ({"bias": "lora_only"}, "bias"), ({"modules_to_save": ["lm_head"]}, "modules_to_save"),
    ({"fan_in_fan_out": True}, "fan_in_fan_out"), ({"rank_pattern": {"q_proj": 16}}, "rank_pattern"),
    ({"alpha_pattern": {"q_proj": 32}}, "alpha_pattern"), ({"peft_type": "IA3"}, "peft_type"),
])
def test_loader_refuses_what_it_does_not_implement(tmp_path, override, match):
    _write_peft_dir(str(tmp_path), {"layers.0.q_proj": (256, 128)}, **override)
    with pytest.raises(NotImplementedError, match=match):
        load_lora_adapter(_Model(), str(tmp_path))


def test_loader_refuses_tensors_that_match_no_adapted_linear(tmp_path):
    _write_peft_dir(str(tmp_path), {"layers.0.q_proj": (256, 128), "layers.0.v_proj": (256, 128)})
    with pytest.raises(ValueError, match="v_proj"):
        load_lora_adapter(_Model(), str(tmp_path))


def test_add_lora_refuses_experts_sharded_and_grouped_linears():
    from aqlm_b200.moe import QuantizedMixtralExperts
    from aqlm_b200.sharded import ShardedQuantizedLinear

    class WithExperts(nn.Module):
        def __init__(self):
            super().__init__()
            self.experts = QuantizedMixtralExperts(2, 64, 128, torch.nn.functional.silu, 8, 1, 1, 16,
                                                   device="meta", dtype=torch.float16)

    with pytest.raises(NotImplementedError, match="QuantizedMixtralExperts"):
        add_lora(WithExperts(), ["w1"], 8, 16)

    class WithSharded(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj = ShardedQuantizedLinear(256, 128, 8, 1, 1, 16, bias=False, rank=0, world_size=1,
                                                 device="meta", dtype=torch.float16)

    with pytest.raises(NotImplementedError, match="sharded"):
        add_lora(WithSharded(), ["q_proj"], 8, 16)

    m = _Model(1)
    m.layers[0].q_proj._aqlm_b200_group = object()  # what fuse_shared_input_linears marks its members with
    with pytest.raises(ValueError, match="before fusing"):
        add_lora(m, ["q_proj"], 8, 16)
    with pytest.raises(ValueError, match="before fusing"):
        LoraQuantizedLinear(m.layers[0].q_proj, 8, 16)


def test_trainable_base_weights_are_refused():
    m = LoraQuantizedLinear(_base("cpu"), 8, 16)
    m.base_layer.scales.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="frozen"):
        m(torch.zeros(1, 256, dtype=torch.float16))


def test_package_exports():
    for name in ("LoraQuantizedLinear", "add_lora", "save_lora_adapter", "load_lora_adapter"):
        assert hasattr(aqlm_b200, name)
