"""Model-level glue either side of the hot path (SURVEY §8 f1/f2): checkpoints in the reference's Hugging Face format and
grouped launches wired into a loaded model.

* `save_quantized_checkpoint` writes a directory in the format the reference's `convert_to_hf.py:50-100` produces
  (`config.json` with a `quantization_config` block {quant_method: aqlm, nbits_per_codebook, num_codebooks, out_group_size,
  in_group_size, linear_weights_not_to_quantize}; a state dict whose quantized linears are stored as `<name>.codes`
  (packed ints, `utils.pack_int_data`), `<name>.codebooks`, `<name>.scales` (fp16) and everything else as fp16).
  `AutoModelForCausalLM.from_pretrained(dir)` then builds `aqlm.QuantizedLinear` modules through Hugging Face's own AQLM
  integration (`transformers/integrations/aqlm.py`) -- with `aqlm_b200.install_as_aqlm()` those are OUR modules.
* `fuse_shared_input_linears` finds, in a loaded model, the quantized linears that read the same activation (attention
  q/k/v, MLP gate/up) and makes each set run as ONE grouped launch (`QuantizedLinearGroup`: the grouped GEMV at decode,
  the grouped GEMM at prefill and in training), without changing module names, the state dict, or the model's forward
  code: the members' `forward` is routed through a small per-group cache.
* `load_quantized_mixtral` loads an AQLM Mixtral checkpoint (e.g. `ISTA-DASLab/Mixtral-8x7b-AQLM-2Bit-1x16-hf`) with
  quantized experts.  `from_pretrained` alone cannot: in transformers 5.x a Mixtral block keeps all its experts as two
  dense 3-D parameters (`MixtralExperts.gate_up_proj` / `down_proj`), Hugging Face's AQLM integration replaces
  `nn.Linear` modules only, so the experts stay dense placeholders (about 90 GB of fp16 for Mixtral-8x7B) and the
  checkpoint's per-expert tensors `block_sparse_moe.experts.{e}.w{1,2,3}.{codes,codebooks,scales}` have nowhere to
  load.  `replace_mixtral_experts` swaps every block's experts for `moe.QuantizedMixtralExperts` (one routed GEMM per
  projection over all experts), whose state-dict names are the checkpoint's.
"""
from __future__ import annotations

import json
import os
import types
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch
from torch import nn

from .grouped import QuantizedLinearGroup, _rows, gemm_scheme
from .inference import QuantizedLinear
from .moe import QuantizedMixtralExperts
from .utils import pack_int_data

#: attribute-name sets of linears that share their input, per parent module (Llama / Mistral / Qwen2 / Gemma layouts)
SHARED_INPUT_SETS: Tuple[Tuple[str, ...], ...] = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


class _SharedInputGroup:
    """Runs the members as one grouped launch the first time any of them sees a new activation and hands the other
    members their slice when they are called with the SAME tensor object (q_proj(x), k_proj(x), v_proj(x) in HF code)."""

    def __init__(self, members: Sequence[QuantizedLinear]):
        self.group = QuantizedLinearGroup(list(members))
        self._x: Optional[torch.Tensor] = None
        self._version = -1
        self._outs: Optional[Tuple[torch.Tensor, ...]] = None
        self._left = 0
        self._in_group = False

    def member_forward(self, index: int, member: QuantizedLinear, x: torch.Tensor) -> torch.Tensor:
        rows = _rows(x)
        # the group's own fallback to its members (a layout no grouped kernel takes) lands here: the member's own op
        if self._in_group or not self.group.fused or rows < 1:
            return QuantizedLinear.forward(member, x)
        if self._x is not x or self._version != x._version:  # a new activation (or the same tensor modified in place)
            self._in_group = True
            try:
                self._outs = self.group(x)  # decode, prefill and training: one grouped launch where a kernel takes it
            finally:
                self._in_group = False
            self._x, self._version, self._left = x, x._version, len(self._outs)
        y = self._outs[index]
        self._left -= 1
        if self._left <= 0:  # every member consumed its slice: drop the references
            self._x = self._outs = None
        return y


def fuse_shared_input_linears(model: nn.Module, sets: Iterable[Sequence[str]] = SHARED_INPUT_SETS) -> int:
    """Group q/k/v and gate/up `QuantizedLinear`s of every block of `model` (already on its final CUDA device).
    Returns the number of groups created.  Module names and `state_dict()` are unchanged; call once, after loading."""
    created = 0
    keep: List[_SharedInputGroup] = []
    for parent in model.modules():
        for names in sets:
            members = [getattr(parent, n, None) for n in names]
            if not all(isinstance(m, QuantizedLinear) for m in members):
                continue
            if any(getattr(m, "_aqlm_b200_group", None) is not None for m in members):
                continue
            m0 = members[0]
            if not m0.codes.is_cuda or not gemm_scheme(m0):
                continue
            if any(m.in_features != m0.in_features or (m.bias is None) != (m0.bias is None) for m in members):
                continue
            shared = _SharedInputGroup(members)
            for i, m in enumerate(members):
                m._aqlm_b200_group = shared
                m.forward = types.MethodType(lambda self, x, _i=i, _g=shared: _g.member_forward(_i, self, x), m)
            keep.append(shared)
            created += 1
    model._aqlm_b200_groups = getattr(model, "_aqlm_b200_groups", []) + keep
    return created


def quantization_config_dict(num_codebooks: int, nbits_per_codebook: int, in_group_size: int = 8, out_group_size: int = 1,
                             linear_weights_not_to_quantize: Optional[List[str]] = None) -> Dict:
    """The `quantization_config` block of config.json (reference convert_to_hf.py:90-98)."""
    return {
        "quant_method": "aqlm",
        "nbits_per_codebook": nbits_per_codebook,
        "num_codebooks": num_codebooks,
        "out_group_size": out_group_size,
        "in_group_size": in_group_size,
        "linear_weights_not_to_quantize": list(linear_weights_not_to_quantize or []),
    }


def quantized_state_entries(prefix: str, codes_unsigned: torch.Tensor, codebooks: torch.Tensor, scales: torch.Tensor,
                            nbits: int, bias: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """State-dict entries of one quantized linear exactly as the reference converter stores them
    (convert_to_hf.py:59-68: floats -> fp16, integer codes -> pack_int_data)."""
    out = {
        f"{prefix}.codes": pack_int_data(codes_unsigned.clone().to(torch.int64), nbits),
        f"{prefix}.codebooks": codebooks.half(),
        f"{prefix}.scales": scales.half(),
    }
    if bias is not None:
        out[f"{prefix}.bias"] = bias.half()
    return out


def save_quantized_checkpoint(save_dir: str, config_dict: Dict, state_dict: Dict[str, torch.Tensor],
                              quantization_config: Dict) -> str:
    """Write `config.json` (+ quantization_config, torch_dtype float16 as in convert_to_hf.py:90-98) and the weights
    (`model.safetensors` when safetensors is importable, else `pytorch_model.bin`)."""
    os.makedirs(save_dir, exist_ok=True)
    cfg = dict(config_dict)
    cfg["quantization_config"] = quantization_config
    cfg["torch_dtype"] = "float16"
    with open(os.path.join(save_dir, "config.json"), "w") as f:
        json.dump(cfg, f, indent=2)
    tensors = {k: v.detach().cpu().contiguous() for k, v in state_dict.items()}
    try:
        from safetensors.torch import save_file

        save_file(tensors, os.path.join(save_dir, "model.safetensors"), metadata={"format": "pt"})
    except ImportError:
        torch.save(tensors, os.path.join(save_dir, "pytorch_model.bin"))
    return save_dir


def _aqlm_config(model: nn.Module) -> Dict:
    qc = getattr(model.config, "quantization_config", None)
    if qc is None:
        raise ValueError("the model's config has no quantization_config (not an AQLM checkpoint)")
    return qc if isinstance(qc, dict) else qc.to_dict()


def replace_mixtral_experts(model: nn.Module) -> int:
    """Swap the experts of every `MixtralSparseMoeBlock` of `model` for `QuantizedMixtralExperts` with the model's AQLM
    scheme, on the device (meta included) and in the dtype of the block's router.  Returns the number of blocks."""
    from transformers.models.mixtral.modeling_mixtral import MixtralSparseMoeBlock

    qc = _aqlm_config(model)
    n = 0
    for block in model.modules():
        if not isinstance(block, MixtralSparseMoeBlock) or isinstance(block.experts, QuantizedMixtralExperts):
            continue
        old, w = block.experts, block.gate.weight
        block.experts = QuantizedMixtralExperts(
            old.num_experts, old.hidden_dim, old.intermediate_dim, old.act_fn, in_group_size=qc["in_group_size"],
            out_group_size=qc["out_group_size"], num_codebooks=qc["num_codebooks"],
            nbits_per_codebook=qc["nbits_per_codebook"], device=w.device, dtype=w.dtype)
        n += 1
    return n


def _checkpoint_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """Every tensor of the checkpoint directory (safetensors shards, else `.bin` shards), by name."""
    files = sorted(f for f in os.listdir(path) if f.endswith(".safetensors"))
    sd: Dict[str, torch.Tensor] = {}
    if files:
        from safetensors.torch import load_file

        for f in files:
            sd.update(load_file(os.path.join(path, f)))
        return sd
    for f in sorted(f for f in os.listdir(path) if f.endswith(".bin")):
        sd.update(torch.load(os.path.join(path, f), map_location="cpu", weights_only=True))
    if not sd:
        raise FileNotFoundError(f"no .safetensors or .bin weights in {path}")
    return sd


def load_quantized_mixtral(path: str, dtype: torch.dtype = torch.float16, device="cuda") -> nn.Module:
    """Load an AQLM Mixtral checkpoint directory with quantized experts (see the module docstring for why
    `from_pretrained` does not).  The model is built on the meta device, Hugging Face's `replace_with_aqlm_linear` makes
    the attention projections `QuantizedLinear`s (ours, through `install_as_aqlm`), `replace_mixtral_experts` the
    experts; the weights are loaded by name (`.block_sparse_moe.` renamed to `.mlp.`, as transformers does) strictly,
    then the model moves to `device`.  No dense expert tensor is ever allocated."""
    from transformers import AutoConfig, AutoModelForCausalLM
    from transformers.integrations.aqlm import replace_with_aqlm_linear
    from transformers.utils.quantization_config import AqlmConfig

    from . import install_as_aqlm

    install_as_aqlm()  # replace_with_aqlm_linear builds `aqlm.QuantizedLinear`
    config = AutoConfig.from_pretrained(path)
    with torch.device("meta"):
        model = AutoModelForCausalLM.from_config(config, dtype=dtype)
    qc = _aqlm_config(model)
    # the reference converter lists PARAMETER names (`lm_head.weight`); transformers >= 5 matches MODULE names
    keep = list(qc.get("linear_weights_not_to_quantize") or [])
    keep += [n[: -len(".weight")] for n in keep if n.endswith(".weight")]
    replace_with_aqlm_linear(model, modules_to_not_convert=keep, quantization_config=AqlmConfig.from_dict(qc))
    replace_mixtral_experts(model)
    sd = {k.replace(".block_sparse_moe.", ".mlp."): v for k, v in _checkpoint_state_dict(path).items()}
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    if getattr(config, "tie_word_embeddings", False) and "lm_head.weight" not in sd:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    model.load_state_dict(sd, strict=True, assign=True)
    if getattr(config, "tie_word_embeddings", False):
        model.tie_weights()
    for m in model.modules():
        if isinstance(m, QuantizedMixtralExperts):
            m.fuse_storage()  # the load replaced the members' parameters
    # modules with buffers that are not in the checkpoint (the rotary embedding's inverse frequencies) still hold meta
    # tensors: build them again for real
    for name, mod in list(model.named_modules()):
        if any(b.is_meta for b in mod.buffers(recurse=False)):
            model.set_submodule(name, type(mod)(mod.config, device="cpu"))
    return model.to(device).eval()
