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
