"""LoRA adapters on quantized linears, with the adapter's up-projection fused into the base kernel.

PEFT's LoRA linear on an AQLM base computes `base(x) + lora_B(lora_A(dropout(x))) * scaling`: several launches next to
the base GEMV or GEMM and a full [T, out] tensor written, read and written again.  A quantized base cannot absorb the
adapter, so the adapter stays on the hot path for training and for serving.  `LoraQuantizedLinear` computes the
rank-sized product U = dropout(x) A^T in torch and hands U and B to the base kernel, whose epilogue adds
scaling * U B^T in fp32 before the output's one rounding: ONE launch for the base and the up-projection.

  * up to GEMV_MAX_ROWS rows: the 1x16 gather GEMV (`cuda_kernel.matmat_lora`); more: the wgmma GEMM
    (`cuda_kernel.matmat_dequant_lora`), the rule `QuantizedLinear` uses;
  * gradient w.r.t. the input: with dropout inactive (p = 0 or eval) ONE transposed wgmma GEMM that adds
    scaling * V A (V = grad_y B); with dropout active the plain transposed GEMM, and autograd adds the masked adapter
    term through U;
  * grad_A = scaling V^T dropout(x) and grad_B = scaling grad_y^T U in torch; the base stays frozen;
  * a call no fused kernel takes (another scheme at decode, a rank outside 8..64 or not a multiple of 8, adapters in a
    third dtype) runs PEFT's own formulation in torch instead.

`add_lora`, `save_lora_adapter` and `load_lora_adapter` put adapters on a model and read and write them in PEFT's
on-disk format (`adapter_config.json`, `adapter_model.safetensors` with keys `base_model.model.<module>.lora_{A,B}.weight`),
so adapters trained here load into PEFT and back.  Adapters are added before `fuse_shared_input_linears`: a set with an
adapted member is left ungrouped, because `LoraQuantizedLinear` is not a `QuantizedLinear`.
"""
from __future__ import annotations

import json
import math
import os
import re
from typing import Iterable, List, Union

import torch
from torch import nn

from .inference import QuantizedLinear, weights_require_grad

ADAPTER_CONFIG = "adapter_config.json"
ADAPTER_WEIGHTS = "adapter_model.safetensors"
_PEFT_PREFIX = "base_model.model."


def _fused_ops():
    from .inference_kernels import cuda_kernel

    return cuda_kernel


class _LoraMatmul(torch.autograd.Function):
    """y = base(x) + scaling * U B^T from ONE fused launch (`y`, computed by the caller).  Inputs x, U and B; U carries
    the graph U = dropout(x) A^T, so autograd turns grad_U = scaling grad_y B into grad_A and, with dropout active, into
    the masked adapter term of grad_x.  With dropout inactive U is computed from x detached and grad_x comes from ONE
    fused transposed launch."""

    @staticmethod
    def forward(ctx, x, u, weight_b, y, layer, fused_input_grad: bool):
        ctx.layer, ctx.fused_input_grad = layer, fused_input_grad
        ctx.save_for_backward(u, weight_b)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        layer = ctx.layer
        u, weight_b = ctx.saved_tensors
        base, s = layer.base_layer, layer.scaling
        g = grad_y.contiguous()
        v = g.to(weight_b.dtype) @ weight_b  # V = grad_y B, [..., rank]
        grad_x = grad_u = grad_b = None
        if ctx.needs_input_grad[0]:
            ck = _fused_ops()
            if ctx.fused_input_grad:
                weight_a = layer.lora_A.weight
                grad_x = ck.matmat_dequant_transposed_lora(g, base.codes, base.codebooks, base.scales, v, weight_a, s)
                if grad_x is None:  # a layout the fused kernel does not take
                    grad_x = ck.matmat_dequant_transposed(g, base.codes, base.codebooks, base.scales) + \
                        ((v @ weight_a) * s).to(g.dtype)
            else:
                grad_x = ck.matmat_dequant_transposed(g, base.codes, base.codebooks, base.scales)
        if ctx.needs_input_grad[1]:
            grad_u = v * s
        if ctx.needs_input_grad[2]:
            grad_b = (g.reshape(-1, g.shape[-1]).to(u.dtype).t() @ u.reshape(-1, u.shape[-1])) * s
        return grad_x, grad_u, grad_b, None, None, None


class LoraQuantizedLinear(nn.Module):
    """A frozen `QuantizedLinear` (`base_layer`) with one LoRA adapter, in PEFT's layout: `lora_A` (nn.Linear in ->
    r, no bias, kaiming-uniform a=sqrt(5)), `lora_B` (nn.Linear r -> out, no bias, zeros), `lora_dropout`, and
    `scaling` = lora_alpha / r (lora_alpha / sqrt(r) with rsLoRA).  The adapter is fp32, PEFT's default; it may be cast
    to the weight's dtype."""

    def __init__(self, base: QuantizedLinear, r: int, lora_alpha: float, lora_dropout: float = 0.0,
                 use_rslora: bool = False):
        super().__init__()
        if type(base) is not QuantizedLinear:
            raise TypeError(f"LoraQuantizedLinear wraps a QuantizedLinear, got {type(base).__name__}")
        if getattr(base, "_aqlm_b200_group", None) is not None:
            raise ValueError("this linear belongs to a fuse_shared_input_linears group: add adapters before fusing")
        if r < 1:
            raise ValueError(f"LoRA rank must be positive, got {r}")
        self.base_layer = base
        for p in base.parameters():
            p.requires_grad_(False)
        self.r, self.lora_alpha, self.use_rslora = int(r), lora_alpha, use_rslora
        self.scaling = lora_alpha / (math.sqrt(r) if use_rslora else r)
        self.lora_dropout = nn.Dropout(p=lora_dropout) if lora_dropout > 0.0 else nn.Identity()
        device = base.codebooks.device
        self.lora_A = nn.Linear(base.in_features, r, bias=False, device=device, dtype=torch.float32)
        self.lora_B = nn.Linear(r, base.out_features, bias=False, device=device, dtype=torch.float32)
        self.reset_lora_parameters()

    def reset_lora_parameters(self) -> None:
        nn.init.kaiming_uniform_(self.lora_A.weight, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B.weight)

    @property
    def in_features(self) -> int:
        return self.base_layer.in_features

    @property
    def out_features(self) -> int:
        return self.base_layer.out_features

    def _dropout_active(self) -> bool:
        return isinstance(self.lora_dropout, nn.Dropout) and self.training and self.lora_dropout.p > 0.0

    def peft_forward(self, x: torch.Tensor) -> torch.Tensor:
        """PEFT's formulation (its AQLM LoRA linear): base(x) + (lora_B(lora_A(dropout(x))) cast to the result's dtype) *
        scaling.  Runs where no fused kernel takes the call."""
        result = self.base_layer(x)
        out = self.lora_B(self.lora_A(self.lora_dropout(x.to(self.lora_A.weight.dtype))))
        return result + out.to(result.dtype) * self.scaling

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        base = self.base_layer
        grad = torch.is_grad_enabled()
        if grad and weights_require_grad(base):
            raise NotImplementedError("LoraQuantizedLinear keeps its base frozen: freeze codebooks, scales and bias, "
                                      "or train them without an adapter")
        if not x.is_cuda:
            return self.peft_forward(x)  # raises in the base, which has no CPU path
        wa, wb = self.lora_A.weight, self.lora_B.weight
        dropout = self._dropout_active()
        needs_grad = grad and (x.requires_grad or wa.requires_grad or wb.requires_grad)
        # U = dropout(x) A^T; with dropout inactive from x detached, so that grad_x comes from the fused launch alone
        x_for_u = x if dropout else x.detach()
        u = self.lora_A(self.lora_dropout(x_for_u.to(wa.dtype)))
        ck = _fused_ops()
        op = ck.matmat_lora if base.use_gemv_rule(x) else ck.matmat_dequant_lora
        y = op(x.detach(), base.codes, base.codebooks, base.scales, base.bias, u.detach(), wb.detach(), self.scaling)
        if y is None:
            return self.peft_forward(x)
        if not needs_grad:
            return y
        return _LoraMatmul.apply(x, u, wb, y, self, not dropout)

    def extra_repr(self) -> str:
        return f"r={self.r}, lora_alpha={self.lora_alpha}, scaling={self.scaling:g}"


# ---- model-level functions -------------------------------------------------------------------------------------------
def _matches(name: str, target_modules: Union[str, Iterable[str]]) -> bool:
    """PEFT's rule: a string is a regex the whole module name must match; a list matches a name equal to an entry or
    ending in '.' + entry."""
    if isinstance(target_modules, str):
        return re.fullmatch(target_modules, name) is not None
    return any(name == t or name.endswith("." + t) for t in target_modules)


def _set_submodule(model: nn.Module, name: str, module: nn.Module) -> None:
    parent, _, leaf = name.rpartition(".")
    setattr(model.get_submodule(parent) if parent else model, leaf, module)


def add_lora(model: nn.Module, target_modules: Union[str, List[str]], r: int, lora_alpha: float,
             lora_dropout: float = 0.0, use_rslora: bool = False) -> List[str]:
    """Wrap every `QuantizedLinear` of `model` whose name matches `target_modules` (PEFT's matching) in a
    `LoraQuantizedLinear`; returns the wrapped names.  Refuses members of `QuantizedMixtralExperts`, sharded linears,
    linears already grouped by `fuse_shared_input_linears` (add adapters first), and targets that match nothing."""
    from .moe import QuantizedMixtralExperts
    from .sharded import ShardedQuantizedLinear

    experts = [n for n, m in model.named_modules() if isinstance(m, QuantizedMixtralExperts)]
    picked = []
    for name, m in model.named_modules():
        if not name or not _matches(name, target_modules):
            continue
        if any(name.startswith(e + ".") for e in experts):
            raise NotImplementedError(f"{name}: adapters on QuantizedMixtralExperts members are not implemented")
        if isinstance(m, ShardedQuantizedLinear):
            raise NotImplementedError(f"{name}: adapters on sharded linears are not implemented")
        if isinstance(m, LoraQuantizedLinear):
            raise ValueError(f"{name} already has an adapter (one adapter per linear)")
        if type(m) is QuantizedLinear:
            if getattr(m, "_aqlm_b200_group", None) is not None:
                raise ValueError(f"{name} belongs to a fuse_shared_input_linears group: add adapters before fusing")
            picked.append((name, m))
    if not picked:
        raise ValueError(f"target_modules {target_modules!r} match no QuantizedLinear of the model")
    for name, m in picked:
        _set_submodule(model, name, LoraQuantizedLinear(m, r, lora_alpha, lora_dropout, use_rslora))
    model._aqlm_b200_lora_config = dict(target_modules=target_modules, r=r, lora_alpha=lora_alpha,
                                        lora_dropout=lora_dropout, use_rslora=use_rslora)
    return [n for n, _ in picked]


def _adapted(model: nn.Module):
    return [(n, m) for n, m in model.named_modules() if isinstance(m, LoraQuantizedLinear)]


def save_lora_adapter(model: nn.Module, save_dir: str) -> None:
    """Write the model's adapters in PEFT's format: `adapter_config.json` (peft_type LORA, task_type None) and
    `adapter_model.safetensors` with `base_model.model.<module>.lora_A.weight` / `lora_B.weight`."""
    from safetensors.torch import save_file

    mods = _adapted(model)
    if not mods:
        raise ValueError("the model has no LoRA adapters")
    m0 = mods[0][1]
    if any((m.r, m.lora_alpha, m.use_rslora) != (m0.r, m0.lora_alpha, m0.use_rslora) for _, m in mods):
        raise NotImplementedError("adapters of different ranks or alphas need rank_pattern / alpha_pattern")
    cfg = getattr(model, "_aqlm_b200_lora_config", None) or {}
    targets = cfg.get("target_modules") or sorted({n.rsplit(".", 1)[-1] for n, _ in mods})
    p = m0.lora_dropout.p if isinstance(m0.lora_dropout, nn.Dropout) else 0.0
    config = {
        "peft_type": "LORA", "task_type": None, "r": m0.r, "lora_alpha": m0.lora_alpha, "lora_dropout": p,
        "use_rslora": m0.use_rslora, "target_modules": targets if isinstance(targets, str) else list(targets),
        "bias": "none", "fan_in_fan_out": False, "modules_to_save": None, "use_dora": False, "rank_pattern": {},
        "alpha_pattern": {}, "init_lora_weights": True, "inference_mode": True, "base_model_name_or_path": None,
    }
    tensors = {}
    for name, m in mods:
        tensors[f"{_PEFT_PREFIX}{name}.lora_A.weight"] = m.lora_A.weight.detach().contiguous().cpu()
        tensors[f"{_PEFT_PREFIX}{name}.lora_B.weight"] = m.lora_B.weight.detach().contiguous().cpu()
    os.makedirs(save_dir, exist_ok=True)
    with open(os.path.join(save_dir, ADAPTER_CONFIG), "w") as f:
        json.dump(config, f, indent=2)
    save_file(tensors, os.path.join(save_dir, ADAPTER_WEIGHTS), metadata={"format": "pt"})


def _check_config(cfg: dict) -> None:
    """Refuse the PEFT options this loader does not implement."""
    if cfg.get("peft_type", "LORA") != "LORA":
        raise NotImplementedError(f"peft_type {cfg.get('peft_type')!r}: only LORA adapters load")
    refusals = [
        (cfg.get("use_dora"), "DoRA (use_dora)"),
        (cfg.get("bias", "none") != "none", f"bias={cfg.get('bias')!r} (only 'none')"),
        (cfg.get("modules_to_save"), "modules_to_save"),
        (cfg.get("fan_in_fan_out"), "fan_in_fan_out"),
        (cfg.get("rank_pattern"), "rank_pattern"),
        (cfg.get("alpha_pattern"), "alpha_pattern"),
    ]
    for bad, what in refusals:
        if bad:
            raise NotImplementedError(f"adapter_config.json: {what} is not supported by this loader")


def load_lora_adapter(model: nn.Module, load_dir: str) -> List[str]:
    """Load a PEFT LoRA adapter directory into `model`: adds the adapters of `adapter_config.json` (targets matched as
    PEFT matches them) where the model has none yet, then copies the weights (cast to each adapter's dtype).  Returns
    the adapted module names.  Refuses what `_check_config` lists, and tensors that match no adapted linear."""
    from safetensors.torch import load_file

    with open(os.path.join(load_dir, ADAPTER_CONFIG)) as f:
        cfg = json.load(f)
    _check_config(cfg)
    if not _adapted(model):
        add_lora(model, cfg["target_modules"], cfg["r"], cfg["lora_alpha"], cfg.get("lora_dropout", 0.0),
                 cfg.get("use_rslora", False))
    mods = dict(_adapted(model))
    tensors = load_file(os.path.join(load_dir, ADAPTER_WEIGHTS))
    seen = set()
    with torch.no_grad():
        for key, t in tensors.items():
            m = re.fullmatch(re.escape(_PEFT_PREFIX) + r"(.+)\.(lora_A|lora_B)(?:\.default)?\.weight", key)
            if m is None or m.group(1) not in mods:
                raise ValueError(f"adapter tensor {key!r} matches no adapted linear of the model")
            lin = getattr(mods[m.group(1)], m.group(2))
            if tuple(t.shape) != tuple(lin.weight.shape):
                raise ValueError(f"{key}: shape {tuple(t.shape)}, the model's adapter has {tuple(lin.weight.shape)}")
            lin.weight.copy_(t.to(lin.weight.dtype))
            seen.add(m.group(1))
    missing = sorted(set(mods) - seen)
    if missing:
        raise ValueError(f"adapter file has no weights for {missing}")
    return sorted(mods)
