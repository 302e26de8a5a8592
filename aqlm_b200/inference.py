"""`QuantizedLinear`: the module-level API of the AQLM hot path, CUDA (sm_90a) only.

Public contract kept from the reference module (inference_lib/src/aqlm/inference.py:11-142), because Hugging Face's AQLM
integration and existing checkpoints depend on it:
  * constructor `QuantizedLinear(in_features, out_features, in_group_size, out_group_size, num_codebooks,
    nbits_per_codebook, bias=True, device=None, dtype=None)` (inference.py:12-23), also on the meta device;
  * frozen parameters `codebooks [K, 2^nbits, og, ig]`, `codes [out/og, in/ig, K]` (signed storage of unsigned codes),
    `scales [out/og, 1, 1, 1]`, optional `bias [out]` (inference.py:39-61) -- the state_dict names / shapes / dtypes;
  * small inputs (<= 6 rows, inference.py:95-96) go to the fused GEMV op, larger ones to the fused dequant + tensor-core
    GEMM op; gradients flow to the input only (inference.py:99-142).
What differs: no CPU path (CPU inputs raise), no in-place re-layout of `codes` on first use (inference.py:78-83), no JIT
build on first call -- the ops are bound once and cached.
"""
from __future__ import annotations

import math
from typing import Callable, Optional, Tuple

import torch
from torch import nn

from .inference_kernels import get_backward_pass_kernel, get_forward_pass_kernel
from .utils import get_int_dtype

#: largest number of input rows (product of the leading dims) served by the GEMV op; same threshold as the reference
GEMV_MAX_ROWS = 6


class _AqlmMatmul(torch.autograd.Function):
    """y = op(x; codes, codebooks, scales, bias).  Only `x` receives a gradient; the quantized weight is frozen."""

    @staticmethod
    def forward(ctx, x, codes, codebooks, scales, bias, forward_op: Callable, backward_op: Callable):
        ctx.backward_op = backward_op
        ctx.save_for_backward(codes, codebooks, scales, bias)
        return forward_op(x, codes, codebooks, scales, bias)

    @staticmethod
    def backward(ctx, grad_y):
        codes, codebooks, scales, bias = ctx.saved_tensors
        grad_x = ctx.backward_op(grad_y, codes, codebooks, scales, bias)
        return grad_x, None, None, None, None, None, None


def _frozen(shape, **kwargs) -> nn.Parameter:
    return nn.Parameter(torch.empty(shape, **kwargs), requires_grad=False)


class QuantizedLinear(nn.Module):
    def __init__(
        self,
        in_features: int,
        out_features: int,
        in_group_size: int,
        out_group_size: int,
        num_codebooks: int,
        nbits_per_codebook: int,
        bias=True,
        device=None,
        dtype=None,
    ):
        super().__init__()
        if in_features % in_group_size or out_features % out_group_size:
            raise AssertionError(f"features ({in_features}, {out_features}) must be multiples of the group sizes "
                                 f"({in_group_size}, {out_group_size})")
        self.in_features, self.out_features = in_features, out_features
        self.in_group_size, self.out_group_size = in_group_size, out_group_size
        self.num_codebooks, self.nbits_per_codebook = num_codebooks, nbits_per_codebook
        self.codebook_size = 1 << nbits_per_codebook
        out_groups, in_groups = out_features // out_group_size, in_features // in_group_size

        self.codebooks = _frozen((num_codebooks, self.codebook_size, out_group_size, in_group_size), device=device,
                                 dtype=dtype)
        self.codes = _frozen((out_groups, in_groups, num_codebooks), device=device,
                             dtype=get_int_dtype(nbits_per_codebook))
        self.scales = _frozen((out_groups, 1, 1, 1), device=device, dtype=dtype)
        if bias:
            self.bias = _frozen((out_features,), device=device, dtype=dtype)
        else:
            self.register_parameter("bias", None)
        self._ops: Optional[Tuple[Callable, Callable, Callable, Callable]] = None  # (gemv fwd, gemv bwd, gemm fwd, gemm bwd)

    # -- kernel binding ---------------------------------------------------------------------------------------------
    def prepare_matmul_op(self, input: torch.Tensor) -> None:
        """Bind the four ops for this module's scheme (reference inference.py:77-96).  CUDA only."""
        if not input.is_cuda:
            raise NotImplementedError(
                f"aqlm_b200.QuantizedLinear runs on CUDA (sm_90a) only; got input on {input.device}. "
                "There is no CPU fallback in this package.")
        self._ops = tuple(select(self.codebooks, large_batch)
                          for large_batch in (False, True)
                          for select in (get_forward_pass_kernel, get_backward_pass_kernel))

    # names kept for code that pokes at the reference's attributes
    @property
    def gemv_op(self):
        return None if self._ops is None else self._ops[0]

    @property
    def gemm_op(self):
        return None if self._ops is None else self._ops[2]

    def use_gemv_rule(self, input: torch.Tensor) -> bool:
        return math.prod(input.shape[:-1]) <= GEMV_MAX_ROWS

    # -- forward ----------------------------------------------------------------------------------------------------
    def forward(self, input: torch.Tensor) -> torch.Tensor:
        if self._ops is None:
            self.prepare_matmul_op(input)
        fwd, bwd = self._ops[:2] if self.use_gemv_rule(input) else self._ops[2:]
        if not (torch.is_grad_enabled() and input.requires_grad):
            return fwd(input, self.codes, self.codebooks, self.scales, self.bias)  # inference: skip the autograd node
        return _AqlmMatmul.apply(input, self.codes, self.codebooks, self.scales, self.bias, fwd, bwd)

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, "
                f"scheme={self.num_codebooks}x{self.nbits_per_codebook}, in_group_size={self.in_group_size}, "
                f"bias={self.bias is not None}")
