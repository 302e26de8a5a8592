"""Shape/device -> kernel table (reference inference_kernels/kernel_selector.py:21-163).

Same signature and the same op names as the reference for the schemes it has CUDA kernels for; every other
KxN scheme with out_group_size == 1 gets `aqlm::generic_matmat*` (the reference uses Triton, 91-94, or
embedding_bag + F.linear, 99-102).  Non-CUDA devices raise: this package has no CPU path.
"""
from __future__ import annotations

import warnings
from contextlib import contextmanager
from typing import Callable, Optional

import torch


@contextmanager
def optimize_for_training():
    """Deprecated no-op kept for API compatibility (reference kernel_selector.py:8-18)."""
    warnings.warn("`optimize_for_training` is deprecated. The optimization now happens automatically at runtime.")
    try:
        yield
    finally:
        return


def _scheme_prefix(codebooks: torch.Tensor) -> str:
    num_codebooks, codebook_size, out_group_size, in_group_size = codebooks.shape
    if codebooks.device.type != "cuda":
        raise NotImplementedError(
            f"aqlm_b200 implements the CUDA (sm_90a) hot path only; codebooks are on {codebooks.device}. "
            "Use the reference `aqlm` package for CPU inference.")
    if out_group_size != 1:
        raise NotImplementedError(f"aqlm_b200 kernels require out_group_size == 1, got {out_group_size}")
    if in_group_size not in (8, 16):
        raise NotImplementedError(
            f"AQLM CUDA kernels only support codebooks with 8 or 16 features. Got {in_group_size}.")
    if (num_codebooks, codebook_size) == (1, 65536):
        return "code1x16"  # kernel_selector.py:27-46
    if (num_codebooks, codebook_size, in_group_size) == (2, 256, 8):
        return "code2x8"  # 47-57, 69-79
    if (num_codebooks, codebook_size, in_group_size) == (1, 256, 8):
        return "code1x8"  # 58-68, 80-90
    return "generic"


def get_forward_pass_kernel(
    codebooks: torch.Tensor,
    optimize_for_training: bool,
) -> Callable[[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, Optional[torch.Tensor]], torch.Tensor]:
    """reference kernel_selector.py:21-102.  `optimize_for_training=True` selects the large-batch (GEMM) op."""
    prefix = _scheme_prefix(codebooks)
    from . import cuda_kernel  # noqa: F401  (registers the ops)

    name = f"{prefix}_matmat_dequant" if optimize_for_training else f"{prefix}_matmat"
    return getattr(torch.ops.aqlm, name)


def get_backward_pass_kernel(
    codebooks: torch.Tensor,
    optimize_for_training: bool,
) -> Callable[[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, Optional[torch.Tensor]], torch.Tensor]:
    """reference kernel_selector.py:105-163: grad w.r.t. the input, [..., out] -> [..., in]."""
    prefix = _scheme_prefix(codebooks)
    from . import cuda_kernel  # noqa: F401

    return getattr(torch.ops.aqlm, f"{prefix}_matmat_dequant_transposed")
