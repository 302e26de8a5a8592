"""Format utilities of the `aqlm` package surface (reference inference_lib/src/aqlm/utils.py).

`get_int_dtype` / `pack_int_data` / `unpack_int_data` are the integer-code contract (utils.py:11-31) and are
device-agnostic bookkeeping.  `_dequantize_weight` (utils.py:43-70) is compute: here it runs the CUDA dequant
kernel and refuses CPU tensors (no CPU fallback in the product; the CPU restatement lives in oracle/).
"""
from __future__ import annotations

from typing import Optional

import torch


def get_int_dtype(nbits: int) -> torch.dtype:
    """reference utils.py:11-20"""
    if nbits <= 8:
        return torch.int8
    if nbits <= 16:
        return torch.int16
    if nbits <= 32:
        return torch.int32
    if nbits <= 64:
        return torch.int64
    raise ValueError(f"No dtype available for {nbits}-bit codebooks")


@torch.inference_mode()
def pack_int_data(data: torch.Tensor, nbits: int) -> torch.Tensor:
    """reference utils.py:23-26 -- like the reference, wraps values >= 2^(nbits-1) IN PLACE, then casts."""
    data[data >= 2 ** (nbits - 1)] -= 2**nbits
    return data.to(get_int_dtype(nbits))


@torch.inference_mode()
def unpack_int_data(data: torch.Tensor, nbits: int) -> torch.Tensor:
    """reference utils.py:29-31"""
    return data.to(torch.int64) % (2**nbits)


def _dequantize_weight(codes: torch.Tensor, codebooks: torch.Tensor,
                       scales: Optional[torch.Tensor] = None) -> torch.Tensor:
    """reference utils.py:43-70, CUDA only.

    codes [num_out_groups, num_in_groups, num_codebooks] UNSIGNED code values (any int dtype, as returned by
    `unpack_int_data`) or already-packed int8/int16 storage; codebooks [K, 2^nbits, 1, in_group_size] fp16/bf16;
    scales broadcastable [num_out_groups,1,1,1] or None.  Returns W [out_features, in_features].
    """
    from .inference_kernels import cuda_kernel

    if not codebooks.is_cuda:
        raise NotImplementedError(
            "aqlm_b200._dequantize_weight runs on CUDA (sm_90a) only; there is no CPU fallback in this package")
    nbits = codebooks.shape[1].bit_length() - 1
    storage = get_int_dtype(nbits)
    if codes.dtype != storage:
        codes = pack_int_data(codes.clone(), nbits)
    return cuda_kernel.dequant(codes, codebooks, scales)
