"""in_features-sharded QuantizedLinear: one process per GPU, ONE all-reduce of the partial output vector.

New work with no reference counterpart (the reference hot path is single-GPU, SURVEY §8e); it implements
BASELINE.json configs[4]: rank r holds `codes[:, r*in_g/W:(r+1)*in_g/W, :]` (made contiguous once at load),
the full codebooks / scales / bias (replicated, <= 1 MiB), and its slice of x.  Each rank runs the fused
gather+dequant+GEMV on its slice producing UNSCALED fp32 partials [batch, out]; a single NCCL all-reduce
(sum) over NVLink/NVSwitch combines them; scale and bias are applied once after the reduce.

Host logic (slicing, collective, epilogue order) is exercised on CPU with the gloo backend in
tests/test_sharded_gloo.py, where the two compute callables are injected by the test (the oracle stands in
for the CUDA kernels there; the product defaults below are the CUDA kernels and refuse CPU tensors).
"""
from __future__ import annotations

import os
from typing import Callable, Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .inference import weights_require_grad
from .utils import get_int_dtype


def shard_bounds(num_in_groups: int, rank: int, world_size: int) -> tuple[int, int]:
    """[begin, end) in-group range of `rank`.  Requires divisibility (SURVEY §8e: 1024 and 3584 divide by 2/4/8)."""
    if num_in_groups % world_size != 0:
        raise ValueError(f"in_groups={num_in_groups} is not divisible by world_size={world_size}")
    per = num_in_groups // world_size
    return rank * per, (rank + 1) * per


def shard_codes(codes: torch.Tensor, rank: int, world_size: int) -> torch.Tensor:
    """Contiguous copy of this rank's K-slice of codes [out_g, in_g, K] (a strided view in the natural layout)."""
    b, e = shard_bounds(codes.shape[1], rank, world_size)
    return codes[:, b:e, :].contiguous()


class ShardedQuantizedLinear(nn.Module):
    def __init__(self, in_features: int, out_features: int, in_group_size: int, out_group_size: int,
                 num_codebooks: int, nbits_per_codebook: int, bias: bool = True, process_group=None,
                 rank: Optional[int] = None, world_size: Optional[int] = None, device=None, dtype=None,
                 partial_fn: Optional[Callable] = None, epilogue_fn: Optional[Callable] = None, peer_comm=None):
        super().__init__()
        self.process_group = process_group
        self.rank = dist.get_rank(process_group) if rank is None else rank
        self.world_size = dist.get_world_size(process_group) if world_size is None else world_size
        assert in_features % in_group_size == 0 and out_group_size == 1
        self.in_features, self.out_features = in_features, out_features
        self.in_group_size, self.out_group_size = in_group_size, out_group_size
        self.num_codebooks, self.nbits_per_codebook = num_codebooks, nbits_per_codebook
        num_in_groups = in_features // in_group_size
        b, e = shard_bounds(num_in_groups, self.rank, self.world_size)
        self.in_begin, self.in_end = b * in_group_size, e * in_group_size
        kw = {"device": device, "dtype": dtype}
        self.codebooks = nn.Parameter(torch.empty((num_codebooks, 2**nbits_per_codebook, 1, in_group_size), **kw),
                                      requires_grad=False)
        self.codes = nn.Parameter(torch.empty((out_features, e - b, num_codebooks), device=device,
                                              dtype=get_int_dtype(nbits_per_codebook)), requires_grad=False)
        self.scales = nn.Parameter(torch.empty((out_features, 1, 1, 1), **kw), requires_grad=False)
        if bias:
            self.bias = nn.Parameter(torch.empty(out_features, **kw), requires_grad=False)
        else:
            self.register_parameter("bias", None)
        self._partial_fn = partial_fn
        self._epilogue_fn = epilogue_fn
        # optional aqlm_b200.peer.PeerComm: the all-reduce + epilogue then run as ONE kernel over NVLink peer memory
        self.peer_comm = peer_comm
        # with a peer communicator: run GEMV + exchange + epilogue as ONE kernel when the scheme allows (1x16)
        self.fused_exchange = os.environ.get("AQLM_B200_FUSED_EXCHANGE", "1") != "0"

    @classmethod
    def from_full(cls, codes, codebooks, scales, bias, process_group=None, rank=None, world_size=None, **kw):
        """Build this rank's shard from full (replicated-on-load) tensors."""
        K, cb_size, og, g = codebooks.shape
        out_f, in_groups, _ = codes.shape
        m = cls(in_groups * g, out_f, g, og, K, int(cb_size).bit_length() - 1, bias is not None, process_group, rank,
                world_size, device=codebooks.device, dtype=codebooks.dtype, **kw)
        m.codes.data = shard_codes(codes, m.rank, m.world_size)
        m.codebooks.data = codebooks
        m.scales.data = scales
        if bias is not None:
            m.bias.data = bias
        return m

    def _compute_fns(self):
        if self._partial_fn is None or self._epilogue_fn is None:
            from .inference_kernels import cuda_kernel

            self._default_fns = self._partial_fn is None and self._epilogue_fn is None
            self._partial_fn = self._partial_fn or cuda_kernel.matmat_partial
            self._epilogue_fn = self._epilogue_fn or cuda_kernel.scale_bias
        return self._partial_fn, self._epilogue_fn

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        """`input` is either the full [..., in_features] activation or this rank's [..., in_features/W] slice."""
        if torch.is_grad_enabled() and weights_require_grad(self):
            raise NotImplementedError("the sharded path has no weight gradient: freeze codebooks, scales and bias")
        injected = self._partial_fn is not None and not getattr(self, "_default_fns", False)
        partial_fn, epilogue_fn = self._compute_fns()
        local = self.in_end - self.in_begin
        if input.shape[-1] == self.in_features and self.world_size > 1:
            input = input[..., self.in_begin:self.in_end]
        elif input.shape[-1] != local:
            raise ValueError(f"input has {input.shape[-1]} features; expected {self.in_features} or {local}")
        flat = input.reshape(-1, local)
        if self.world_size > 1 and self.peer_comm is not None and self.fused_exchange and not injected:
            # ONE kernel: GEMV + NVLink exchange + scale/bias (1x16, <= 8 rows); None when the case is not covered
            y = self.peer_comm.matmat_allreduce(flat, self.codes, self.codebooks, self.scales, self.bias)
            if y is not None:
                return y.reshape(input.shape[:-1] + (self.out_features,))
        partial = partial_fn(flat, self.codes, self.codebooks)  # [batch, out] fp32, unscaled
        if self.world_size > 1 and self.peer_comm is not None:
            out = self.peer_comm.allreduce_scale_bias(partial, self.scales, self.bias, input.dtype)  # the ONE exchange
            return out.reshape(input.shape[:-1] + (self.out_features,))
        if self.world_size > 1:
            dist.all_reduce(partial, op=dist.ReduceOp.SUM, group=self.process_group)  # the ONE collective
        out = epilogue_fn(partial, self.scales, self.bias, input.dtype)
        return out.reshape(input.shape[:-1] + (self.out_features,))
