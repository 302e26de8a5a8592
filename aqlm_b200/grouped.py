"""Grouped launch for quantized linears that share their input (q/k/v, gate/up): one kernel instead of n.

New work (SURVEY §8f.2; the reference launches every linear on its own).  `QuantizedLinearGroup` fuses the STORAGE of its
members — codes and scales (and biases) are concatenated along the output dimension, the 1 MiB codebooks are stacked — and
re-points every member's parameters at views of the fused buffers, so the members keep working on their own and
`state_dict()` (names, shapes, dtypes) is unchanged.  `forward(x)` returns one output per member.

Which launch serves a call:
  * up to 8 rows of a 1x16 / in_group 8 group: the grouped GEMV (one launch);
  * more rows, or an input that needs a gradient, for every scheme the wgmma GEMM covers (in_group 8, 8/16-bit codes,
    1/2/4/8 codebooks): the grouped GEMM over the row-concatenated weight (one launch), and for the gradient w.r.t. the
    input one grouped transposed GEMM (`_GroupedMatmul`);
  * anything else -- up to 8 rows of other schemes, or a layout the library refuses -- the members one by one;
  * so do calls that need a gradient w.r.t. a member's codebooks, scales or bias (no grouped weight-gradient kernel).
"""
from __future__ import annotations

from typing import Sequence, Tuple

import torch
import torch.nn as nn

from .inference import QuantizedLinear, weights_require_grad
from .sharded import ShardedQuantizedLinear


def _fuse_storage(members) -> dict:
    with torch.no_grad():
        codes = torch.cat([m.codes.data for m in members], dim=0).contiguous()
        codebooks = torch.stack([m.codebooks.data for m in members], dim=0).contiguous()
        scales = torch.cat([m.scales.data for m in members], dim=0).contiguous()
        bias = None
        if members[0].bias is not None:
            bias = torch.cat([m.bias.data for m in members], dim=0).contiguous()
        off = 0
        for i, m in enumerate(members):
            n = m.codes.shape[0]
            m.codes.data = codes[off:off + n]
            m.codebooks.data = codebooks[i]
            m.scales.data = scales[off:off + n]
            if bias is not None:
                m.bias.data = bias[off:off + n]
            off += n
    return dict(codes=codes, codebooks=codebooks, scales=scales, bias=bias)


def gemm_scheme(m) -> bool:
    """The schemes the grouped wgmma GEMM takes: in_group 8, 8- or 16-bit codes, 1/2/4/8 codebooks."""
    return m.in_group_size == 8 and m.out_group_size == 1 and m.nbits_per_codebook in (8, 16) and \
        m.num_codebooks in (1, 2, 4, 8)


def _gemv_scheme(m) -> bool:
    """The scheme the grouped GEMV takes (up to 8 rows): 1x16, in_group 8."""
    return (m.num_codebooks, m.nbits_per_codebook, m.in_group_size, m.out_group_size) == (1, 16, 8, 1)


def _rows(x: torch.Tensor) -> int:
    rows = 1
    for d in x.shape[:-1]:
        rows *= d
    return rows


def _check_members(members) -> bool:
    """True when the storage is fused (a grouped kernel applies); raises on members that cannot be grouped at all."""
    m0 = members[0]
    for m in members:
        if m.in_features != m0.in_features or m.codebooks.dtype != m0.codebooks.dtype or \
                m.codes.device != m0.codes.device or (m.bias is None) != (m0.bias is None) or \
                (m.num_codebooks, m.nbits_per_codebook, m.in_group_size) != \
                (m0.num_codebooks, m0.nbits_per_codebook, m0.in_group_size):
            raise ValueError("grouped linears must share in_features, scheme, dtype, device and bias-ness")
    return gemm_scheme(m0) and len(members) <= 4 and m0.codes.is_cuda


class _GroupedMatmul(torch.autograd.Function):
    """Autograd node of a group's concatenated output y = [x W_1^T | x W_2^T | ...] (+ scales, bias).  `y` is what the
    group's forward kernel computed from `x` (the group has to know that the kernel took the layout before it builds this
    node).  Only `x` receives a gradient, as in `_AqlmMatmul`: ONE grouped transposed GEMM over the concatenated weight,
    or, for a layout it does not take, the members' own backward ops, summed."""

    @staticmethod
    def forward(ctx, x, y, group):
        ctx.group = group
        return y

    @staticmethod
    def backward(ctx, grad_y):
        from .inference_kernels import cuda_kernel

        g = ctx.group
        gx = cuda_kernel.matmat_dequant_transposed_grouped(grad_y, g._fused_codes, g._fused_codebooks, g._fused_scales,
                                                           g.seg_rows)
        if gx is None:
            from .inference_kernels import get_backward_pass_kernel

            gx, off = None, 0
            for m in g.members:
                n = m.out_features
                d = get_backward_pass_kernel(m.codebooks, True)(grad_y[..., off:off + n].contiguous(), m.codes,
                                                                m.codebooks, m.scales, m.bias)
                gx = d if gx is None else gx + d
                off += n
        return gx, None, None


class QuantizedLinearGroup(nn.Module):
    def __init__(self, members: Sequence[QuantizedLinear]):
        super().__init__()
        self.members = nn.ModuleList(members)
        self.fused = _check_members(list(members))
        self.seg_rows = [m.out_features for m in members]
        if self.fused:
            for k, v in _fuse_storage(list(members)).items():
                if v is not None:
                    self.register_buffer(f"_fused_{k}", v, persistent=False)
            if members[0].bias is None:
                self._fused_bias = None

    def forward(self, input: torch.Tensor) -> Tuple[torch.Tensor, ...]:
        rows = _rows(input)
        # a gradient w.r.t. the input (LoRA / PEFT on frozen AQLM weights) goes through the grouped GEMM and its autograd
        # node at any batch
        needs_grad = torch.is_grad_enabled() and input.requires_grad
        if not self.fused or not input.is_cuda or rows < 1:
            return tuple(m(input) for m in self.members)
        if torch.is_grad_enabled() and any(weights_require_grad(m) for m in self.members):
            # trainable codebooks / scales / bias: each member's own autograd node computes its weight gradients, which
            # land on the member parameters (views into the fused storage)
            return tuple(m(input) for m in self.members)
        from .inference_kernels import cuda_kernel

        if rows <= 8 and _gemv_scheme(self.members[0]):
            try:
                y = cuda_kernel.matmat_grouped(input.detach(), self._fused_codes, self._fused_codebooks,
                                               self._fused_scales, self._fused_bias, self.seg_rows)
            except NotImplementedError:
                # a layout the grouped GEMV refuses (e.g. an input that is not 16-byte aligned): without a gradient this
                # raises, as it always has; with one, the members take it, as they did before the group had a backward
                if not needs_grad:
                    raise
                y = None
        elif rows > 8 or needs_grad:
            y = cuda_kernel.matmat_dequant_grouped(input.detach(), self._fused_codes, self._fused_codebooks,
                                                   self._fused_scales, self._fused_bias, self.seg_rows)
        else:
            y = None  # up to 8 rows of a scheme the grouped GEMV does not take: the members' GEMV / LUT kernels
        if y is None:
            return tuple(m(input) for m in self.members)
        if needs_grad:
            y = _GroupedMatmul.apply(input, y, self)
        return tuple(torch.split(y, self.seg_rows, dim=-1))


class ShardedQuantizedLinearGroup(nn.Module):
    """Same for the in_features-sharded path: ONE GEMV (up to 8 rows) or grouped GEMM (prefill) launch and ONE exchange
    for the whole group.  A gradient w.r.t. the input goes through the members."""

    def __init__(self, members: Sequence[ShardedQuantizedLinear]):
        super().__init__()
        self.members = nn.ModuleList(members)
        self.fused = _check_members(list(members))
        self.seg_rows = [m.out_features for m in members]
        m0 = members[0]
        self.world_size, self.process_group, self.peer_comm = m0.world_size, m0.process_group, m0.peer_comm
        self.in_begin, self.in_end, self.in_features = m0.in_begin, m0.in_end, m0.in_features
        if self.fused:
            for k, v in _fuse_storage(list(members)).items():
                if v is not None:
                    self.register_buffer(f"_fused_{k}", v, persistent=False)
            if m0.bias is None:
                self._fused_bias = None

    def forward(self, input: torch.Tensor) -> Tuple[torch.Tensor, ...]:
        if torch.is_grad_enabled() and any(weights_require_grad(m) for m in self.members):
            raise NotImplementedError("the sharded path has no weight gradient: freeze codebooks, scales and bias")
        local = self.in_end - self.in_begin
        if input.shape[-1] == self.in_features and self.world_size > 1:
            input = input[..., self.in_begin:self.in_end]
        rows = _rows(input)
        if not self.fused or not input.is_cuda or rows < 1 or (torch.is_grad_enabled() and input.requires_grad):
            return tuple(m(input) for m in self.members)
        import torch.distributed as dist

        from .inference_kernels import cuda_kernel

        flat = input.reshape(-1, local)
        if rows <= 8:
            if not _gemv_scheme(self.members[0]):
                return tuple(m(input) for m in self.members)
            if self.world_size > 1 and self.peer_comm is not None and getattr(self.members[0], "fused_exchange", True):
                # ONE kernel for the whole group: grouped GEMV + NVLink exchange + scale/bias
                y = self.peer_comm.matmat_allreduce(flat, self._fused_codes, self._fused_codebooks, self._fused_scales,
                                                    self._fused_bias, self.seg_rows)
                if y is not None:
                    y = y.reshape(input.shape[:-1] + (sum(self.seg_rows),))
                    return tuple(torch.split(y, self.seg_rows, dim=-1))
            partial = cuda_kernel.matmat_grouped(flat, self._fused_codes, self._fused_codebooks, None, None,
                                                 self.seg_rows, partial=True)
        else:
            # prefill: the group's fp32 partials in ONE grouped GEMM, then the same single exchange as above
            partial = cuda_kernel.matmat_dequant_grouped(flat, self._fused_codes, self._fused_codebooks, None, None,
                                                         self.seg_rows, partial=True)
            if partial is None:
                return tuple(m(input) for m in self.members)
        if self.world_size > 1 and self.peer_comm is not None:
            y = self.peer_comm.allreduce_scale_bias(partial, self._fused_scales, self._fused_bias, input.dtype)
        else:
            if self.world_size > 1:
                dist.all_reduce(partial, op=dist.ReduceOp.SUM, group=self.process_group)
            y = cuda_kernel.scale_bias(partial, self._fused_scales, self._fused_bias, input.dtype)
        y = y.reshape(input.shape[:-1] + (sum(self.seg_rows),))
        return tuple(torch.split(y, self.seg_rows, dim=-1))
