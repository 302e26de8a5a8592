"""Mixture-of-experts blocks on the routed wgmma GEMM: `QuantizedMixtralExperts`, a drop-in for transformers'
`MixtralExperts` whose experts are AQLM-quantized.

transformers 5.x keeps all experts of a Mixtral block as two 3-D parameters (`gate_up_proj`, `down_proj`), which Hugging
Face's AQLM integration does not replace (it swaps `nn.Linear` modules only).  This module holds the checkpoint's
per-expert linears instead -- submodules `"{e}".w1 / w2 / w3` are `QuantizedLinear`, so the state-dict names are the
checkpoint's `experts.{e}.w{1,2,3}.{codes,codebooks,scales}` -- and runs them as ONE routed launch per projection over
all experts:

  * routing (PyTorch plumbing, no host sync): a stable sort of the flattened expert ids, per-expert row offsets by
    `searchsorted`, `index_select` of the token rows.  Ids outside [0, E) are dropped and contribute nothing;
  * one routed GEMM for w1|w3 (row-concatenated per expert: a 2-segment weight), `act(gate) * up`, one routed GEMM for
    w2;
  * the combine sum_j w[t, j] * y[pair(t, j)], in fp32 in slot order, rounded once to the activation dtype.

Nothing reads the routing on the host, so a decode step can be captured in a CUDA graph and replayed with new routing.
Gradients flow to `hidden_states` (one routed transposed GEMM per projection) and to `top_k_weights` (ordinary
autograd); the quantized weights are frozen.  A scheme the routed GEMM does not take (e.g. in_group 16) runs the
transformers algorithm over the member `QuantizedLinear`s: correct, but it syncs with the host and is not capturable.

The member parameters are views into stacked per-projection buffers (as `grouped._fuse_storage` does for a group); the
stacks are rebuilt whenever the module is moved or cast (`_apply`) or after a load that replaced the parameters.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch
from torch import nn

from .grouped import gemm_scheme
from .inference import QuantizedLinear, weights_require_grad


def route(top_k_index: torch.Tensor, n_experts: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Sort the (token, slot) pairs of `top_k_index` [T, k] by expert, on the device.

    Returns (order, offsets, valid): `order` [T*k] int64, the flat pair index (t * k + j) of each sorted row, pairs of
    ids outside [0, E) last; `offsets` [E + 1] int32, expert e owns sorted rows [offsets[e], offsets[e + 1]) and
    offsets[E] is the count of valid pairs; `valid` [T*k] bool, per flat pair, whether its id is in range."""
    flat = top_k_index.reshape(-1)
    valid = (flat >= 0) & (flat < n_experts)
    key = torch.where(valid, flat, torch.full_like(flat, n_experts))
    sorted_key, order = torch.sort(key, stable=True)
    bounds = torch.arange(n_experts + 1, device=flat.device, dtype=sorted_key.dtype)
    offsets = torch.searchsorted(sorted_key, bounds).to(torch.int32)
    return order, offsets, valid


class _RoutedMatmul(torch.autograd.Function):
    """Autograd node of a routed projection y = routed(x; stacked weights).  `y` is what the routed forward kernel
    computed from `x`; the backward is one routed transposed GEMM.  Rows that belong to no expert (dropped pairs, at the
    end of the sorted rows) are never written by the kernels; their input gradient is set to zero here."""

    @staticmethod
    def forward(ctx, x, y, weights, offsets, row_valid):
        ctx.weights, ctx.row_valid = weights, row_valid
        ctx.save_for_backward(offsets)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        from .inference_kernels import cuda_kernel

        (offsets,) = ctx.saved_tensors
        codes, codebooks, scales, seg_rows = ctx.weights
        gx = cuda_kernel.matmat_dequant_transposed_routed(grad_y.contiguous(), codes, codebooks, scales, offsets, seg_rows)
        if gx is None:
            raise NotImplementedError("the routed transposed GEMM refused a layout its forward took")
        return torch.where(ctx.row_valid[:, None], gx, torch.zeros((), dtype=gx.dtype, device=gx.device)), None, None, \
            None, None


class _Expert(nn.Module):
    """One expert's three linears, named as in the checkpoint (w1 gate, w3 up, w2 down)."""

    def __init__(self, hidden: int, inter: int, qargs: dict, device, dtype):
        super().__init__()
        self.w1 = QuantizedLinear(hidden, inter, bias=False, device=device, dtype=dtype, **qargs)
        self.w2 = QuantizedLinear(inter, hidden, bias=False, device=device, dtype=dtype, **qargs)
        self.w3 = QuantizedLinear(hidden, inter, bias=False, device=device, dtype=dtype, **qargs)


class QuantizedMixtralExperts(nn.Module):
    """Drop-in for `MixtralExperts`: forward(hidden_states [T, H], top_k_index [T, k], top_k_weights [T, k]) -> [T, H]."""

    def __init__(self, num_experts: int, hidden_dim: int, intermediate_dim: int, act_fn: Callable, in_group_size: int,
                 out_group_size: int, num_codebooks: int, nbits_per_codebook: int, device=None,
                 dtype: Optional[torch.dtype] = None):
        super().__init__()
        self.num_experts, self.hidden_dim, self.intermediate_dim = num_experts, hidden_dim, intermediate_dim
        self.act_fn = act_fn
        qargs = dict(in_group_size=in_group_size, out_group_size=out_group_size, num_codebooks=num_codebooks,
                     nbits_per_codebook=nbits_per_codebook)
        for e in range(num_experts):
            self.add_module(str(e), _Expert(hidden_dim, intermediate_dim, qargs, device, dtype))
        self.routed = gemm_scheme(self.expert(0).w1)
        self.fuse_storage()

    def expert(self, e: int) -> _Expert:
        return getattr(self, str(e))

    @torch.no_grad()
    def fuse_storage(self) -> None:
        """Stack the experts' tensors per projection and re-point every member parameter at its view:
        w1|w3 codes [E, 2I, H/8, K], codebooks [E, 2, K, 2^nbits, 1, 8], scales [E, 2I, 1, 1, 1]; w2 likewise with one
        segment.  Called at construction, after every move / cast and after a load that replaced the parameters."""
        ex = [self.expert(e) for e in range(self.num_experts)]
        I = self.intermediate_dim
        c13 = torch.stack([torch.cat([m.w1.codes, m.w3.codes]) for m in ex])
        b13 = torch.stack([torch.stack([m.w1.codebooks, m.w3.codebooks]) for m in ex])
        s13 = torch.stack([torch.cat([m.w1.scales, m.w3.scales]) for m in ex])
        c2 = torch.stack([m.w2.codes for m in ex])
        b2 = torch.stack([m.w2.codebooks[None] for m in ex])
        s2 = torch.stack([m.w2.scales for m in ex])
        for e, m in enumerate(ex):
            m.w1.codes.data, m.w3.codes.data = c13[e, :I], c13[e, I:]
            m.w1.codebooks.data, m.w3.codebooks.data = b13[e, 0], b13[e, 1]
            m.w1.scales.data, m.w3.scales.data = s13[e, :I], s13[e, I:]
            m.w2.codes.data, m.w2.codebooks.data, m.w2.scales.data = c2[e], b2[e, 0], s2[e]
        # plain attributes, not buffers: _apply moves the members' parameters, then re-stacks them
        self._w13 = (c13, b13, s13, [I, I])
        self._w2 = (c2, b2, s2, None)

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        self.fuse_storage()
        return self

    # -- forward ------------------------------------------------------------------------------------------------------
    def forward(self, hidden_states: torch.Tensor, top_k_index: torch.Tensor, top_k_weights: torch.Tensor) -> torch.Tensor:
        # trainable codebooks / scales: the members' own autograd nodes (no routed weight-gradient kernel)
        train_weights = torch.is_grad_enabled() and any(weights_require_grad(m) for m in self.modules()
                                                        if isinstance(m, QuantizedLinear))
        if self.routed and hidden_states.is_cuda and not train_weights:
            out = self._forward_routed(hidden_states, top_k_index, top_k_weights)
            if out is not None:
                return out
        return self._forward_loop(hidden_states, top_k_index, top_k_weights)

    def _project(self, x, weights, offsets, row_valid):
        from .inference_kernels import cuda_kernel

        codes, codebooks, scales, seg_rows = weights
        y = cuda_kernel.matmat_dequant_routed(x.detach(), codes, codebooks, scales, offsets, seg_rows)
        if y is None or not (torch.is_grad_enabled() and x.requires_grad):
            return y
        return _RoutedMatmul.apply(x, y, weights, offsets, row_valid)

    def _forward_routed(self, hidden_states, top_k_index, top_k_weights) -> Optional[torch.Tensor]:
        T, k = top_k_index.shape
        order, offsets, valid = route(top_k_index, self.num_experts)
        row_valid = valid[order]  # per sorted row: the valid pairs come first
        xs = hidden_states.index_select(0, order // k)
        gu = self._project(xs, self._w13, offsets, row_valid)
        if gu is None:
            return None
        gate, up = gu.split(self.intermediate_dim, dim=-1)
        h = self.act_fn(gate) * up
        ys = self._project(h, self._w2, offsets, row_valid)
        if ys is None:
            return None
        # back to (token, slot) order; rows of dropped pairs hold whatever the kernels left there: masked, not scaled
        pos = torch.empty_like(order)
        pos[order] = torch.arange(order.numel(), device=order.device)
        y = ys.index_select(0, pos).view(T, k, -1)
        zero = torch.zeros((), dtype=torch.float32, device=y.device)
        w = torch.where(valid.view(T, k), top_k_weights.float(), zero)
        acc = None
        for j in range(k):  # slot order, fp32, rounded once
            yj = torch.where(valid.view(T, k)[:, j, None], y[:, j].float(), zero)
            term = yj * w[:, j, None]
            acc = term if acc is None else acc + term
        return acc.to(hidden_states.dtype)

    def _forward_loop(self, hidden_states, top_k_index, top_k_weights) -> torch.Tensor:
        """transformers' MixtralExperts algorithm over the member linears (syncs with the host; not capturable)."""
        final = torch.zeros_like(hidden_states)
        with torch.no_grad():
            ids = torch.where((top_k_index >= 0) & (top_k_index < self.num_experts), top_k_index, self.num_experts)
            mask = torch.nn.functional.one_hot(ids, num_classes=self.num_experts + 1)
            mask = mask.permute(2, 1, 0)
            hit = torch.greater(mask.sum(dim=(-1, -2)), 0).nonzero()
        for e in hit:
            e = int(e[0])
            if e >= self.num_experts:
                continue
            pos, tok = torch.where(mask[e])
            m = self.expert(e)
            x = hidden_states[tok]
            h = m.w2(self.act_fn(m.w1(x)) * m.w3(x))
            h = h * top_k_weights[tok, pos, None]
            final.index_add_(0, tok, h.to(final.dtype))
        return final

    def extra_repr(self) -> str:
        m = self.expert(0).w1
        return (f"num_experts={self.num_experts}, hidden={self.hidden_dim}, intermediate={self.intermediate_dim}, "
                f"scheme={m.num_codebooks}x{m.nbits_per_codebook}, in_group_size={m.in_group_size}, routed={self.routed}")
