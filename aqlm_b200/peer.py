"""Peer-memory communicator for the in_features-sharded path (one process per GPU, NVLink P2P via cudaIpc).

`PeerComm.allreduce_scale_bias(partial, scales, bias, dtype)` is the fused replacement for
`dist.all_reduce(partial); scale_bias(partial)`: ONE kernel pushes the fp32 partials into every peer's buffer,
publishes a release flag, waits for all ranks' flags, adds the W partial vectors in rank order and applies scale + bias
(`csrc/peer_allreduce.cuh`).  A batch larger than the communicator's `max_elems` runs as consecutive exchanges of whole
rows.  `torch.distributed` is used only at construction, to check that every rank has the same `max_elems` and to
exchange the 64-byte IPC handles.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch
import torch.distributed as dist

from . import _cabi
from .inference_kernels.cuda_kernel import _DTYPES, _on_device, _require_cuda, _stream_ptr, make_weight


def check_same_max_elems(sizes) -> None:
    """Raise ValueError unless every rank's communicator has the same max_elems (`sizes[r]` is rank r's)."""
    if len(set(sizes)) > 1:
        raise ValueError("PeerComm: every rank must pass the same max_elems; got "
                         + ", ".join(f"rank {r}: {v}" for r, v in enumerate(sizes)))


class PeerComm:
    def __init__(self, group=None, max_elems: int = 8 * 28672, device: Optional[torch.device] = None):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.max_elems = (int(max_elems) + 3) // 4 * 4
        # An exchange larger than max_elems runs in chunks of max_elems // out_features rows: ranks with different
        # max_elems would run different numbers of steps and wait for each other forever.  Checked before anything is
        # allocated, and every rank sees the same gathered list, so either all ranks raise or none does.
        sizes = [None] * self.world
        dist.all_gather_object(sizes, self.max_elems, group=group)
        check_same_max_elems(sizes)
        L = _cabi.lib()
        with torch.cuda.device(self.device):
            nbytes = L.aqlm_b200_comm_shared_bytes(self.world, self.max_elems)
            if nbytes == 0:
                raise ValueError(f"unsupported world size {self.world}")
            own = ctypes.c_void_p()
            handle = ctypes.create_string_buffer(64)
            _cabi.check(L.aqlm_b200_shared_alloc(nbytes, ctypes.byref(own), handle))
            handles = [None] * self.world
            dist.all_gather_object(handles, bytes(handle.raw), group=group)
            ptrs = (ctypes.c_void_p * self.world)()
            for r in range(self.world):
                if r == self.rank:
                    ptrs[r] = own
                else:
                    p = ctypes.c_void_p()
                    buf = ctypes.create_string_buffer(handles[r], 64)
                    _cabi.check(L.aqlm_b200_shared_open(buf, ctypes.byref(p)))
                    ptrs[r] = p
            comm = ctypes.c_void_p()
            _cabi.check(L.aqlm_b200_comm_create(self.rank, self.world, ptrs, self.max_elems, ctypes.byref(comm)))
            self._comm = comm
            torch.cuda.synchronize()
        dist.barrier(group=group)  # every rank has mapped every buffer before anyone pushes

    def allreduce_scale_bias(self, partial: torch.Tensor, scales: torch.Tensor, bias: Optional[torch.Tensor],
                             dtype: torch.dtype) -> torch.Tensor:
        device = _require_cuda(partial, scales, bias)
        assert partial.dtype == torch.float32 and partial.is_contiguous()
        batch, out_features = partial.shape
        out = torch.empty((batch, out_features), dtype=dtype, device=device)
        with _on_device(device):
            _cabi.check(_cabi.lib().aqlm_b200_allreduce_scale_bias(
                self._comm, partial.data_ptr(), scales.reshape(-1).data_ptr(),
                bias.data_ptr() if bias is not None else None, out.data_ptr(), batch, out_features, _DTYPES[dtype],
                _stream_ptr(device)))
        return out

    def matmat_allreduce(self, input: torch.Tensor, codes: torch.Tensor, codebooks: torch.Tensor, scales: torch.Tensor,
                         bias: Optional[torch.Tensor], seg_rows=None) -> Optional[torch.Tensor]:
        """The sharded linear as ONE kernel (1x16 / in_group 8, <= 8 rows): GEMV on this rank's shard whose epilogue does the
        exchange over peer memory and applies scale + bias (`aqlm_b200_matmat_allreduce`).  `codebooks` is the member's
        [1, 65536, 1, 8] tensor, or the [n_seg, 1, 65536, 1, 8] stack of a grouped launch with `seg_rows`.  Returns None when
        the fused kernel does not cover the case (the caller then runs GEMV + exchange as two launches)."""
        device = _require_cuda(input, codes, codebooks, scales, bias)
        cb0 = codebooks[0] if codebooks.dim() == 5 else codebooks
        n_seg = codebooks.shape[0] if codebooks.dim() == 5 else 1
        if tuple(cb0.shape) != (1, 65536, 1, 8) or input.dtype not in _DTYPES:
            return None
        flat = input.reshape(-1, input.shape[-1])
        if not flat.is_contiguous():
            flat = flat.contiguous()
        batch = flat.shape[0]
        w = make_weight(codes, cb0, scales.reshape(-1), bias)
        if batch < 1 or batch > 8 or w.out_features % 4 or batch * w.out_features > self.max_elems or \
                (w.in_features // 8 * 2) % 16 or flat.shape[1] != w.in_features:
            return None
        out = torch.empty((batch, w.out_features), dtype=input.dtype, device=device)
        seg = (ctypes.c_int64 * n_seg)(*[int(r) for r in seg_rows]) if n_seg > 1 else None
        with _on_device(device):
            _cabi.check(_cabi.lib().aqlm_b200_matmat_allreduce(self._comm, ctypes.byref(w), seg, n_seg, flat.data_ptr(),
                                                               out.data_ptr(), batch, _stream_ptr(device)))
        return out.reshape(input.shape[:-1] + (w.out_features,))
