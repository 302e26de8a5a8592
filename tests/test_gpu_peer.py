"""Multi-GPU exchange tests: the fused GEMV + peer exchange and the stand-alone exchange kernel on 2 GPUs (skipped when fewer
are visible), and the same kernels on ONE GPU through a one-rank communicator (always runs)."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)  # only used to exchange IPC handles
    try:
        from helpers import oracle_output, to_torch

        from aqlm_b200.peer import PeerComm
        from aqlm_b200.sharded import ShardedQuantizedLinear
        from oracle import aqlm_oracle as O

        comm = PeerComm(max_elems=4 * 4096)
        errs = []
        for it, (K, nbits, batch) in enumerate([(1, 16, 1), (2, 8, 1), (1, 16, 3), (1, 16, 1)]):
            case = O.make_case(5150 + it, 2048, 512, K, nbits, 8, batch, bias=True)
            t = to_torch(case, f"cuda:{rank}")
            m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=rank,
                                                 world_size=world, peer_comm=comm)
            for fused in (True, False):  # ONE kernel (GEMV + exchange) and the two-kernel form share the step counter
                m.fused_exchange = fused
                for _ in range(3):  # repeated calls exercise the step counter / buffer-set alternation
                    y = m(t["x"])
                torch.cuda.synchronize()
                errs.append(O.relative_error(y.float().cpu().numpy(), oracle_output(case)))
        # grouped: three linears sharing x -> ONE GEMV launch + ONE fused exchange
        from aqlm_b200.grouped import ShardedQuantizedLinearGroup

        cases = [O.make_case(5300 + i, 2048, o, 1, 16, 8, 1, bias=False) for i, o in enumerate((512, 128, 128))]
        for c in cases[1:]:
            c["x"] = cases[0]["x"]
        ms = []
        for c in cases:
            t = to_torch(c, f"cuda:{rank}")
            ms.append(ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=rank,
                                                       world_size=world, peer_comm=comm))
        grp = ShardedQuantizedLinearGroup(ms)
        assert grp.fused
        x = to_torch(cases[0], f"cuda:{rank}")["x"]
        for fused in (True, False):
            for mm in ms:
                mm.fused_exchange = fused
            for _ in range(2):
                ys = grp(x)
            torch.cuda.synchronize()
            for c, y in zip(cases, ys):
                errs.append(O.relative_error(y.float().cpu().numpy(), oracle_output(c)))
        # a BASELINE configs[4] shard shape (Llama-3-70B o_proj, 8192 -> 8192) through the fused kernel, inside a CUDA graph
        from helpers import c_oracle_check, gpu_case

        t = gpu_case(8192, 8192, 1, 16, 1, seed=77, device=f"cuda:{rank}")  # same seed on every rank: identical full tensors
        m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], None, rank=rank, world_size=world,
                                             peer_comm=comm)
        y = m(t["x"])
        torch.cuda.synchronize()
        dist.barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = m(t["x"])
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        errs.append(c_oracle_check(t, y))
        ret[rank] = errs
    finally:
        dist.barrier()
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_peer_allreduce_two_gpus():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    for r in range(2):
        assert all(e < 5e-4 for e in ret[r]), (r, ret[r])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_one_process_two_devices_opt_in_shared_memory():
    """ADVICE r1: cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device; a process that drives several GPUs
    (HF device_map='auto') must configure every one of them -- kernels needing > 48 KiB must work on cuda:1 after cuda:0."""
    from helpers import c_oracle_check, gpu_case

    from aqlm_b200.inference_kernels import cuda_kernel

    for dev in ("cuda:0", "cuda:1"):
        for K, nbits, batch in ((2, 8, 1), (1, 16, 64), (1, 16, 5)):  # LUT GEMV, wgmma GEMM, batched gather GEMV
            t = gpu_case(4096, 4096, K, nbits, batch, seed=K + batch, device=dev)
            op = cuda_kernel.matmat_dequant if batch > 6 else cuda_kernel.matmat
            y = op(t["x"], t["codes"], t["codebooks"], t["scales"], None)
            torch.cuda.synchronize(dev)
            assert c_oracle_check(t, y) < 5e-4, (dev, K, nbits, batch)


def _self_exchange_worker(rank, port, ret):
    """ONE GPU, one-rank communicator: the fused GEMV + exchange kernel pushes its tagged words into its OWN buffer and
    waits for them there -- the same code path (contiguous row blocks, {fp32, step} words, set alternation, epilogue) as on
    N GPUs, minus the NVLink hop, so the driver's single-GPU box exercises it too."""
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        from helpers import c_oracle_check, gpu_case, oracle_output, to_torch

        from aqlm_b200 import _cabi
        from aqlm_b200.grouped import ShardedQuantizedLinearGroup
        from aqlm_b200.peer import PeerComm
        from aqlm_b200.sharded import ShardedQuantizedLinear
        from oracle import aqlm_oracle as O

        comm = PeerComm(max_elems=4 * 28672)
        errs = []

        def shard(t):
            m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t.get("bias"), rank=0, world_size=1,
                                                 peer_comm=comm)
            m.world_size = 2  # take the exchange path; the communicator itself has one rank
            return m

        for it, (K, nbits, batch) in enumerate([(1, 16, 1), (1, 16, 3), (2, 8, 1), (1, 16, 8)]):
            case = O.make_case(6150 + it, 2048, 520, K, nbits, 8, batch, bias=(it % 2 == 0))
            t = to_torch(case, "cuda:0")
            m = shard(t)
            for fused in (True, False):
                m.fused_exchange = fused
                before = _cabi.launch_count()
                for _ in range(3):  # odd number of steps: the two buffer sets alternate across linears as well
                    y = m(t["x"])
                torch.cuda.synchronize()
                launches = (_cabi.launch_count() - before) // 3
                if fused and (K, nbits) == (1, 16):
                    assert launches == 1, launches  # GEMV + exchange + epilogue is ONE kernel
                errs.append(O.relative_error(y.float().cpu().numpy(), oracle_output(case)))
        # grouped q/k/v-like launch through the fused kernel
        cases = [O.make_case(6300 + i, 2048, o, 1, 16, 8, 1, bias=False) for i, o in enumerate((512, 128, 128))]
        for c in cases[1:]:
            c["x"] = cases[0]["x"]
        ms = [shard(to_torch(c, "cuda:0")) for c in cases]
        grp = ShardedQuantizedLinearGroup(ms)
        x = to_torch(cases[0], "cuda:0")["x"]
        for _ in range(2):
            ys = grp(x)
        torch.cuda.synchronize()
        for c, y in zip(cases, ys):
            errs.append(O.relative_error(y.float().cpu().numpy(), oracle_output(c)))
        # a Llama-3-70B 1/8 shard shape (down_proj: 28672/8 -> 8192) in a CUDA graph, against the C oracle
        t = gpu_case(3584, 8192, 1, 16, 1, seed=78, device="cuda:0")
        m = shard(t)
        y = m(t["x"])
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = m(t["x"])
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        errs.append(c_oracle_check(t, y))
        ret[0] = errs
    finally:
        dist.destroy_process_group()


def test_fused_exchange_kernel_on_one_gpu_self_communicator():
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_self_exchange_worker, args=(port, ret), nprocs=1, join=True)
    assert len(ret[0]) == 12 and all(e < 5e-4 for e in ret[0]), ret[0]
