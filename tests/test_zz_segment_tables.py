"""Segment tables of the grouped GEMV calls: a table that describes no split of the rows -- an empty or negative segment,
even when the sum comes out right -- is ERR_SHAPE, as it is for the grouped and routed GEMMs
(test_zz_grouped_gemm.py, test_zz_routed_gemm.py).  Such a table would give the kernel non-monotonic segment ends."""
import ctypes
import os
import socket

import pytest
import torch
from test_zz_sharded_prefill import _descriptor

BAD_TABLES = [[300, -44], [256, 0]]  # for 256 rows: a negative segment that makes the sum right, an empty one


@pytest.mark.parametrize("seg", BAD_TABLES, ids=["negative", "empty"])
def test_grouped_gemv_rejects_a_bad_table_without_a_device(seg):
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    w = _descriptor()  # 1024 -> 256, 1x16, in_group 8, dummy 16-byte aligned pointers
    table = (ctypes.c_int64 * len(seg))(*seg)
    # checked before any device query, so the dummy pointers are never launched on
    assert L.aqlm_b200_matmat_grouped(ctypes.byref(w), table, len(seg), 16, 16, 1, 0, None) == _cabi.ERR_SHAPE


def _allreduce_worker(rank, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        from aqlm_b200 import _cabi
        from aqlm_b200.inference_kernels.cuda_kernel import make_weight
        from aqlm_b200.peer import PeerComm

        comm = PeerComm(max_elems=4096)
        dev = "cuda:0"
        codes = torch.zeros((256, 128, 1), dtype=torch.int16, device=dev)
        codebooks = torch.zeros((1, 65536, 1, 8), dtype=torch.float16, device=dev)
        scales = torch.ones((256,), dtype=torch.float16, device=dev)
        x = torch.zeros((1, 1024), dtype=torch.float16, device=dev)
        y = torch.zeros((1, 256), dtype=torch.float16, device=dev)
        w = make_weight(codes, codebooks, scales, None)
        L = _cabi.lib()
        rcs = []
        for seg in BAD_TABLES:
            table = (ctypes.c_int64 * len(seg))(*seg)
            rcs.append(L.aqlm_b200_matmat_allreduce(comm._comm, ctypes.byref(w), table, len(seg), x.data_ptr(),
                                                    y.data_ptr(), 1, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        ret[0] = rcs
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_fused_exchange_rejects_a_bad_table_on_a_self_communicator():
    import torch.multiprocessing as mp

    from aqlm_b200 import _cabi

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_allreduce_worker, args=(port, ret), nprocs=1, join=True)
    assert ret[0] == [_cabi.ERR_SHAPE] * len(BAD_TABLES), ret[0]
