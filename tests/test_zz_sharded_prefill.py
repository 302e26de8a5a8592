"""The in_features-sharded path at prefill batch sizes: fp32 partials from the wgmma GEMM and exchanges of any batch.

Partials are checked bit-exactly on the integer lattice of test_zz_gemm_exact.py: without scales every partial is an
integer well inside fp32's significand, so it does not depend on tile shape, split count or summation order.  Runs
after test_zz_gemm_exact.py (`zz`): the forced-plan cases set AQLM_B200_* switches and restore them on the way out.
"""
import ctypes
import math
import os
import socket

import numpy as np
import pytest
import torch
from helpers import TOL_NORTH_STAR, make_module, to_torch
from test_zz_gemm_exact import (DEV, DT_ID, DTYPES, GEMM_SCHEMES, WS_COUNTERS, _assert_tickets_clean, assert_exact,
                                exact_forward, expected_ws, lattice_case, n_tile_of, round_to, seed_of, tunables)

from oracle import aqlm_oracle as O

gpu = pytest.mark.gpu

PARTIAL_SHAPE = (1152, 456)  # 18 k-blocks; out % 8 != 0 and not a multiple of any tile height
PARTIAL_BATCHES = [7, 9, 64, 300]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _descriptor(**kw):
    """A weight descriptor with dummy, never dereferenced device pointers."""
    from aqlm_b200 import _cabi

    w = _cabi.Weight()
    w.codes, w.codebooks, w.scales = 16, 16, 16
    w.in_features, w.out_features = 1024, 256
    w.num_codebooks, w.nbits_per_codebook, w.in_group_size, w.out_group_size = 1, 16, 8, 1
    w.dtype = _cabi.F16
    for k, v in kw.items():
        setattr(w, k, v)
    return w


def _exact_partial(c, x=None):
    return O.dequantize_gemm(c["x"] if x is None else x, c["codes"], c["codebooks"], None, None, dtype=np.float64)


# ==== CPU ============================================================================================================
def test_dequant_ex_argument_checks_without_a_device():
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    P = _cabi.FLAG_PARTIAL_F32
    w = _descriptor()
    for flags in (0, P):
        assert L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), None, 16, 64, flags, None, 0, None) == _cabi.ERR_SHAPE
        assert L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), 16, None, 64, flags, None, 0, None) == _cabi.ERR_SHAPE
    w.scales = None
    assert L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), 16, 16, 64, 0, None, 0, None) == _cabi.ERR_SHAPE
    assert b"scales" in L.aqlm_b200_last_error()
    assert L.aqlm_b200_matmat_dequant_ws(ctypes.byref(w), 16, 16, 64, None, 0, None) == _cabi.ERR_SHAPE
    if torch.cuda.is_available():
        return  # the call below would launch on the dummy pointers
    # without scales the flagged call passes validation and fails only where it needs the device
    rc = L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), 16, 16, 64, P, None, 0, None)
    assert rc in (_cabi.ERR_CUDA, _cabi.ERR_ARCH), rc
    assert L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), 64) == 0


def test_same_max_elems_check():
    from aqlm_b200.peer import check_same_max_elems

    check_same_max_elems([1024])
    check_same_max_elems([1024, 1024, 1024])
    with pytest.raises(ValueError, match="rank 1: 2048"):
        check_same_max_elems([1024, 2048])


def _max_elems_worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from aqlm_b200.peer import PeerComm

        try:
            PeerComm(max_elems=1024 * (rank + 1), device=torch.device("cuda", rank))
            ret[rank] = "constructed"
        except ValueError as e:
            ret[rank] = f"ValueError: {e}"
    finally:
        dist.destroy_process_group()


def test_peer_comm_rejects_different_max_elems_gloo():
    """Every rank raises, before allocating anything: the check is the first thing the constructor does after the
    (CPU-only) gather, so this runs without a GPU."""
    import torch.multiprocessing as mp

    ret = mp.Manager().dict()
    mp.spawn(_max_elems_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    for r in range(2):
        assert ret[r].startswith("ValueError") and "rank 0: 1024, rank 1: 2048" in ret[r], ret[r]


# ==== GPU: fp32 partials from the forward wgmma GEMM =================================================================
def _run_partial(t, batch):
    """cuda_kernel.matmat_partial; returns (partials as numpy, workspace bytes the plan asked for, kernel launches)."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], None, None)
    need = _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), batch)
    w_scaled = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), None)
    assert need == _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w_scaled), batch)
    before = _cabi.launch_count()
    p = cuda_kernel.matmat_partial(t["x"], t["codes"], t["codebooks"])
    launches = _cabi.launch_count() - before
    assert p.dtype == torch.float32 and p.shape == (batch, w.out_features)
    if need:
        _assert_tickets_clean("partial")
    return p.cpu().numpy(), need, launches


def _partial_cases():
    return [pytest.param(K, nbits, dtype, batch, id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}")
            for K, nbits in GEMM_SCHEMES for dtype in DTYPES for batch in PARTIAL_BATCHES]


@gpu
@pytest.mark.parametrize("K,nbits,dtype,batch", _partial_cases())
def test_partial_gemm_exact(K, nbits, dtype, batch):
    fin, fout = PARTIAL_SHAPE
    c = lattice_case(seed_of("partial-gemm", K, nbits, batch), fin, fout, K, nbits, batch=batch, bias=False, dtype=dtype)
    p, need, launches = _run_partial(to_torch(c, DEV, dtype), batch)
    assert launches == 1, "the partial product above 6 rows is one wgmma GEMM launch"
    assert_exact(p, _exact_partial(c), f"partial {K}x{nbits} {fin}->{fout} bs={batch}", n_tile=n_tile_of(batch))


FORCED = [(1, 16, 128, 2, 9), (1, 16, 97, 3, 64), (1, 16, 64, 16, 300), (8, 8, 40, 3, 7), (8, 8, 127, 16, 64),
          (2, 16, 65, 5, 300), (2, 16, None, 3, 64), (1, 8, 32, 16, 9)]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits,tile_m,ksplit,batch", FORCED,
                         ids=[f"{k}x{n}-tm{tm}-ks{ks}-bs{b}" for k, n, tm, ks, b in FORCED])
def test_partial_forced_plan_exact(K, nbits, tile_m, ksplit, batch, dtype):
    """Forced tile height and split count (seen in the workspace the plan asks for); the split-K fix-up writes the
    fp32 sums and leaves its ticket words at zero."""
    fin, fout = PARTIAL_SHAPE
    c = lattice_case(seed_of("partial-forced", K, nbits, tile_m, ksplit, batch), fin, fout, K, nbits, batch=batch,
                     bias=False, dtype=dtype)
    with tunables(gemm_tile_m=tile_m, gemm_ksplit=ksplit):
        p, need, launches = _run_partial(to_torch(c, DEV, dtype), batch)
    assert launches == 1
    ks = min(ksplit, fin // 64)
    if tile_m is not None:
        assert need == expected_ws(math.ceil(fout / tile_m), batch, ks), (need, tile_m, ks)
    else:
        per_tile_split = math.ceil(batch / n_tile_of(batch)) * n_tile_of(batch) * 128 * 4
        m_tiles, rem = divmod(need - WS_COUNTERS, ks * per_tile_split)
        assert rem == 0 and math.ceil(fout / 128) <= m_tiles <= math.ceil(fout / 32), (need, ks)
    assert_exact(p, _exact_partial(c), f"partial {K}x{nbits} bs={batch} tile_m={tile_m} ksplit={ksplit}", tile_m=tile_m,
                 n_tile=n_tile_of(batch))


@gpu
@pytest.mark.parametrize("K,nbits,g,fin", [(1, 16, 16, 1024), (1, 16, 8, 1096), (2, 8, 8, 1096)],
                         ids=["1x16-g16", "1x16-in1096", "2x8-in1096"])
@pytest.mark.parametrize("batch", [9, 64, 300])
def test_partial_gemv_fallback_exact(K, nbits, g, fin, batch):
    """Layouts the wgmma GEMM does not take (in_group 16, in_features % 64 != 0) run GEMV passes of 8 rows."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    fout = 200
    c = lattice_case(seed_of("partial-fallback", K, nbits, g, fin, batch), fin, fout, K, nbits, g, batch=batch, bias=False)
    t = to_torch(c, DEV)
    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], None, None)
    assert _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), batch) == 0
    before = _cabi.launch_count()
    p = cuda_kernel.matmat_partial(t["x"], t["codes"], t["codebooks"])
    assert _cabi.launch_count() - before == math.ceil(batch / 8)
    assert_exact(p.cpu().numpy(), _exact_partial(c), f"GEMV partial {K}x{nbits} g={g} in={fin} bs={batch}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("batch", [64, 300])
def test_shard_partials_plus_scale_bias_exact(dtype, batch):
    from aqlm_b200.inference_kernels import cuda_kernel

    c = lattice_case(seed_of("prefill-shards", batch), 2048, 192, 1, 16, batch=batch, dtype=dtype)
    t = to_torch(c, DEV, dtype)
    parts = 0
    for r in range(4):
        parts = parts + cuda_kernel.matmat_partial(t["x"][:, r * 512:(r + 1) * 512].contiguous(),
                                                   t["codes"][:, r * 64:(r + 1) * 64].contiguous(), t["codebooks"])
    y = cuda_kernel.scale_bias(parts, t["scales"], t["bias"], dtype)
    assert_exact(y.float().cpu().numpy(), round_to(exact_forward(c), dtype), f"4 shards + scale_bias bs={batch}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_sharded_module_world1_prefill_exact(dtype):
    """One GEMM launch for the partials and one for scale + bias."""
    from aqlm_b200 import _cabi
    from aqlm_b200.sharded import ShardedQuantizedLinear

    batch = 64
    c = lattice_case(seed_of("sharded-w1", dtype), 2048, 456, 1, 16, batch=batch, dtype=dtype)
    t = to_torch(c, DEV, dtype)
    m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=0, world_size=1)
    with torch.no_grad():
        m(t["x"])
        torch.cuda.synchronize()
        before = _cabi.launch_count()
        y = m(t["x"])
    assert _cabi.launch_count() - before == 2
    assert_exact(y.float().cpu().numpy(), round_to(exact_forward(c), dtype), f"sharded world 1 bs={batch}")


# ==== GPU: chunked exchange through a one-rank communicator ===========================================================
def _chunked_exchange_worker(rank, port, ret):
    """ONE GPU, one-rank communicator whose max_elems holds 5 rows: every chunk is a real exchange (push into its own
    buffer, flag, wait, sum, epilogue), so this checks the chunking on a single GPU."""
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        from aqlm_b200 import _cabi
        from aqlm_b200.inference_kernels import cuda_kernel
        from aqlm_b200.peer import PeerComm
        from aqlm_b200.sharded import ShardedQuantizedLinear

        fin, fout, batch = 2048, 200, 64
        comm = PeerComm(max_elems=5 * fout + 8)
        chunks = math.ceil(batch / (comm.max_elems // fout))
        assert chunks == 13 and batch * fout > comm.max_elems
        for dtype in DTYPES:
            c = lattice_case(seed_of("chunked", dtype), fin, fout, 1, 16, batch=batch, dtype=dtype)
            t = to_torch(c, DEV, dtype)
            ref = round_to(exact_forward(c), dtype)
            # the stand-alone exchange: one launch per chunk
            parts = cuda_kernel.matmat_partial(t["x"], t["codes"], t["codebooks"])
            torch.cuda.synchronize()
            before = _cabi.launch_count()
            y = comm.allreduce_scale_bias(parts, t["scales"], t["bias"], dtype)
            torch.cuda.synchronize()
            assert _cabi.launch_count() - before == chunks
            assert_exact(y.float().cpu().numpy(), ref, f"chunked exchange {DT_ID[dtype]}")
            # the module: one GEMM launch + the chunked exchange, eagerly and replayed from a CUDA graph
            m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=0,
                                                 world_size=1, peer_comm=comm)
            m.world_size = 2  # take the exchange path; the communicator itself has one rank
            with torch.no_grad():
                before = _cabi.launch_count()
                y = m(t["x"])
                torch.cuda.synchronize()
                assert _cabi.launch_count() - before == 1 + chunks
                assert_exact(y.float().cpu().numpy(), ref, f"sharded module, chunked exchange {DT_ID[dtype]}")
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    yg = m(t["x"])
                for _ in range(3):
                    yg.fill_(float("nan"))
                    g.replay()
                    torch.cuda.synchronize()
                    assert_exact(yg.float().cpu().numpy(), ref, f"graph replay, chunked exchange {DT_ID[dtype]}")
        ret[0] = "ok"
    except BaseException as e:  # pytest.fail raises a BaseException: report it through `ret`
        ret[0] = f"{type(e).__name__}: {e}"
    finally:
        dist.destroy_process_group()


@gpu
def test_chunked_exchange_one_gpu_self_communicator():
    import torch.multiprocessing as mp

    ret = mp.Manager().dict()
    mp.spawn(_chunked_exchange_worker, args=(_free_port(), ret), nprocs=1, join=True)
    assert ret[0] == "ok", ret[0]


# ==== GPU: two ranks ==================================================================================================
def _two_gpu_worker(rank, world, port, ret):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)  # only used to exchange IPC handles
    try:
        from aqlm_b200.grouped import ShardedQuantizedLinearGroup
        from aqlm_b200.peer import PeerComm
        from aqlm_b200.sharded import ShardedQuantizedLinear

        dev, batch = f"cuda:{rank}", 64
        comm = PeerComm(max_elems=4 * 4096)  # batch 64 x 512 outputs: two exchanges
        errs = []

        def check(case, y):
            layer, t = make_module(case, dev)
            with torch.no_grad():
                ref = layer(t["x"]).float().cpu().numpy()
            errs.append(O.relative_error(y.float().cpu().numpy(), ref))

        case = O.make_case(8150, 2048, 512, 1, 16, 8, batch, bias=True)
        t = to_torch(case, dev)
        m = ShardedQuantizedLinear.from_full(t["codes"], t["codebooks"], t["scales"], t["bias"], rank=rank,
                                             world_size=world, peer_comm=comm)
        with torch.no_grad():
            for _ in range(3):
                y = m(t["x"])
        torch.cuda.synchronize()
        check(case, y)
        # q/k/v-like group: above 8 rows each member runs its own GEMM + exchange
        cases = [O.make_case(8300 + i, 2048, o, 1, 16, 8, batch, bias=False) for i, o in enumerate((512, 128, 128))]
        for cc in cases[1:]:
            cc["x"] = cases[0]["x"]
        ms = []
        for cc in cases:
            tt = to_torch(cc, dev)
            ms.append(ShardedQuantizedLinear.from_full(tt["codes"], tt["codebooks"], tt["scales"], None, rank=rank,
                                                       world_size=world, peer_comm=comm))
        grp = ShardedQuantizedLinearGroup(ms)
        with torch.no_grad():
            ys = grp(to_torch(cases[0], dev)["x"])
        torch.cuda.synchronize()
        for cc, y in zip(cases, ys):
            check(cc, y)
        ret[rank] = errs
    finally:
        dist.barrier()
        dist.destroy_process_group()


@gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_prefill_two_gpus():
    import torch.multiprocessing as mp

    ret = mp.Manager().dict()
    mp.spawn(_two_gpu_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    for r in range(2):
        assert len(ret[r]) == 4 and all(e < TOL_NORTH_STAR for e in ret[r]), (r, ret[r])
