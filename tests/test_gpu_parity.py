"""GPU parity tests: the CUDA path (through the C-ABI) vs the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): mean|y - y_ref| / mean|y_ref| <= 1e-3 for fp16 (the reference's own metric,
benchmark/matmul_benchmark.py:108).  We additionally hold the fp16 path to 5e-4 and check the committed golden
vectors produced by the reference itself.
"""
import ctypes

import numpy as np
import pytest
import torch
from conftest import case_from_meta, golden_cases
from helpers import (TOL_BF16, TOL_FP16_TIGHT, TOL_NORTH_STAR, c_oracle_check, gpu_case, make_module, oracle_output,
                     to_torch)

from oracle import aqlm_oracle as O

pytestmark = pytest.mark.gpu

CASES = golden_cases()
IDS = [c["name"] for c in CASES]
DEV = "cuda:0"


def test_extension_is_loaded_and_device_is_h100():
    from aqlm_b200 import _cabi

    assert _cabi.lib().aqlm_b200_version() == 100
    assert torch.cuda.get_device_capability(0) == (9, 0)
    with open("/proc/self/maps") as f:
        assert "libaqlm_b200.so" in f.read()


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_module_forward_matches_golden_reference_outputs(c, golden):
    """QuantizedLinear.forward on CUDA vs the reference's own outputs (tests/golden, generated from the reference)."""
    data, _ = golden
    case = case_from_meta(c)
    layer, t = make_module(case, DEV)
    before = aqlm_launches()
    y = layer(t["x"]).float().cpu().numpy()
    assert aqlm_launches() > before, "no aqlm_b200 kernel was launched"
    ref32 = data[f"{c['name']}/y_dequantize_gemm_fp32"]
    ref_mod = data[f"{c['name']}/y_module_cpu_fp32"]
    assert y.shape == ref32.shape
    assert O.relative_error(y, ref32) < TOL_FP16_TIGHT
    assert O.relative_error(y, ref_mod) < TOL_FP16_TIGHT
    assert O.relative_error(y, ref32) < TOL_NORTH_STAR
    # no single output may be off by more than a few fp16 ulps of the output scale
    assert np.max(np.abs(y - ref32)) <= 4e-3 * np.max(np.abs(ref32)) + 1e-3


def aqlm_launches():
    from aqlm_b200 import _cabi

    return _cabi.launch_count()


@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_gemm_op_matches_oracle(c):
    """The large-batch op (`*_matmat_dequant`) must agree with the oracle at every batch size too."""
    from aqlm_b200.inference_kernels import get_forward_pass_kernel

    case = case_from_meta(c)
    t = to_torch(case, DEV)
    op = get_forward_pass_kernel(t["codebooks"], True)
    y = op(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT


@pytest.mark.parametrize("c", [c for c in CASES if c["in_features"] <= 1100], ids=lambda c: c["name"])
def test_dequant_matches_oracle_weight(c):
    from aqlm_b200.inference_kernels import cuda_kernel

    case = case_from_meta(c)
    t = to_torch(case, DEV)
    W = cuda_kernel.dequant(t["codes"], t["codebooks"], t["scales"]).float().cpu().numpy()
    Wref = O.dequantize_weight(O.unpack_int_data(case["codes"], c["nbits"]), case["codebooks"], case["scales"])
    assert W.shape == Wref.shape
    # one rounding of an fp32 value to fp16: relative error <= 2^-11
    np.testing.assert_allclose(W, Wref, rtol=2.0**-10, atol=1e-6)
    Wu = cuda_kernel.dequant(t["codes"], t["codebooks"], None).float().cpu().numpy()
    Wuref = O.dequantize_weight(O.unpack_int_data(case["codes"], c["nbits"]), case["codebooks"], None)
    np.testing.assert_allclose(Wu, Wuref, rtol=2.0**-10, atol=1e-6)
    if c["num_codebooks"] == 1:  # a single codebook vector is copied, not recomputed: bit-exact
        np.testing.assert_array_equal(Wu, Wuref)


SCHEMES = [(1, 16, 8), (1, 16, 16), (2, 8, 8), (1, 8, 8), (8, 8, 8), (4, 8, 8), (2, 12, 8), (3, 8, 8)]


@pytest.mark.parametrize("K,nbits,g", SCHEMES)
@pytest.mark.parametrize("batch", [1, 2, 3, 6, 8, 11])
def test_all_schemes_and_batches(K, nbits, g, batch):
    case = O.make_case(7000 + K * 100 + nbits + batch, 1024, 200, K, nbits, g, batch, bias=(batch % 2 == 0))
    layer, t = make_module(case, DEV)
    y = layer(t["x"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT


@pytest.mark.parametrize("K,nbits,g", [(1, 16, 8), (2, 8, 8), (8, 8, 8)])
def test_bf16_against_bf16_fed_oracle(K, nbits, g):
    case = O.make_case(7100 + K, 2048, 256, K, nbits, g, 2, bias=True)
    layer, t = make_module(case, DEV, torch.bfloat16)
    y = layer(t["x"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case, torch.bfloat16)) < TOL_BF16


@pytest.mark.parametrize("fin,fout", [(8, 1), (8, 7), (64, 3), (136, 33), (4096, 5), (14336, 16), (1032, 40)])
def test_edge_shapes_1x16(fin, fout):
    """Tiny, ragged (row bytes not a multiple of 16) and long-row shapes."""
    case = O.make_case(7200 + fin + fout, fin, fout, 1, 16, 8, 1, False)
    layer, t = make_module(case, DEV)
    y = layer(t["x"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT


def test_leading_dims_and_noncontiguous_input():
    case = O.make_case(7300, 512, 64, 2, 8, 8, 6, True)
    layer, t = make_module(case, DEV)
    ref = oracle_output(case)
    y = layer(t["x"].reshape(2, 3, 512))
    assert y.shape == (2, 3, 64)
    assert O.relative_error(y.reshape(6, 64).float().cpu().numpy(), ref) < TOL_FP16_TIGHT
    xt = t["x"].t().contiguous().t()  # same values, non-contiguous strides
    assert not xt.is_contiguous()
    assert O.relative_error(layer(xt).float().cpu().numpy(), ref) < TOL_FP16_TIGHT


def test_empty_batch():
    case = O.make_case(7301, 256, 32, 1, 16, 8, 1, False)
    layer, t = make_module(case, DEV)
    y = layer(t["x"][:0])
    assert y.shape == (0, 32)


def test_signed_storage_codes_are_not_sign_extended():
    """Codes >= 2^(nbits-1) are stored negative (utils.py:23-26); all-0xFFFF must index the LAST codebook entry."""
    case = O.make_case(7302, 256, 16, 1, 16, 8, 1, False)
    case["codes"][:] = -1  # unsigned 65535
    layer, t = make_module(case, DEV)
    y = layer(t["x"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT
    case8 = O.make_case(7303, 256, 16, 2, 8, 8, 1, False)
    case8["codes"][:] = -128  # unsigned 128
    layer8, t8 = make_module(case8, DEV)
    assert O.relative_error(layer8(t8["x"]).float().cpu().numpy(), oracle_output(case8)) < TOL_FP16_TIGHT


def test_linearity_and_zero_input_at_full_size():
    """Size-independent properties at BASELINE configs[1] size (4096 -> 14336, 1x16): f(0)=bias-free 0,
    f(a*x1 + x2) = a*f(x1) + f(x2) up to fp16 rounding."""
    fin, fout = 4096, 14336
    g = torch.Generator(device=DEV).manual_seed(1)
    codes = torch.randint(-32768, 32768, (fout, fin // 8, 1), dtype=torch.int16, device=DEV, generator=g)
    codebooks = torch.randn((1, 65536, 1, 8), dtype=torch.float16, device=DEV, generator=g)
    scales = (0.75 + 0.5 * torch.rand((fout, 1, 1, 1), device=DEV, generator=g)).half()
    from aqlm_b200.inference_kernels import cuda_kernel

    x1 = torch.randn((1, fin), dtype=torch.float16, device=DEV, generator=g)
    x2 = torch.randn((1, fin), dtype=torch.float16, device=DEV, generator=g)
    f = lambda x: cuda_kernel.matmat(x, codes, codebooks, scales, None).float()  # noqa: E731
    assert torch.count_nonzero(f(torch.zeros_like(x1))) == 0
    lhs = f((2.0 * x1 + x2))
    rhs = 2.0 * f(x1) + f(x2)
    rel = (lhs - rhs).abs().mean() / rhs.abs().mean()
    assert rel < 2e-3
    # batched rows equal the row-by-row results exactly (same kernel arithmetic per row)
    xb = torch.cat([x1, x2, x1 - x2], 0)
    yb = cuda_kernel.matmat(xb, codes, codebooks, scales, None)
    for i in range(3):
        assert torch.equal(yb[i], cuda_kernel.matmat(xb[i : i + 1], codes, codebooks, scales, None)[0])
    # and the full-size result itself against the C oracle (every output row)
    t = dict(x=x1, codes=codes, codebooks=codebooks, scales=scales, bias=None)
    assert c_oracle_check(t, f(x1)) < TOL_FP16_TIGHT


def test_full_size_config0_matches_oracle_c_port():
    """BASELINE configs[0]: 4096->4096 1x16 bs=1 against the C oracle on the same inputs."""
    from oracle import c_oracle

    case = O.make_case(1000, 4096, 4096, 1, 16, 8, 1, False)
    layer, t = make_module(case, DEV)
    y = layer(t["x"]).float().cpu().numpy()
    ref = c_oracle.dequantize_gemm(case["x"], case["codes"], case["codebooks"], case["scales"], None)
    assert O.relative_error(y, ref) < TOL_FP16_TIGHT


def test_flat_c_abi_wrappers():
    """Call the flat entry points (named after the reference pybind functions) directly through ctypes."""
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    for K, nbits, entry in [(1, 16, "code1x16"), (2, 8, "code2x8"), (1, 8, "code1x8")]:
        case = O.make_case(7400 + K + nbits, 512, 96, K, nbits, 8, 2, True)
        t = to_torch(case, DEV)
        y = torch.empty((2, 96), dtype=torch.float16, device=DEV)
        st = torch.cuda.current_stream().cuda_stream
        args = [t["x"].data_ptr(), t["codes"].data_ptr(), t["codebooks"].data_ptr(), t["scales"].data_ptr(),
                t["bias"].data_ptr(), y.data_ptr(), 2, 512, 96]
        for suffix in ("_matmat", "_matmat_dequant"):
            fn = getattr(L, f"aqlm_b200_{entry}{suffix}")
            rc = fn(*args, 8, _cabi.F16, st) if entry == "code1x16" else fn(*args, _cabi.F16, st)
            _cabi.check(rc)
            assert O.relative_error(y.float().cpu().numpy(), oracle_output(case)) < TOL_FP16_TIGHT
        W = torch.empty((96, 512), dtype=torch.float16, device=DEV)
        fn = getattr(L, f"aqlm_b200_{entry}_dequant")
        dargs = [t["codes"].data_ptr(), t["codebooks"].data_ptr(), t["scales"].data_ptr(), W.data_ptr(), 512, 96]
        rc = fn(*dargs, 8, _cabi.F16, st) if entry == "code1x16" else fn(*dargs, _cabi.F16, st)
        _cabi.check(rc)
        Wref = O.dequantize_weight(O.unpack_int_data(case["codes"], nbits), case["codebooks"], case["scales"])
        np.testing.assert_allclose(W.float().cpu().numpy(), Wref, rtol=2.0**-10, atol=1e-6)


def test_host_buffer_entry_point():
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(7500, 1024, 128, 1, 16, 8, 1, False)
    t = to_torch(case, DEV)
    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), None)
    xh = torch.from_numpy(case["x"]).pin_memory()
    yh = torch.empty((1, 128), dtype=torch.float16).pin_memory()
    xd, yd = torch.empty_like(t["x"]), torch.empty((1, 128), dtype=torch.float16, device=DEV)
    _cabi.check(_cabi.lib().aqlm_b200_matmat_host(ctypes.byref(w), xh.data_ptr(), yh.data_ptr(), xd.data_ptr(),
                                                  yd.data_ptr(), 1, torch.cuda.current_stream().cuda_stream))
    assert O.relative_error(yh.float().numpy(), oracle_output(case)) < TOL_FP16_TIGHT


def test_partial_f32_plus_epilogue_equals_fused():
    """The sharded path's building blocks: sum of per-shard fp32 partials + scale_bias == fused result."""
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(7600, 2048, 192, 1, 16, 8, 3, True)
    t = to_torch(case, DEV)
    full = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    parts = 0
    for r in range(4):
        cs = t["codes"][:, r * 64 : (r + 1) * 64].contiguous()
        xs = t["x"][:, r * 512 : (r + 1) * 512].contiguous()
        parts = parts + cuda_kernel.matmat_partial(xs, cs, t["codebooks"])
    y = cuda_kernel.scale_bias(parts, t["scales"], t["bias"], torch.float16)
    assert O.relative_error(y.float().cpu().numpy(), oracle_output(case)) < TOL_FP16_TIGHT
    assert (y.float() - full.float()).abs().max() <= 2e-3 * full.float().abs().max()


def test_error_behaviour_matches_reference():
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(7700, 256, 32, 1, 16, 8, 1, False)
    t = to_torch(case, DEV)
    with pytest.raises(NotImplementedError, match="only support float16 and bfloat16"):
        cuda_kernel.matmat(t["x"].float(), t["codes"], t["codebooks"].float(), t["scales"].float(), None)
    with pytest.raises(ValueError):
        cuda_kernel.matmat(t["x"][:, :128], t["codes"], t["codebooks"], t["scales"], None)
    with pytest.raises(NotImplementedError):
        cuda_kernel.matmat(t["x"].cpu(), t["codes"].cpu(), t["codebooks"].cpu(), t["scales"].cpu(), None)


def test_backward_wrt_input():
    case = O.make_case(7800, 512, 96, 2, 8, 8, 9, False)
    layer, t = make_module(case, DEV)
    x = t["x"].clone().requires_grad_(True)
    y = layer(x)
    go = torch.randn_like(y)
    (gx,) = torch.autograd.grad(y, x, go)
    W = O.dequantize_weight(O.unpack_int_data(case["codes"], 8), case["codebooks"], case["scales"])
    ref = go.float().cpu().numpy() @ W
    assert O.relative_error(gx.float().cpu().numpy(), ref) < 2e-3


def test_cuda_graph_capture_and_replay():
    case = O.make_case(7900, 1024, 256, 1, 16, 8, 1, False)
    layer, t = make_module(case, DEV)
    x = t["x"].clone()
    layer(x)  # bind ops outside capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = layer(x)
    x.copy_(t["x"] * 0.5)
    g.replay()
    torch.cuda.synchronize()
    ref = 0.5 * oracle_output(case)
    assert O.relative_error(y.float().cpu().numpy(), ref) < 1e-3


# ---- fused dequant + wgmma GEMM (large batch) -----------------------------------------------------------------
# The test_tcgen05_gemm_* names predate the Hopper port and are kept so that the test ids stay stable; they test the
# wgmma kernels of csrc/gemm_wgmma.cuh.  Bit-exact checks of every plan are in test_zz_gemm_exact.py.
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8), (8, 8), (1, 8)])
@pytest.mark.parametrize("batch", [7, 16, 64, 100, 256, 300])
def test_tcgen05_gemm_vs_oracle_small(K, nbits, batch):
    """Sizes the numpy oracle finishes in seconds; in_features % 64 == 0 so the tensor-core kernel is used."""
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(8000 + K + nbits + batch, 512, 200, K, nbits, 8, batch, bias=(batch % 2 == 0))
    t = to_torch(case, DEV)
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT


@pytest.mark.parametrize("batch", [16, 64, 256])
@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336), (14336, 4096)])
def test_tcgen05_gemm_full_size_1x16(shape, batch):
    """BASELINE configs[3]: Llama-3-8B shapes, bs in {16,64,256}, fp16 operands, against the C ORACLE (row sample that
    includes both tile edges; every batch row)."""
    from aqlm_b200.inference_kernels import cuda_kernel

    fin, fout = shape
    t = gpu_case(fin, fout, 1, 16, batch, seed=fin + fout + batch)
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    rel = c_oracle_check(t, y)
    assert rel < TOL_FP16_TIGHT, rel
    # deterministic (fixed-order split-K reduction): bitwise identical on a second run
    y2 = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    assert torch.equal(y, y2)
    # gemm op and gemv op agree on the first rows
    yv = cuda_kernel.matmat(t["x"][:4], t["codes"], t["codebooks"], t["scales"], None).float()
    assert ((yv - y[:4].float()).abs().mean() / yv.abs().mean()).item() < 1e-3


@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336)])
def test_tcgen05_gemm_bf16_operands(shape):
    """bf16 operands (the run north_star names) at BASELINE shapes: C oracle fed with the bf16 values, bf16 tolerance."""
    from aqlm_b200.inference_kernels import cuda_kernel

    fin, fout = shape
    t = gpu_case(fin, fout, 1, 16, 256, dtype=torch.bfloat16, seed=5 + fout)
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    assert c_oracle_check(t, y) < TOL_BF16


@pytest.mark.parametrize("K,nbits,shape", [(2, 8, (4096, 11008)), (2, 8, (11008, 4096)), (8, 8, (4096, 4096)),
                                           (1, 8, (4096, 11008))])
def test_tcgen05_gemm_full_size_kx8(K, nbits, shape):
    """BASELINE configs[2] shapes through the large-batch op (Kx8 schemes), against the C oracle."""
    from aqlm_b200.inference_kernels import cuda_kernel

    fin, fout = shape
    t = gpu_case(fin, fout, K, nbits, 64, seed=K * 7 + fin, bias=True)
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    assert c_oracle_check(t, y) < TOL_FP16_TIGHT


def test_tcgen05_gemm_without_workspace_matches_split():
    """The C-ABI entry point without a workspace (no split-K) gives the same result up to fp32 summation order."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(8100, 1024, 256, 1, 16, 8, 32, True)
    t = to_torch(case, DEV)
    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), t["bias"])
    y = torch.empty((32, 256), dtype=torch.float16, device=DEV)
    _cabi.check(_cabi.lib().aqlm_b200_matmat_dequant(ctypes.byref(w), t["x"].data_ptr(), y.data_ptr(), 32,
                                                     torch.cuda.current_stream().cuda_stream))
    assert O.relative_error(y.float().cpu().numpy(), oracle_output(case)) < TOL_FP16_TIGHT


def test_gemm_1x8_row_stride_not_tma_compatible_falls_back():
    """1x8 with in_features % 128 != 0: the code rows are not a 16-byte multiple, so the TMA kernel cannot be used; the
    large-batch op must still answer (GEMV passes), not fail in cuTensorMapEncodeTiled."""
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(8200, 192, 72, 1, 8, 8, 9, True)
    t = to_torch(case, DEV)
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"]).float().cpu().numpy()
    assert O.relative_error(y, oracle_output(case)) < TOL_FP16_TIGHT


# ---- fused dequant-transpose GEMM (backward w.r.t. the input; SURVEY §8 a6 / f3) ------------------------------------
def _transposed_ref(t, go):
    """(grad_out * scales) @ W_unscaled with the C oracle's dequantized weights, fp32 (reference cuda_kernel.cpp:303-354)."""
    from oracle import c_oracle

    f32 = lambda a: a.float().cpu().numpy()  # noqa: E731
    W = c_oracle.dequantize_weight(t["codes"].cpu().numpy(), f32(t["codebooks"]), f32(t["scales"]))  # scaled rows
    return f32(go) @ W


@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8), (1, 8), (8, 8), (4, 8)])
@pytest.mark.parametrize("batch", [1, 7, 64, 256, 300])
def test_transposed_gemm_vs_oracle_small(K, nbits, batch):
    from aqlm_b200.inference_kernels import cuda_kernel

    # ragged in out only (out % 64 != 0); in is a multiple of 128 in both shapes -- test_zz_gemm_exact covers ragged in
    fin, fout = (512, 200) if batch != 64 else (1152, 456)
    t = gpu_case(fin, fout, K, nbits, 1, seed=8300 + K + nbits + batch)
    go = torch.randn((batch, fout), dtype=torch.float16, device=DEV)
    before = aqlm_launches()
    gx = cuda_kernel.matmat_dequant_transposed(go, t["codes"], t["codebooks"], t["scales"], None)
    assert aqlm_launches() == before + 1, "the backward must be ONE fused kernel (no dequant + library GEMM)"
    assert gx.shape == (batch, fin)
    assert O.relative_error(gx.float().cpu().numpy(), _transposed_ref(t, go)) < TOL_NORTH_STAR


@pytest.mark.parametrize("K,nbits,shape,dtype", [(1, 16, (4096, 14336), torch.float16), (1, 16, (14336, 4096), torch.float16),
                                                 (2, 8, (4096, 11008), torch.float16), (1, 16, (4096, 4096), torch.bfloat16)])
def test_transposed_gemm_full_size(K, nbits, shape, dtype):
    from aqlm_b200.inference_kernels import cuda_kernel

    fin, fout = shape
    t = gpu_case(fin, fout, K, nbits, 1, dtype=dtype, seed=8400 + fin)
    go = torch.randn((256, fout), dtype=dtype, device=DEV)
    gx = cuda_kernel.matmat_dequant_transposed(go, t["codes"], t["codebooks"], t["scales"], None)
    rel = O.relative_error(gx.float().cpu().numpy(), _transposed_ref(t, go))
    assert rel < (TOL_NORTH_STAR if dtype == torch.float16 else TOL_BF16), rel
    gx2 = cuda_kernel.matmat_dequant_transposed(go, t["codes"], t["codebooks"], t["scales"], None)
    assert torch.equal(gx, gx2)  # deterministic split-K


def test_module_backward_uses_the_fused_kernel():
    """autograd through QuantizedLinear at a training-size batch: grad w.r.t. the input comes from the fused kernel."""
    case = O.make_case(8500, 1024, 384, 1, 16, 8, 32, False)
    layer, t = make_module(case, DEV)
    x = t["x"].clone().requires_grad_(True)
    y = layer(x)
    go = torch.randn_like(y)
    before = aqlm_launches()
    (gx,) = torch.autograd.grad(y, x, go)
    assert aqlm_launches() == before + 1
    W = O.dequantize_weight(O.unpack_int_data(case["codes"], 16), case["codebooks"], case["scales"])
    assert O.relative_error(gx.float().cpu().numpy(), go.float().cpu().numpy() @ W) < TOL_NORTH_STAR


def test_misaligned_input_through_the_c_abi():
    """x only element-aligned (2 bytes off a 16-byte boundary): the C-ABI must take the slow path, not fault."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    case = O.make_case(8600, 512, 64, 1, 16, 8, 1, True)
    t = to_torch(case, DEV)
    buf = torch.zeros(512 + 8, dtype=torch.float16, device=DEV)
    buf[1:513] = t["x"][0]
    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), t["bias"])
    y = torch.empty((1, 64), dtype=torch.float16, device=DEV)
    _cabi.check(_cabi.lib().aqlm_b200_matmat(ctypes.byref(w), buf.data_ptr() + 2, y.data_ptr(), 1,
                                             torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert O.relative_error(y.float().cpu().numpy(), oracle_output(case)) < TOL_FP16_TIGHT


# ---- full-size matvec parity against the C oracle (every output row) ------------------------------------------------
LLAMA3_8B = [(4096, 4096), (4096, 1024), (4096, 14336), (14336, 4096)]
LLAMA3_70B = [(8192, 8192), (8192, 1024), (8192, 28672), (28672, 8192)]


@pytest.mark.parametrize("fin,fout", LLAMA3_8B + LLAMA3_70B)
def test_gemv_1x16_baseline_shapes_vs_c_oracle(fin, fout):
    """BASELINE configs[1] (Llama-3-8B) and configs[4] (Llama-3-70B, unsharded) 1x16 matvec, all rows, vs the C oracle."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(fin, fout, 1, 16, 1, seed=fin * 3 + fout)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    assert c_oracle_check(t, y) < TOL_FP16_TIGHT


@pytest.mark.parametrize("batch", [2, 4, 6])
def test_gemv_1x16_small_batches_full_size(batch):
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(4096, 14336, 1, 16, batch, seed=77 + batch, bias=True)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    assert c_oracle_check(t, y) < TOL_FP16_TIGHT


@pytest.mark.parametrize("K,nbits,fin,fout", [(1, 16, 4096, 14336), (1, 16, 14336, 4096), (2, 8, 4096, 11008),
                                              (8, 8, 4096, 4096), (1, 8, 4096, 11008)])
def test_gemv_bf16_baseline_shapes_vs_c_oracle(K, nbits, fin, fout):
    """bf16 GEMV / batch-1 LUT GEMV at BASELINE shapes against a bf16-fed C oracle (all rows)."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(fin, fout, K, nbits, 1, dtype=torch.bfloat16, seed=K + fin)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    assert c_oracle_check(t, y) < TOL_BF16


# ---- Kx8 dot-product-LUT GEMV (batch 1) -------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("fin,fout", [(4096, 4096), (4096, 11008), (11008, 4096), (1032, 77), (264, 33), (1040, 77),
                                      (2048, 300), (16, 5)])
def test_lut_gemv_kx8(K, fin, fout):
    """BASELINE configs[2] shapes (Llama-2-7B: q/k/v/o, gate/up, down) plus ragged sizes (in_groups not a multiple of the
    slab), all rows against the C oracle."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(fin, fout, K, 8, 1, seed=K * 1000 + fin + fout, bias=True)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    rel = c_oracle_check(t, y)
    assert rel < TOL_FP16_TIGHT, rel
    y2 = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    assert torch.equal(y, y2)  # fixed-order slab reduction


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("fin,fout", [(4096, 4096), (4096, 12288), (4096, 22016), (1024, 200)])
def test_lut_cluster_kernel(dtype, bias, K, fin, fout):
    """The cluster LUT GEMV (K <= 2, in_features <= 4096; csrc/gemv_lut.cuh) on row blocks of 32 .. 1472 rows: one
    round of warps and several, both the 768- and the 1024-thread build, all rows against the C oracle."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(fin, fout, K, 8, 1, dtype=dtype, seed=K * 77 + fin + fout, bias=bias)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    rel = c_oracle_check(t, y)
    assert rel < (TOL_FP16_TIGHT if dtype == torch.float16 else TOL_BF16), rel
    y2 = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    assert torch.equal(y, y2)  # fixed-order cross-slab sum


@pytest.mark.parametrize("K,batch", [(2, 2), (2, 5), (8, 3), (1, 6)])
def test_kx8_small_batches_full_size(K, batch):
    """Batch 2-6 on 256-entry codebooks (the reference loops its matvec per row, cuda_kernel.cpp:387-421)."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(4096, 11008, K, 8, batch, seed=K * 10 + batch)
    y = cuda_kernel.matmat(t["x"], t["codes"], t["codebooks"], t["scales"], None)
    assert c_oracle_check(t, y) < TOL_FP16_TIGHT


def test_cuda_graph_with_workspace_ops():
    """Graph capture of the ops that use the persistent workspace (LUT GEMV tickets/partials, split-K GEMM), warmed up on
    a side stream as in the PyTorch recipe; the workspace later GROWS (bigger eager call) and the graph must still replay
    correctly (outgrown buffers are retired, never freed)."""
    from aqlm_b200.inference_kernels import cuda_kernel

    t2 = gpu_case(4096, 4096, 2, 8, 1, seed=901)
    t16 = gpu_case(4096, 4096, 1, 16, 64, seed=902)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            cuda_kernel.matmat(t2["x"], t2["codes"], t2["codebooks"], t2["scales"], None)
            cuda_kernel.matmat_dequant(t16["x"], t16["codes"], t16["codebooks"], t16["scales"], None)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ya = cuda_kernel.matmat(t2["x"], t2["codes"], t2["codebooks"], t2["scales"], None)
        yb = cuda_kernel.matmat_dequant(t16["x"], t16["codes"], t16["codebooks"], t16["scales"], None)
    g.replay()
    torch.cuda.synchronize()
    assert c_oracle_check(t2, ya) < TOL_FP16_TIGHT and c_oracle_check(t16, yb) < TOL_FP16_TIGHT
    # grow the eager workspace well past its initial size, then replay the old graph with new inputs
    big = gpu_case(4096, 14336, 1, 16, 200, seed=903)
    cuda_kernel.matmat_dequant(big["x"], big["codes"], big["codebooks"], big["scales"], None)
    t2["x"].mul_(0.5)
    t16["x"].mul_(0.5)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert c_oracle_check(t2, ya) < TOL_FP16_TIGHT and c_oracle_check(t16, yb) < TOL_FP16_TIGHT


# ---- grouped launch (q/k/v, gate/up) -----------------------------------------------------------------------------
@pytest.mark.parametrize("batch", [1, 3, 8])
def test_grouped_launch_equals_members(batch):
    import aqlm_b200

    outs = [512, 128, 128]
    cases = [O.make_case(9100 + i, 1024, o, 1, 16, 8, batch, bias=True) for i, o in enumerate(outs)]
    for c in cases[1:]:
        c["x"] = cases[0]["x"]  # same activation
    members, ts = zip(*[make_module(c, DEV) for c in cases])
    before = {f"{i}.{k}": v.clone() for i, m in enumerate(members) for k, v in m.state_dict().items()}
    group = aqlm_b200.QuantizedLinearGroup(list(members))
    assert group.fused
    # fusing re-points the members' parameters at views of the fused storage: values and state_dict layout unchanged
    for i, m in enumerate(members):
        for k, v in m.state_dict().items():
            assert v.shape == before[f"{i}.{k}"].shape and torch.equal(v, before[f"{i}.{k}"])
    assert sorted(group.state_dict().keys()) == sorted(f"members.{k}" for k in before)
    x = ts[0]["x"]
    ys = group(x)
    assert len(ys) == 3
    for m, c, y in zip(members, cases, ys):
        if batch <= 6:  # members use the same GEMV arithmetic per row: bit-identical (above 6 rows they take the GEMM op)
            assert torch.equal(y, m(x))
        assert O.relative_error(y.float().cpu().numpy(), oracle_output(c)) < TOL_FP16_TIGHT
    # large batches fall back to the members (tensor-core op)
    xb = torch.randn((16, 1024), dtype=torch.float16, device=DEV)
    yb = group(xb)
    assert yb[0].shape == (16, 512)
