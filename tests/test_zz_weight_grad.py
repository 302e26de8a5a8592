"""The weight gradient of a quantized linear: codebook and scale gradients from the fused wgmma GEMM (csrc/gemm_wgrad.cuh).

CPU: the plan (`gemm_wgrad_plan` in plan.cuh, through a driver compiled as test_host_plans.py compiles one) and the C-ABI's
argument checks, which run before any device query.

GPU: bit-exact on an integer lattice.  x, grad_output and codebooks are small integers and scales are powers of two, so
D = grad_output^T x is exact in fp32; every codebook-gradient term s_r * D[r, j] is a multiple of 2^-E_HI, and the test
asserts, from the drawn data, that the sum of the ABSOLUTE terms landing on any one output stays below 2^(24 - E_HI).  Then
every partial sum is exact whatever the order of the atomic reductions, and the kernel's fp32 output equals the fp64
reference exactly.  The same holds for grad_scales (integer terms D * Wu).  Random data at Llama sizes, the modules'
autograd wiring, CUDA graphs and a tiny Llama end to end are checked against dense references within tolerance.
"""
import ctypes
import math
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch

from aqlm_b200 import _cabi
from oracle import aqlm_oracle as O

DEV = "cuda:0"
gpu = pytest.mark.gpu
SMEM_OPTIN = 232448        # H100 opt-in shared memory per block
WS_COUNTERS = 65536        # counter region at the head of every workspace (plan.cuh kWsCountersBytes)
SCHEMES = [(K, nbits) for K in (1, 2, 4, 8) for nbits in (8, 16)]
DTYPES = [torch.float16, torch.bfloat16]
DT_ID = {torch.float16: "f16", torch.bfloat16: "bf16"}
X_MAX, CB_MAX, E_HI = 2, 2, 3


# ---- plan (CPU) ------------------------------------------------------------------------------------------------------
def wgrad_smem(stages, K, nbits):
    """gemm_wgrad_smem_layout().total: the stages, or the epilogue's staged D (128 x 132 fp32) and, for 8-bit codes, the
    CTA's K x 256 x 8 fp32 codebook gradient; then barriers, flag and alignment slack."""
    epi = 128 * 132 * 4 + (K * 256 * 8 * 4 if nbits <= 8 else 0)
    return max(stages * 32768, epi) + 8 * 8 * 2 + 4 + 1024


def expected_plan(K, nbits, g, fin, fout, off, batch, smem=SMEM_OPTIN, forced=0):
    cb = 1 if nbits <= 8 else 2
    if g != 8 or nbits not in (8, 16) or K not in (1, 2, 4, 8) or off % 16 or (fin // 8 * K * cb) % 16 or fout % 8:
        return "0"
    size = lambda s: wgrad_smem(s, K, nbits)  # noqa: E731
    stages = 3
    while stages > 2 and size(stages) > smem:
        stages -= 1
    if size(stages) > smem:
        return "0"
    if 2 <= forced <= 4 and size(forced) <= smem:
        stages = forced
    out_tiles, in_tiles = -(-fout // 128), -(-fin // 128)
    return (f"1 {out_tiles} {in_tiles} {stages} {-(-batch // 64)} {size(stages)} {WS_COUNTERS} "
            f"{in_tiles * fout * 4}")


DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

#include "plan.cuh"

using namespace aqlm_b200;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    long long K, nbits, g, fin, fout, off, batch, smem;
    int stages;
    is >> K >> nbits >> g >> fin >> fout >> off >> batch >> smem >> stages;
    Tunables t;
    t.load();
    t.gemm_stages = stages;
    DeviceInfo di;
    di.max_smem_optin = (int)smem;
    di.sm_count = 132;
    di.cc_major = 9;
    di.ok = true;
    aqlm_b200_weight_t w = {};
    w.codes = reinterpret_cast<const void*>(0x7f0000000000ull + off);
    w.codebooks = reinterpret_cast<const void*>(0x7f1000000000ull);
    w.scales = reinterpret_cast<const void*>(0x7f2000000000ull);
    w.in_features = fin;
    w.out_features = fout;
    w.num_codebooks = (int)K;
    w.nbits_per_codebook = (int)nbits;
    w.in_group_size = (int)g;
    w.out_group_size = 1;
    w.dtype = AQLM_B200_F16;
    const WgradPlan p = gemm_wgrad_plan(w, batch, di, t);
    if (!p.ok) std::printf("0\n");
    else std::printf("1 %d %d %d %d %zu %zu %zu\n", p.out_tiles, p.in_tiles, p.stages, p.total_kblocks, p.smem,
                     p.counters_bytes, p.dots_bytes);
  }
  return 0;
}
"""


def plan_cases():
    """(K, nbits, g, in, out, codes offset, batch, smem, forced stages)"""
    shapes = [(128, 8), (1088, 200), (1152, 456), (4096, 4096), (4096, 14336), (14336, 4096), (8192, 28672)]
    batches = [1, 7, 63, 64, 65, 129, 300, 1024, 4096, 16384]
    for K, nbits in SCHEMES:
        for fin, fout in shapes:
            for b in batches:
                yield (K, nbits, 8, fin, fout, 0, b, SMEM_OPTIN, 0)
    for K, nbits, g, off in [(1, 16, 16, 0), (3, 8, 8, 0), (1, 12, 8, 0), (1, 16, 8, 8), (2, 8, 8, 4)]:
        for b in (1, 300):
            yield (K, nbits, g, 4096, 4096, off, b, SMEM_OPTIN, 0)
    for fin, fout in [(64, 1), (4096, 4100), (1032, 512)]:  # out % 8 != 0; 1x8 code rows of 129 bytes
        for K, nbits in [(1, 16), (1, 8), (2, 8)]:
            yield (K, nbits, 8, fin, fout, 0, 64, SMEM_OPTIN, 0)
    for smem in (60000, 70000, 99000, 120000, 140000):  # fewer stages, then none, as the opt-in shared memory shrinks
        for K, nbits in [(1, 16), (2, 8), (8, 8)]:
            yield (K, nbits, 8, 4096, 4096, 0, 1024, smem, 0)
    for forced in (2, 4, 5):
        for K, nbits in [(1, 16), (8, 8)]:
            yield (K, nbits, 8, 4096, 4096, 0, 1024, SMEM_OPTIN, forced)


def test_weight_grad_plan_pins(tmp_path):
    src = tmp_path / "wgrad_plans.cu"
    src.write_text(DRIVER)
    exe = tmp_path / "wgrad_plans"
    flags = [f for f in _cabi.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    subprocess.run(["nvcc", *flags, "-I", _cabi.CSRC, "-o", str(exe), str(src)], check=True, capture_output=True, text=True)
    cases = list(plan_cases())
    env = {k: v for k, v in os.environ.items() if not k.startswith("AQLM_B200_")}
    got = subprocess.run([str(exe)], input="\n".join(" ".join(map(str, c)) for c in cases) + "\n", check=True,
                         capture_output=True, text=True, env=env).stdout.splitlines()
    assert len(got) == len(cases)
    want = [expected_plan(*c[:7], smem=c[7], forced=c[8]) for c in cases]
    diff = [f"{c}: want [{w}] got [{g}]" for c, w, g in zip(cases, want, got) if w != g]
    assert not diff, f"{len(diff)} of {len(cases)} plans differ:\n" + "\n".join(diff[:20])
    assert sum(w == "0" for w in want) >= 20 and any(w.split()[3] == "2" for w in want if w != "0")


# ---- C-ABI argument checks (CPU: no device is touched) ---------------------------------------------------------------
def _weight(K=2, nbits=8, g=8, fin=256, fout=64):
    w = _cabi.Weight()
    w.codes, w.codebooks, w.scales = 16, 16, 16  # dummy non-null aligned pointers (never dereferenced)
    w.in_features, w.out_features = fin, fout
    w.num_codebooks, w.nbits_per_codebook, w.in_group_size, w.out_group_size = K, nbits, g, 1
    w.dtype = _cabi.F16
    return w


def test_weight_grad_c_abi_checks_without_a_device():
    L = _cabi.lib()
    for name in ("aqlm_b200_matmat_weight_grad", "aqlm_b200_matmat_weight_grad_workspace_bytes"):
        assert name in _cabi.header_symbols() and hasattr(ctypes.CDLL(_cabi.LIB_PATH), name)
    call = lambda w, x=16, go=16, b=64, gcb=16, gs=16: L.aqlm_b200_matmat_weight_grad(  # noqa: E731
        ctypes.byref(w), x, go, b, gcb, gs, None, 0, None)
    w = _weight()
    assert call(w, x=None) == _cabi.ERR_SHAPE
    assert call(w, go=None) == _cabi.ERR_SHAPE
    assert call(w, gcb=None, gs=None) == _cabi.ERR_SHAPE
    assert b"neither" in L.aqlm_b200_last_error()
    assert call(w, b=-1) == _cabi.ERR_SHAPE
    w.scales = None
    assert call(w, gs=None) == _cabi.ERR_SHAPE                          # grad_codebooks needs the scales
    assert call(_weight(fin=60)) == _cabi.ERR_SHAPE                      # in % in_group != 0
    w = _weight()
    w.dtype = 7
    assert call(w) == _cabi.ERR_DTYPE
    assert call(_weight(K=1, nbits=16, g=16)) == _cabi.ERR_UNSUPPORTED    # in_group 16
    assert call(_weight(K=3)) == _cabi.ERR_UNSUPPORTED                    # 3 codebooks
    assert call(_weight(fout=60)) == _cabi.ERR_UNSUPPORTED                # out % 8
    assert call(_weight(K=1, fin=1032)) == _cabi.ERR_UNSUPPORTED          # 129-byte code rows
    assert call(_weight(), x=24) == _cabi.ERR_UNSUPPORTED                 # input 8-byte aligned only
    assert call(_weight(), go=8) == _cabi.ERR_UNSUPPORTED
    w = _weight()
    w.codes = 24
    assert call(w) == _cabi.ERR_UNSUPPORTED
    if not torch.cuda.is_available():
        assert call(_weight(), b=0) == _cabi.OK                           # batch 0: no launch, no device query
        assert call(_weight()) in (_cabi.ERR_CUDA, _cabi.ERR_ARCH)        # a valid call needs the device, never falls back
        assert L.aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(_weight()), 64) == 0


# ---- lattice (GPU) ---------------------------------------------------------------------------------------------------
def lattice_linear(seed, fin, fout, K, nbits, g=8):
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 2 ** nbits, size=(fout, fin // g, K), dtype=np.int64)
    top = 2 ** nbits - 1
    raw[::7, 0, :] = top  # both extremes of the unsigned range
    raw[3::11, -1, :] = 0
    cb = rng.integers(-CB_MAX, CB_MAX + 1, size=(K, 2 ** nbits, 1, g)).astype(np.float32)
    sc = np.ldexp(np.float32(1.0), -rng.integers(0, E_HI + 1, size=fout)).astype(np.float32).reshape(fout, 1, 1, 1)
    return dict(raw=raw, codes=O.pack_int_data(raw.copy(), nbits), codebooks=cb, scales=sc)


def exact_weight_grad(lin, x, go):
    """fp64 (grad_codebooks [K, 2^nbits, 1, g], grad_scales [out]) and the premise that fp32 sums of them are exact."""
    raw, cb, sc = lin["raw"], lin["codebooks"].astype(np.float64), lin["scales"].reshape(-1).astype(np.float64)
    K, n, _, g = cb.shape
    fout = raw.shape[0]
    D = go.astype(np.float64).T @ x.astype(np.float64)  # [out, in]
    Wu = np.zeros_like(D).reshape(fout, -1, g)
    for k in range(K):
        Wu += cb[k, raw[:, :, k], 0, :]
    gs = (D.reshape(fout, -1, g) * Wu).sum(axis=(1, 2))
    sD = (D * sc[:, None]).reshape(-1, g)
    gcb = np.zeros((K, n, g))
    mag = np.zeros((K, n, g))
    for k in range(K):
        idx = raw[:, :, k].reshape(-1)
        for i in range(g):
            gcb[k, :, i] = np.bincount(idx, weights=sD[:, i], minlength=n)
            mag[k, :, i] = np.bincount(idx, weights=np.abs(sD[:, i]), minlength=n)
    assert mag.max() < 2.0 ** (24 - E_HI), "codebook-gradient sums may round: shrink the lattice"
    assert np.abs(D.reshape(fout, -1, g) * Wu).sum(axis=(1, 2)).max() < 2.0 ** 24
    return gcb.reshape(K, n, 1, g), gs


def to_dev(a, dtype):
    return torch.from_numpy(np.asarray(a, dtype=np.float32)).to(dtype).to(DEV)


def c_weight_grad(t, x, go, gcb, gs, ws):
    """The C-ABI call on device tensors; returns its status."""
    from aqlm_b200.inference_kernels import cuda_kernel

    w = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), None)
    rc = _cabi.lib().aqlm_b200_matmat_weight_grad(
        ctypes.byref(w), x.data_ptr(), go.data_ptr(), x.shape[0], gcb.data_ptr() if gcb is not None else None,
        gs.data_ptr() if gs is not None else None, ws.data_ptr() if ws is not None else None,
        ws.numel() if ws is not None else 0, torch.cuda.current_stream().cuda_stream)
    return rc


LATTICE_SHAPES = [(128, 8), (1088, 200), (1152, 456)]
LATTICE_BATCHES = [1, 7, 64, 129, 300, 1024]


@gpu
@pytest.mark.parametrize("shape", LATTICE_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits", SCHEMES, ids=lambda v: str(v))
def test_lattice_weight_grad_is_exact(K, nbits, dtype, shape):
    from aqlm_b200.inference_kernels import cuda_kernel

    fin, fout = shape
    lin = lattice_linear(1000 * K + nbits + fin, fin, fout, K, nbits)
    t = dict(codes=torch.from_numpy(lin["codes"]).to(DEV), codebooks=to_dev(lin["codebooks"], dtype),
             scales=to_dev(lin["scales"], dtype))
    L = _cabi.lib()
    fused = (fin // 8 * K * (1 if nbits <= 8 else 2)) % 16 == 0  # 1x8 at in = 1088: 136-byte code rows
    for batch in LATTICE_BATCHES:
        rng = np.random.default_rng(batch * 7 + fin)
        x = rng.integers(-X_MAX, X_MAX + 1, size=(batch, fin)).astype(np.float32)
        go = rng.integers(-X_MAX, X_MAX + 1, size=(batch, fout)).astype(np.float32)
        ref_cb, ref_s = exact_weight_grad(lin, x, go)
        xd, god = to_dev(x, dtype), to_dev(go, dtype)
        what = f"{K}x{nbits} {DT_ID[dtype]} {fin}x{fout} batch {batch}"
        # the Python op: the parameters' dtypes, rounded once (the dense formulation where the kernel refuses)
        pcb, ps = cuda_kernel.matmat_weight_grad(xd, god, t["codes"], t["codebooks"], t["scales"])
        assert torch.equal(pcb.float().cpu(), to_dev(ref_cb, dtype).float().cpu()), what
        assert torch.equal(ps.float().cpu(), to_dev(ref_s.reshape(-1, 1, 1, 1), dtype).float().cpu()), what
        w = cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), None)
        need = L.aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(w), batch)
        gcb = torch.zeros(ref_cb.shape, dtype=torch.float32, device=DEV)
        gs = torch.full((fout,), -7.0, dtype=torch.float32, device=DEV)
        if not fused:
            assert need == 0 and c_weight_grad(t, xd, god, gcb, gs, None) == _cabi.ERR_UNSUPPORTED
            continue
        assert need == WS_COUNTERS + math.ceil(fin / 128) * fout * 4
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        before = _cabi.launch_count()
        assert c_weight_grad(t, xd, god, gcb, gs, ws) == _cabi.OK
        torch.cuda.synchronize()
        assert _cabi.launch_count() - before == 1
        assert not ws[:WS_COUNTERS].any(), "ticket counters not left at zero"
        assert torch.equal(gcb.cpu(), torch.from_numpy(ref_cb.astype(np.float32))), what + ": grad_codebooks"
        assert torch.equal(gs.cpu(), torch.from_numpy(ref_s.astype(np.float32))), what + ": grad_scales"
        # a second call adds into grad_codebooks and rewrites grad_scales
        assert c_weight_grad(t, xd, god, gcb, gs, ws) == _cabi.OK
        assert torch.equal(gcb.cpu(), torch.from_numpy((2 * ref_cb).astype(np.float32))), what + ": accumulation"
        assert torch.equal(gs.cpu(), torch.from_numpy(ref_s.astype(np.float32)))
        # one output requested: the other buffer is untouched
        sentinel = torch.full_like(gcb, 5.0)
        gs2 = torch.zeros_like(gs)
        assert c_weight_grad(t, xd, god, None, gs2, ws) == _cabi.OK
        assert c_weight_grad(t, xd, god, sentinel, None, None) == _cabi.OK
        assert torch.equal(gs2, gs) and torch.equal(sentinel.cpu(), torch.from_numpy((ref_cb + 5).astype(np.float32)))
        assert not ws[:WS_COUNTERS].any()


# ---- random data at Llama sizes (GPU) --------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def dense_weight_grad(x, go, codes, codebooks, scales):
    """fp64 reference on the device: Wu rounded as the forward rounds it, D = G^T X."""
    from aqlm_b200.inference_kernels import cuda_kernel

    K, n, _, g = codebooks.shape
    Wu = cuda_kernel.dequant(codes, codebooks, None).double()
    D = go.reshape(-1, go.shape[-1]).double().t() @ x.reshape(-1, x.shape[-1]).double()
    gs = (D * Wu).sum(1)
    sD = (D * scales.reshape(-1, 1).double()).reshape(-1, g)
    c = codes.long() % n
    gcb = torch.zeros((K, n, g), dtype=torch.float64, device=D.device)
    for k in range(K):
        gcb[k].index_add_(0, c[:, :, k].reshape(-1), sD)
    return gcb.reshape(codebooks.shape), gs.reshape(scales.shape)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_random_llama_size_matches_fp64(K, nbits, dtype):
    from helpers import TOL_BF16, TOL_NORTH_STAR, gpu_case

    from aqlm_b200.inference_kernels import cuda_kernel

    t = gpu_case(4096, 4096, K, nbits, 2048, dtype=dtype, seed=5)
    go = torch.randn((2048, 4096), dtype=dtype, device=DEV, generator=torch.Generator(DEV).manual_seed(6))
    gcb, gs = cuda_kernel.matmat_weight_grad(t["x"], go, t["codes"], t["codebooks"], t["scales"])
    ref_cb, ref_s = dense_weight_grad(t["x"], go, t["codes"], t["codebooks"], t["scales"])
    tol = TOL_NORTH_STAR if dtype == torch.float16 else TOL_BF16
    assert rel(gcb, ref_cb) < tol and rel(gs, ref_s) < tol, (rel(gcb, ref_cb), rel(gs, ref_s))


# ---- modules (GPU) ---------------------------------------------------------------------------------------------------
def random_linear(fin, fout, K, nbits, g=8, dtype=torch.float16, seed=0, bias=True):
    import aqlm_b200

    gen = torch.Generator(DEV).manual_seed(seed)
    m = aqlm_b200.QuantizedLinear(fin, fout, g, 1, K, nbits, bias=bias, device=DEV, dtype=dtype)
    lo, hi = (-128, 128) if nbits <= 8 else (-(2 ** (nbits - 1)), 2 ** (nbits - 1))
    with torch.no_grad():
        m.codes.data = torch.randint(lo, hi, m.codes.shape, dtype=m.codes.dtype, device=DEV, generator=gen)
        m.codebooks.data = (torch.randn(m.codebooks.shape, device=DEV, generator=gen) / K ** 0.5).to(dtype)
        m.scales.data = (0.75 + 0.5 * torch.rand(m.scales.shape, device=DEV, generator=gen)).to(dtype)
        if bias:
            m.bias.data = torch.randn(m.bias.shape, device=DEV, generator=gen).to(dtype)
    return m


def dense_reference(m, x, go, x_grad):
    """fp32 autograd through W = scales * sum_k codebooks[k, codes[:, :, k]] (the reference project's training layer)."""
    cb = m.codebooks.detach().float().requires_grad_()
    sc = m.scales.detach().float().requires_grad_()
    b = m.bias.detach().float().requires_grad_() if m.bias is not None else None
    xr = x.detach().float().requires_grad_(x_grad)
    n = m.codebook_size
    c = m.codes.long() % n
    Wu = sum(cb[k, c[:, :, k], 0, :] for k in range(m.num_codebooks)).reshape(m.out_features, m.in_features)
    y = xr @ (Wu * sc.reshape(-1, 1)).t()
    if b is not None:
        y = y + b
    y.backward(go.float())
    return xr.grad, cb.grad, sc.grad, (b.grad if b is not None else None)


@gpu
@pytest.mark.parametrize("x_grad", [False, True], ids=["weights", "weights+input"])
@pytest.mark.parametrize("rows", [4, 300])
@pytest.mark.parametrize("scheme", [(1, 16, 8), (2, 8, 8), (8, 8, 8), (1, 16, 16), (3, 8, 8)],
                         ids=["1x16", "2x8", "8x8", "1x16g16", "3x8"])
def test_quantized_linear_trains_codebooks_scales_and_bias(scheme, rows, x_grad):
    K, nbits, g = scheme
    m = random_linear(1024, 512, K, nbits, g, seed=rows)
    for p in (m.codebooks, m.scales, m.bias):
        p.requires_grad_(True)
    gen = torch.Generator(DEV).manual_seed(1)
    x = torch.randn((rows, 1024), device=DEV, generator=gen).half().requires_grad_(x_grad)
    go = torch.randn((rows, 512), device=DEV, generator=gen).half()
    y = m(x)
    before = _cabi.launch_count()
    y.backward(go)
    torch.cuda.synchronize()
    if g == 8 and K != 3:  # one weight-gradient launch, plus the transposed GEMM for the input gradient
        assert _cabi.launch_count() - before == 1 + int(x_grad)
    rx, rcb, rs, rb = dense_reference(m, x, go, x_grad)
    assert rel(m.codebooks.grad, rcb) < 5e-3 and rel(m.scales.grad, rs) < 5e-3 and rel(m.bias.grad, rb) < 2e-3
    assert m.codebooks.grad.dtype == torch.float16 and m.scales.grad.shape == m.scales.shape
    assert (x.grad is not None) == x_grad and (not x_grad or rel(x.grad, rx) < 5e-3)
    assert m.codes.grad is None


@gpu
def test_frozen_weights_keep_the_inference_and_input_gradient_paths():
    m = random_linear(1024, 512, 2, 8)
    x = torch.randn((64, 1024), device=DEV).half()
    before = _cabi.launch_count()
    y = m(x)
    assert y.grad_fn is None and _cabi.launch_count() - before == 1
    x.requires_grad_(True)
    y = m(x)
    before = _cabi.launch_count()
    y.backward(torch.ones_like(y))
    assert _cabi.launch_count() - before == 1 and m.codebooks.grad is None and m.scales.grad is None
    m.scales.requires_grad_(True)
    with torch.no_grad():
        assert m(x).grad_fn is None


@gpu
def test_deterministic_mode_refuses_the_codebook_gradient():
    m = random_linear(1024, 512, 2, 8)
    m.codebooks.requires_grad_(True)
    x = torch.randn((64, 1024), device=DEV).half()
    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="not deterministic"):
            m(x).sum().backward()
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            m(x).sum().backward()
        assert any("not deterministic" in str(r.message) for r in rec) and m.codebooks.grad is not None
    finally:
        torch.use_deterministic_algorithms(False)
    m.codebooks.requires_grad_(False)
    m.scales.requires_grad_(True)
    try:
        torch.use_deterministic_algorithms(True)
        m(x).sum().backward()  # the scale gradient alone is deterministic
    finally:
        torch.use_deterministic_algorithms(False)
    assert m.scales.grad is not None


def lattice_module(K, nbits, fin, fout, seed, dtype=torch.float16):
    import aqlm_b200

    lin = lattice_linear(seed, fin, fout, K, nbits)
    m = aqlm_b200.QuantizedLinear(fin, fout, 8, 1, K, nbits, bias=True, device=DEV, dtype=dtype)
    with torch.no_grad():
        m.codes.data = torch.from_numpy(lin["codes"]).to(DEV)
        m.codebooks.data = to_dev(lin["codebooks"], dtype)
        m.scales.data = to_dev(lin["scales"], dtype)
        m.bias.data = torch.arange(fout, device=DEV, dtype=dtype) % 5 - 2
    return m


def _unfreeze(ms):
    for m in ms:
        for p in (m.codebooks, m.scales, m.bias):
            if p is not None:
                p.requires_grad_(True)


def _grads(ms):
    return [(m.codebooks.grad.clone(), m.scales.grad.clone(), m.bias.grad.clone() if m.bias is not None else None)
            for m in ms]


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_group_weight_grads_equal_the_members_run_alone(K, nbits):
    import copy

    import aqlm_b200

    members = [lattice_module(K, nbits, 256, o, seed=o) for o in (128, 64, 64)]
    alone = [copy.deepcopy(m) for m in members]
    grp = aqlm_b200.QuantizedLinearGroup(members)
    assert grp.fused
    _unfreeze(grp.members)
    _unfreeze(alone)
    rng = np.random.default_rng(3)
    x = to_dev(rng.integers(-X_MAX, X_MAX + 1, size=(96, 256)), torch.float16)
    gos = [to_dev(rng.integers(-X_MAX, X_MAX + 1, size=(96, m.out_features)), torch.float16) for m in members]
    for y, go in zip(grp(x), gos):
        y.backward(go)
    for m, go in zip(alone, gos):
        m(x).backward(go)
    for (a, b, c), (d, e, f) in zip(_grads(grp.members), _grads(alone)):
        assert torch.equal(a, d) and torch.equal(b, e) and torch.equal(c, f)
    # the gradients sit on the member parameters, whose data are views into the fused storage
    assert grp.members[0].scales.data_ptr() == grp._fused_scales.data_ptr()


@gpu
def test_mixtral_weight_grads_equal_the_members_run_alone():
    import copy

    from aqlm_b200.moe import QuantizedMixtralExperts

    E, H, I, T = 4, 64, 64, 24
    blk = QuantizedMixtralExperts(E, H, I, lambda t: t, 8, 1, 2, 8, device=DEV, dtype=torch.float16)
    rng = np.random.default_rng(11)
    with torch.no_grad():
        for e in range(E):
            for name, o in (("w1", I), ("w3", I), ("w2", H)):
                m = getattr(blk.expert(e), name)
                lin = lattice_linear(e * 10 + len(name) + o, m.in_features, m.out_features, 2, 8)
                m.codes.copy_(torch.from_numpy(lin["codes"]))
                m.codebooks.copy_(to_dev(np.clip(lin["codebooks"], -1, 1), torch.float16))
                m.scales.fill_(1.0)
    ref = copy.deepcopy(blk)
    members = lambda b: [getattr(b.expert(e), n) for e in range(E) for n in ("w1", "w2", "w3")]  # noqa: E731
    _unfreeze(members(blk))
    _unfreeze(members(ref))
    x = to_dev(rng.integers(-1, 2, size=(T, H)), torch.float16)
    idx = torch.from_numpy(rng.integers(0, E, size=(T, 1))).to(DEV)
    wts = torch.ones((T, 1), dtype=torch.float16, device=DEV)
    go = to_dev(rng.integers(-1, 2, size=(T, H)), torch.float16)
    blk(x, idx, wts).backward(go)
    # the same members, run one by one outside the block
    for e in range(E):
        tok = (idx[:, 0] == e).nonzero()[:, 0]
        if tok.numel() == 0:
            continue
        m = ref.expert(e)
        (m.w2(m.w1(x[tok]) * m.w3(x[tok])) * wts[tok]).backward(go[tok])
    for a, b in zip(members(blk), members(ref)):
        assert (a.codebooks.grad is None) == (b.codebooks.grad is None)
        if a.codebooks.grad is not None:
            assert torch.equal(a.codebooks.grad, b.codebooks.grad) and torch.equal(a.scales.grad, b.scales.grad)
    assert any(a.codebooks.grad is not None and a.codebooks.grad.abs().sum() > 0 for a in members(blk))


@gpu
def test_sharded_linear_refuses_trainable_weights():
    from aqlm_b200.sharded import ShardedQuantizedLinear

    m = ShardedQuantizedLinear(256, 64, 8, 1, 1, 16, bias=False, rank=0, world_size=1, device=DEV, dtype=torch.float16)
    m.scales.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="weight gradient"):
        m(torch.zeros((2, 256), device=DEV, dtype=torch.float16))


@gpu
def test_cuda_graph_replays_forward_and_weight_backward():
    m = lattice_module(2, 8, 512, 256, seed=9)
    _unfreeze([m])
    rng = np.random.default_rng(4)
    new = lambda *s: to_dev(rng.integers(-X_MAX, X_MAX + 1, size=s), torch.float16)  # noqa: E731
    sx, sg = new(64, 512), new(64, 256)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            m(sx).backward(sg)
    torch.cuda.current_stream().wait_stream(s)
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        m(sx).backward(sg)
    for _ in range(2):
        x2, g2 = new(64, 512), new(64, 256)
        sx.copy_(x2)
        sg.copy_(g2)
        graph.replay()
        torch.cuda.synchronize()
        replayed = _grads([m])[0]
        eager = copy_module_grads(m, x2, g2)
        for a, b in zip(replayed, eager):
            assert torch.equal(a, b)


def copy_module_grads(m, x, go):
    import copy

    e = copy.deepcopy(m)
    e.zero_grad(set_to_none=True)
    e(x).backward(go)
    return _grads([e])[0]


# ---- end to end (GPU) ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_tiny_llama_backward_fills_every_codebook_and_scale_grad(tmp_path, K, nbits):
    pytest.importorskip("transformers")
    import sys

    from transformers import AutoModelForCausalLM, LlamaForCausalLM

    import aqlm_b200
    from test_checkpoint import write_synthetic_checkpoint
    import transformers.quantizers.quantizer_aqlm as QA

    saved = {k: v for k, v in sys.modules.items() if k == "aqlm" or k.startswith("aqlm.")}
    had = QA.is_accelerate_available
    aqlm_b200.install_as_aqlm()
    QA.is_accelerate_available = lambda: True
    try:
        cfg, dense_sd, _ = write_synthetic_checkpoint(str(tmp_path / "m"), K, nbits, seed=4)
        model = AutoModelForCausalLM.from_pretrained(str(tmp_path / "m"), dtype=torch.float16).to(DEV)
    finally:
        QA.is_accelerate_available = had
        for k in [k for k in sys.modules if k == "aqlm" or k.startswith("aqlm.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    dense = LlamaForCausalLM(cfg)
    dense.load_state_dict({k: v.float() for k, v in dense_sd.items()})
    dense = dense.to(DEV)
    qlin = {n: m for n, m in model.named_modules() if isinstance(m, aqlm_b200.QuantizedLinear)}
    assert len(qlin) == 7 * cfg.num_hidden_layers
    for m in qlin.values():
        m.codebooks.requires_grad_(True)
        m.scales.requires_grad_(True)
    ids = torch.randint(0, cfg.vocab_size, (2, 12), device=DEV, generator=torch.Generator(DEV).manual_seed(0))
    model(ids, labels=ids).loss.backward()
    dense(ids, labels=ids).loss.backward()
    dmods = dict(dense.named_modules())
    for n, m in qlin.items():
        assert m.codebooks.grad is not None and m.scales.grad is not None, n
        # chain rule through W = s * Wu: dC from s * dW scattered over the codes, ds = row dot of dW and Wu
        dW = dmods[n].weight.grad.double()
        g = m.in_group_size
        c = m.codes.long() % m.codebook_size
        Wu = sum(m.codebooks.detach().double()[k, c[:, :, k], 0, :] for k in range(m.num_codebooks))
        ref_s = (dW.reshape(Wu.shape) * Wu).sum((1, 2))
        sD = (dW * m.scales.detach().double().reshape(-1, 1)).reshape(-1, g)
        ref_cb = torch.zeros((m.num_codebooks, m.codebook_size, g), dtype=torch.float64, device=DEV)
        for k in range(m.num_codebooks):
            ref_cb[k].index_add_(0, c[:, :, k].reshape(-1), sD)
        assert rel(m.scales.grad.reshape(-1), ref_s) < 3e-2, n
        assert rel(m.codebooks.grad.reshape(ref_cb.shape), ref_cb) < 3e-2, n
