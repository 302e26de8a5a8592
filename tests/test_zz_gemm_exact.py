"""Bit-exact tests of the GEMM, GEMV and LUT kernels on an integer lattice (runs last: `zz`, it sets AQLM_B200_* switches).

Every kernel here multiplies fp16 / bf16 operands and accumulates in fp32.  On lattice inputs -- small-integer activations
and codebooks, power-of-two scales, integer biases -- every product is exact and every partial sum is a multiple of
2^-e_hi well inside fp32's 24-bit significand, so the result does not depend on summation order, split count or tile
shape: it is the exact result rounded ONCE (to nearest even) to the output type.  The tests therefore assert equality of
every output element, and a failure prints where the wrong elements sit (output-row tile, batch tile), which is where an
indexing, swizzle, pipeline or split-K fault shows up.

The lattice (see `lattice_case`):
  codebooks  integers in [-CB_MAX, CB_MAX]            x / grad_out  integers in [-x_max, x_max] (X_MAX by default)
  codes      uniform over [0, 2^nbits), both extremes forced in, stored signed (oracle.pack_int_data)
  scales     2^-e per output row, e in [e_lo, e_hi], neighbouring rows always different
  bias       integers in [-B_MAX, B_MAX], neighbouring rows always different
`lattice_bounds` derives e_lo / e_hi from the shape alone (not from the drawn data) and asserts the exactness premise.

The forced plans go through the experiment switches AQLM_B200_GEMM_{TILE_M,KSPLIT,STAGES,GATHER_MODE}.  Tile height and
split count are observable through the workspace size the plan requests, and every forced case checks it; the stage
count and the gather mode are not observable from the host, so those cases only check the result.
"""
import contextlib
import ctypes
import math
import os
import zlib
from collections import Counter

import numpy as np
import pytest
import torch
from helpers import make_module, to_torch

from oracle import aqlm_oracle as O

DEV = "cuda:0"
gpu = pytest.mark.gpu

CB_MAX, X_MAX, B_MAX = 2, 3, 8
E_SPAN = 3                           # e_hi - e_lo: scales take 4 different values
WS_COUNTERS = 65536                  # counter region at the head of every workspace (plan.cuh kWsCountersBytes)
WS_TICKETS = 8192 * 4                # its split-K ticket words; the LUT GEMV's generation words (monotonic) follow
FINITE_MAX = {torch.float16: 65504.0, torch.bfloat16: float(torch.finfo(torch.bfloat16).max)}
INT_EXACT = {torch.float16: 2048, torch.bfloat16: 256}  # every integer up to this is exact in the type
DTYPES = [torch.float16, torch.bfloat16]
DT_ID = {torch.float16: "f16", torch.bfloat16: "bf16"}


# ---- lattice generator and exact reference (CPU) --------------------------------------------------------------------
def lattice_bounds(fin, fout, K, dtype, e_lo, e_hi, x_max=X_MAX, bias=True):
    """Assert, from the lattice bounds alone, that every kernel computes exactly.  Returns the worst-case magnitudes.

    forward   acc = sum_in x * W  (integers)            |acc| <= fin * x_max * K * CB_MAX      < 2^23
              y   = fmaf(acc, 2^-e, bias)               a multiple of 2^-e_hi, |y| < 2^(23 - e_hi), finite in dtype
    backward  A   = W * 2^-e (the scaled tile, in dtype) exact: |W| <= K * CB_MAX is a small integer
              gx  = sum_out go * A                      a multiple of 2^-e_hi, |gx| < 2^(23 - e_hi), finite in dtype
    """
    w_max = K * CB_MAX
    acc = fin * x_max * w_max
    y = acc * 2.0 ** -e_lo + (B_MAX if bias else 0)
    gx = fout * x_max * w_max * 2.0 ** -e_lo
    assert 0 <= e_lo <= e_hi <= 14, (e_lo, e_hi)  # 2^-e and W * 2^-e stay normal in fp16
    assert x_max <= INT_EXACT[dtype] and B_MAX <= INT_EXACT[dtype] and w_max <= INT_EXACT[dtype]
    assert acc < 2 ** 23, f"unscaled accumulator bound {acc} >= 2^23"
    for name, v in (("forward output", y), ("backward output", gx)):
        assert v < 2.0 ** (23 - e_hi), f"{name} bound {v} >= 2^{23 - e_hi}: not exact in fp32"
        assert v <= FINITE_MAX[dtype], f"{name} bound {v} overflows {dtype}"
    return dict(acc=acc, y=y, gx=gx)


def exponent_range(fin, fout, K, dtype, x_max=X_MAX, bias=True):
    """The smallest e_lo (and e_hi = e_lo + E_SPAN) for which `lattice_bounds` holds."""
    for e_lo in range(0, 12):
        try:
            lattice_bounds(fin, fout, K, dtype, e_lo, e_lo + E_SPAN, x_max, bias)
            return e_lo, e_lo + E_SPAN
        except AssertionError:
            continue
    raise AssertionError(f"no exact lattice for {fin}x{fout} K={K} {dtype} x_max={x_max}")


def _neighbours_differ(rng, n, lo, hi):
    """n integers in [lo, hi], each different from the previous one."""
    span = hi - lo + 1
    v = np.empty(n, dtype=np.int64)
    v[0] = rng.integers(lo, hi + 1)
    steps = rng.integers(1, span, size=n)
    for i in range(1, n):
        v[i] = lo + (v[i - 1] - lo + steps[i]) % span
    return v


def seed_of(*key) -> int:
    return zlib.crc32(repr(key).encode())


def lattice_case(seed, fin, fout, K, nbits, g=8, batch=1, bias=True, dtype=torch.float16, x_max=X_MAX,
                 unit_scales=False):
    """Seeded lattice inputs in the layout of oracle.make_case (float32 arrays, exact in fp16 and bf16)."""
    e_lo, e_hi = exponent_range(fin, fout, K, dtype, x_max, bias)
    rng = np.random.default_rng(seed)
    x = rng.integers(-x_max, x_max + 1, size=(batch, fin)).astype(np.float32)
    raw = rng.integers(0, 2 ** nbits, size=(fout, fin // g, K), dtype=np.int64)
    top = 2 ** nbits - 1
    raw[::7, 0, :] = top           # both extremes of the unsigned range, at fixed and at random positions
    raw[3::11, -1, :] = 0
    pos = rng.integers(0, raw.size, size=max(4, raw.size // 64))
    raw.reshape(-1)[pos[0::2]] = top
    raw.reshape(-1)[pos[1::2]] = 0
    codebooks = rng.integers(-CB_MAX, CB_MAX + 1, size=(K, 2 ** nbits, 1, g)).astype(np.float32)
    # the entries the extreme codes select are never all-zero vectors
    codebooks[:, 0, 0, :] = rng.choice([-2, -1, 1, 2], size=(K, g))
    codebooks[:, top, 0, :] = rng.choice([-2, -1, 1, 2], size=(K, g))
    e = np.zeros(fout, dtype=np.int64) if unit_scales else _neighbours_differ(rng, fout, e_lo, e_hi)
    scales = np.ldexp(np.float32(1.0), -e).astype(np.float32).reshape(fout, 1, 1, 1)
    b = _neighbours_differ(rng, fout, -B_MAX, B_MAX).astype(np.float32) if bias else None
    return dict(x=x, codes=O.pack_int_data(raw, nbits), codebooks=codebooks, scales=scales, bias=b, e_lo=e_lo, e_hi=e_hi)


def lattice_go(seed, batch, fout, x_max=X_MAX):
    return np.random.default_rng(seed).integers(-x_max, x_max + 1, size=(batch, fout)).astype(np.float32)


def exact_forward(case, x=None, dtype=np.float64):
    """y = x . (scales * W)^T + bias, exactly (float64; float32 is exact too under `lattice_bounds`)."""
    x = case["x"] if x is None else x
    return O.dequantize_gemm(x, case["codes"], case["codebooks"], case["scales"], case["bias"], dtype=dtype)


def exact_transposed(case, go, dtype=np.float64):
    """grad_in = (grad_out * scales) . W_unscaled, exactly."""
    nbits = int(case["codebooks"].shape[1]).bit_length() - 1
    W = O.dequantize_weight(O.unpack_int_data(case["codes"], nbits), case["codebooks"], None, dtype=dtype)
    return (np.asarray(go, dtype=dtype) * np.asarray(case["scales"], dtype=dtype).reshape(1, -1)) @ W


def round_to(ref, dtype):
    """Round an exact result once, to nearest even, to the kernel's output type; returned as float32."""
    r32 = np.asarray(ref, dtype=np.float32)
    assert np.array_equal(r32, ref), "reference is not exact in fp32"
    if dtype == torch.float16:
        return r32.astype(np.float16).astype(np.float32)
    return torch.from_numpy(r32).to(torch.bfloat16).float().numpy()


def assert_exact(y, ref, what, tile_m=None, n_tile=None, row_tile=128):
    """Every element equal; on failure, a map of where the mismatches are."""
    y = np.asarray(y, dtype=np.float32)
    ref = np.asarray(ref, dtype=np.float32)
    assert y.shape == ref.shape, (y.shape, ref.shape)
    bad = y != ref
    if not bad.any():
        return
    b, r = np.nonzero(bad)
    diff = np.abs(y.astype(np.float64) - ref.astype(np.float64))

    def hist(label, keys, limit=16):
        c = sorted(Counter(keys.tolist()).items())
        more = f" ... ({len(c)} groups)" if len(c) > limit else ""
        return f"  by {label}: " + ", ".join(f"{k}: {n}" for k, n in c[:limit]) + more

    rows = np.unique(r)
    lines = [f"{what}: {int(bad.sum())} of {bad.size} outputs differ, max |diff| = {np.nanmax(diff):g}",
             "  first (batch row, output row): " + ", ".join(f"({i}, {j})" for i, j in zip(b[:8], r[:8])),
             f"  {len(rows)} output rows affected: " + ", ".join(str(v) for v in rows[:16]) + (" ..." if len(rows) > 16 else "")]
    if tile_m:
        lines += [hist(f"output row // {tile_m}", r // tile_m), hist(f"output row % {tile_m}", r % tile_m)]
    if tile_m != row_tile:
        lines.append(hist(f"output row // {row_tile}", r // row_tile))
    if n_tile:
        lines.append(hist(f"batch row // {n_tile}", b // n_tile))
    pytest.fail("\n".join(lines))


# ---- plan arithmetic (plan.cuh gemm_plan / gemm_t_plan) ------------------------------------------------------------
def n_tile_of(batch):
    n = 16
    while n < 128 and n < batch:
        n <<= 1
    return n


def expected_ws(m_tiles, batch, ksplit):
    """Workspace bytes of a split-K plan: counters + [m_tiles][n_tiles][ksplit][n_tile][128] fp32 partials."""
    if ksplit <= 1:
        return 0
    nt = n_tile_of(batch)
    return WS_COUNTERS + m_tiles * math.ceil(batch / nt) * ksplit * nt * 128 * 4


# ---- device helpers -------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def tunables(**env):
    """Set AQLM_B200_<NAME> switches (None: unset) for the body, then restore the environment and re-read it."""
    from aqlm_b200 import _cabi

    keys = {f"AQLM_B200_{k.upper()}": v for k, v in env.items()}
    saved = {k: os.environ.get(k) for k in keys}
    try:
        for k, v in keys.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        _cabi.reload_tunables()
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        _cabi.reload_tunables()


def _weight(t, bias=True):
    from aqlm_b200.inference_kernels import cuda_kernel

    return cuda_kernel.make_weight(t["codes"], t["codebooks"], t["scales"].reshape(-1), t["bias"] if bias else None)


def _eager_workspace():
    from aqlm_b200.inference_kernels import cuda_kernel

    dev = torch.device(DEV)
    return cuda_kernel._WORKSPACES.get((dev.index, torch.cuda.current_stream(dev).cuda_stream))


def _assert_tickets_clean(what):
    """Split-K CTAs leave their ticket words at zero: graph replays and the next call rely on it."""
    ws = _eager_workspace()
    assert ws is not None, "split-K plan but no workspace"
    torch.cuda.synchronize()
    nz = int(torch.count_nonzero(ws[:WS_TICKETS]))
    assert nz == 0, f"{what}: {nz} nonzero bytes left in the split-K ticket words"


def run_forward(t, batch):
    """matmat_dequant; returns (y as float32 numpy, workspace bytes the plan asked for, kernel launches)."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    w = _weight(t)
    need = _cabi.lib().aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), batch)
    before = _cabi.launch_count()
    y = cuda_kernel.matmat_dequant(t["x"], t["codes"], t["codebooks"], t["scales"], t["bias"])
    launches = _cabi.launch_count() - before
    if need:
        _assert_tickets_clean("forward")
    return y.float().cpu().numpy(), need, launches


def run_transposed(t, go):
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    batch = go.shape[0]
    w = _weight(t, bias=False)
    need = _cabi.lib().aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(w), batch)
    before = _cabi.launch_count()
    gx = cuda_kernel.matmat_dequant_transposed(go, t["codes"], t["codebooks"], t["scales"], None)
    launches = _cabi.launch_count() - before
    if need:
        _assert_tickets_clean("transposed")
    return gx.float().cpu().numpy(), need, launches


def _eligible(fin, K, nbits, g=8):
    """The wgmma forward covers in_group 8, 8/16-bit codes, 1/2/4/8 codebooks, in % 64 == 0, 16-byte code rows."""
    return g == 8 and nbits in (8, 16) and K in (1, 2, 4, 8) and fin % 64 == 0 and (fin // 8 * K * nbits // 8) % 16 == 0


# ---- case lists (shared by the GPU tests and the CPU check of their bounds) -----------------------------------------
GEMM_SCHEMES = [(K, nbits) for nbits in (8, 16) for K in (1, 2, 4, 8)]
FWD_BATCHES = [7, 16, 17, 64, 100, 129, 300]
FWD_SHAPES = [(64, 1), (1088, 200), (1152, 456)]   # (in, out): one k-block / one row; 17 k-blocks; 18 k-blocks, out % 8 != 0
FWD_SHAPES_1X8 = [(128, 1), (1152, 456)]           # 1x8 needs in % 128 == 0 for a 16-byte code row stride


def _fwd_default_cases():
    out = []
    for K, nbits in GEMM_SCHEMES:
        for shape in (FWD_SHAPES_1X8 if (K, nbits) == (1, 8) else FWD_SHAPES):
            for dtype in DTYPES:
                for batch in FWD_BATCHES:
                    out.append(pytest.param(K, nbits, shape, dtype, batch,
                                            id=f"{K}x{nbits}-{shape[0]}x{shape[1]}-{DT_ID[dtype]}-bs{batch}"))
    return out


FORCED_TILE_M = [None, 128, 127, 97, 65, 64, 40, 32]
FORCED_KSPLIT = [None, 1, 2, 3, 5, 16, 999]
FORCED_STAGES = [None, 2, 3, 4]
FORCED_GATHER = [None, 0, 1]
FORCED_SHAPES = [(1152, 456), (1088, 200)]


def _fwd_forced_cases():
    """Every (tile_m, ksplit) pair for 1x16, 8x8 and 2x16; stages, gather mode, dtype, batch and shape rotate."""
    out, i = [], 0
    for K, nbits in [(1, 16), (8, 8), (2, 16)]:
        for tm in FORCED_TILE_M:
            for ks in FORCED_KSPLIT:
                st, gm = FORCED_STAGES[i % 4], FORCED_GATHER[i % 3]
                dtype, batch, shape = DTYPES[(i // 4) % 2], FWD_BATCHES[i % 7], FORCED_SHAPES[(i // 3) % 2]
                out.append(pytest.param(K, nbits, tm, ks, st, gm, dtype, batch, shape,
                                        id=f"{K}x{nbits}-tm{tm}-ks{ks}-st{st}-gm{gm}-{DT_ID[dtype]}-bs{batch}-in{shape[0]}"))
                i += 1
    return out


T_BATCHES = [1, 7, 64, 129, 300]
T_SHAPES = [(128, 8), (1088, 456), (640, 1032)]  # (in, out): one tile; in % 128 == 64, out % 64 == 8; 5 code tiles
T_SHAPES_1X8 = [(128, 8), (1152, 456), (640, 1032)]


def _t_cases():
    out = []
    for K, nbits in GEMM_SCHEMES:
        for shape in (T_SHAPES_1X8 if (K, nbits) == (1, 8) else T_SHAPES):
            for dtype in DTYPES:
                for batch in T_BATCHES:
                    out.append(pytest.param(K, nbits, shape, dtype, batch,
                                            id=f"{K}x{nbits}-{shape[0]}x{shape[1]}-{DT_ID[dtype]}-bs{batch}"))
    return out


T_FORCED_SHAPE = (1088, 1032)  # 17 k-blocks of out rows, ragged in both dimensions


def _t_forced_cases():
    out, i = [], 0
    for K, nbits in [(1, 16), (8, 16)]:
        for ks in [1, 2, 3, 5, 999]:
            for st in [2, 3]:
                dtype, batch = DTYPES[i % 2], T_BATCHES[i % 5]
                out.append(pytest.param(K, nbits, ks, st, dtype, batch, id=f"{K}x{nbits}-ks{ks}-st{st}-{DT_ID[dtype]}-bs{batch}"))
                i += 1
    return out


GEMV_SCHEMES = [(1, 16, 8), (1, 16, 16), (2, 8, 8), (1, 8, 8), (8, 8, 8), (4, 8, 8), (2, 12, 8), (3, 8, 8)]
GEMV_SHAPES = [(1024, 200), (4608, 136)]  # in <= 4096: cluster LUT form; above: the workspace LUT kernel
FULL_FWD = [(1, 16, (4096, 14336), torch.float16, 16), (1, 16, (4096, 14336), torch.float16, 256),
            (1, 16, (14336, 4096), torch.float16, 16), (1, 16, (14336, 4096), torch.float16, 256),
            (2, 8, (4096, 11008), torch.bfloat16, 64)]
FULL_T = (1, 16, (4096, 14336), torch.float16, 256)
PDL_A, PDL_B, PDL_C = (64, 256), (256, 200), (1088, 256)  # (in, out) of the chained layers; A's output feeds B and C
PDL_X_MAX = 64 * X_MAX * CB_MAX                            # A has unit scales and no bias: |y_A| <= in_A * 3 * 2


def _all_lattice_shapes():
    """(in, out, K, dtype, x_max, bias) of every lattice case the GPU tests build."""
    s = set()
    for K, nbits in GEMM_SCHEMES:
        for fin, fout in FWD_SHAPES + FWD_SHAPES_1X8 + FORCED_SHAPES + T_SHAPES + T_SHAPES_1X8 + [T_FORCED_SHAPE]:
            for dtype in DTYPES:
                s.add((fin, fout, K, dtype, X_MAX, True))
    for K, nbits, g in GEMV_SCHEMES:
        for fin, fout in GEMV_SHAPES + [(2048, 192), (1024, 512), (1024, 128)]:
            for dtype in DTYPES:
                s.add((fin, fout, K, dtype, X_MAX, True))
    for K, nbits, (fin, fout), dtype, _ in FULL_FWD + [FULL_T]:
        s.add((fin, fout, K, dtype, X_MAX, True))
    s.add((*PDL_A, 1, torch.float16, X_MAX, False))
    s.add((*PDL_B, 1, torch.float16, PDL_X_MAX, True))
    s.add((*PDL_C, 1, torch.float16, PDL_X_MAX, False))
    return sorted(s, key=repr)


# ==== CPU: the generator and the reference ===========================================================================
@pytest.mark.parametrize("fin,fout,K,dtype,x_max,bias", _all_lattice_shapes(), ids=lambda v: str(v) if not isinstance(v, torch.dtype) else DT_ID[v])
def test_lattice_bounds_hold(fin, fout, K, dtype, x_max, bias):
    """Every shape the GPU tests use has an exact lattice, with scales that really vary (E_SPAN > 0)."""
    e_lo, e_hi = exponent_range(fin, fout, K, dtype, x_max, bias)
    b = lattice_bounds(fin, fout, K, dtype, e_lo, e_hi, x_max, bias)
    assert e_hi - e_lo == E_SPAN and b["acc"] < 2 ** 23


def test_lattice_bounds_reject_inexact_choices():
    with pytest.raises(AssertionError, match="overflows"):
        lattice_bounds(14336, 4096, 1, torch.float16, 0, E_SPAN)  # 86016 > 65504
    with pytest.raises(AssertionError, match="not exact in fp32"):
        lattice_bounds(4096, 4096, 8, torch.bfloat16, 0, 14)
    with pytest.raises(AssertionError):
        lattice_bounds(64, 64, 1, torch.bfloat16, 0, 3, x_max=384)  # 383 is not a bf16 value
    assert exponent_range(14336, 4096, 1, torch.float16) == (1, 1 + E_SPAN)


def test_lattice_case_content():
    c = lattice_case(5, 1088, 200, 2, 8, batch=9)
    raw = O.unpack_int_data(c["codes"], 8)
    assert c["codes"].dtype == np.int8 and raw.min() == 0 and raw.max() == 255
    assert set(np.unique(c["codebooks"])) <= {-2, -1, 0, 1, 2} and set(np.unique(c["x"])) <= set(range(-3, 4))
    e = -np.log2(c["scales"].reshape(-1))
    assert np.all(e == np.round(e)) and np.all(np.diff(e) != 0) and len(np.unique(e)) == E_SPAN + 1
    assert np.all(np.abs(c["bias"]) <= B_MAX) and np.all(np.diff(c["bias"]) != 0)


def test_rounding_is_nearest_even():
    f16 = round_to(np.array([2049.0, 2051.0, 2050.0, -2049.0]), torch.float16)
    assert f16.tolist() == [2048.0, 2052.0, 2050.0, -2048.0]
    bf16 = round_to(np.array([257.0, 259.0, 258.0, -257.0]), torch.bfloat16)
    assert bf16.tolist() == [256.0, 260.0, 258.0, -256.0]


@pytest.mark.parametrize("K,nbits,g", GEMV_SCHEMES + [(4, 16, 8), (8, 16, 8)])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_exact_reference_matches_the_oracles(K, nbits, g, dtype):
    """On lattice inputs the float64 reference, the float32 numpy oracle and the C oracle (double accumulation) agree
    before and after rounding -- the exact reference is the oracle the golden vectors pin, not a new definition."""
    from oracle import c_oracle

    c = lattice_case(seed_of("oracles", K, nbits, g), 1088 if g == 8 else 1024, 456, K, nbits, g, batch=5, dtype=dtype)
    ref = exact_forward(c)
    for other in (exact_forward(c, dtype=np.float32),
                  c_oracle.dequantize_gemm(c["x"], c["codes"], c["codebooks"], c["scales"], c["bias"])):
        np.testing.assert_array_equal(np.asarray(other, np.float64), ref)
        np.testing.assert_array_equal(round_to(other, dtype), round_to(ref, dtype))
    go = lattice_go(seed_of("oracles-go", K, nbits), 5, 456)
    ref_t = exact_transposed(c, go)
    Wc = c_oracle.dequantize_weight(c["codes"], c["codebooks"], c["scales"])  # scaled rows
    np.testing.assert_array_equal((go.astype(np.float64) @ Wc.astype(np.float64)), ref_t)
    np.testing.assert_array_equal(exact_transposed(c, go, dtype=np.float32), ref_t)


# ==== GPU: forward wgmma GEMM ========================================================================================
def _check_forward(c, batch, dtype, what, tile_m=None):
    t = to_torch(c, DEV, dtype)
    y, need, launches = run_forward(t, batch)
    assert_exact(y, round_to(exact_forward(c), dtype), what, tile_m=tile_m, n_tile=n_tile_of(batch))
    return need, launches


@gpu
@pytest.mark.parametrize("K,nbits,shape,dtype,batch", _fwd_default_cases())
def test_forward_default_plan_exact(K, nbits, shape, dtype, batch):
    fin, fout = shape
    c = lattice_case(seed_of("fwd", K, nbits, shape, batch), fin, fout, K, nbits, batch=batch, dtype=dtype)
    assert _eligible(fin, K, nbits)
    need, launches = _check_forward(c, batch, dtype, f"{K}x{nbits} {fin}->{fout} bs={batch}")
    assert launches == 1, "the wgmma GEMM is one launch"
    if need:
        assert (need - WS_COUNTERS) % (math.ceil(batch / n_tile_of(batch)) * n_tile_of(batch) * 512) == 0


@gpu
@pytest.mark.parametrize("K,nbits,tile_m,ksplit,stages,gather,dtype,batch,shape", _fwd_forced_cases())
def test_forward_forced_plan_exact(K, nbits, tile_m, ksplit, stages, gather, dtype, batch, shape):
    """Forced tile height / split count (checked through the requested workspace size), stage count and gather mode
    (not observable from the host: only the result is checked)."""
    fin, fout = shape
    c = lattice_case(seed_of("forced", K, nbits, tile_m, ksplit, batch), fin, fout, K, nbits, batch=batch, dtype=dtype)
    with tunables(gemm_tile_m=tile_m, gemm_ksplit=ksplit, gemm_stages=stages, gemm_gather_mode=gather):
        need, launches = _check_forward(c, batch, dtype, f"{K}x{nbits} {fin}->{fout} bs={batch} tile_m={tile_m} "
                                        f"ksplit={ksplit} stages={stages} gather={gather}", tile_m=tile_m)
    assert launches == 1
    kblocks = fin // 64
    nt = n_tile_of(batch)
    per_tile_split = math.ceil(batch / nt) * nt * 128 * 4
    if ksplit is not None:
        ks = min(ksplit, kblocks)
        if tile_m is not None:
            assert need == expected_ws(math.ceil(fout / tile_m), batch, ks), (need, tile_m, ks)
        elif ks == 1:
            assert need == 0
        else:  # the plan's own tile height: m_tiles must be an integer between ceil(out/128) and ceil(out/32)
            m_tiles, rem = divmod(need - WS_COUNTERS, ks * per_tile_split)
            assert rem == 0 and math.ceil(fout / 128) <= m_tiles <= math.ceil(fout / 32), (need, ks)
    elif tile_m is not None and need:
        ks, rem = divmod(need - WS_COUNTERS, math.ceil(fout / tile_m) * per_tile_split)
        assert rem == 0 and 2 <= ks <= 16, (need, tile_m)


@gpu
@pytest.mark.parametrize("K,nbits,g,batch,dtype", [(1, 16, 8, 9, torch.float16), (1, 16, 8, 17, torch.bfloat16),
                                                   (2, 8, 8, 9, torch.bfloat16), (2, 8, 8, 17, torch.float16),
                                                   (1, 16, 16, 9, torch.float16), (1, 16, 16, 9, torch.bfloat16)])
def test_forward_gemv_fallback_exact(K, nbits, g, batch, dtype):
    """Layouts the wgmma kernel does not take (switched off, or in_group 16) run batch passes of the GEMV."""
    fin, fout = 1088, 200
    c = lattice_case(seed_of("fallback", K, nbits, g, batch), fin, fout, K, nbits, g, batch=batch, dtype=dtype)
    with tunables(disable_wgmma=1 if g == 8 else None):
        need, launches = _check_forward(c, batch, dtype, f"GEMV fallback {K}x{nbits} g={g} bs={batch}")
    assert need == 0 and launches >= 1


# ==== GPU: transposed (backward) wgmma GEMM ==========================================================================
def _check_transposed(c, go_np, dtype, what):
    t = to_torch(c, DEV, dtype)
    go = torch.from_numpy(go_np).to(dtype).to(DEV)
    gx, need, launches = run_transposed(t, go)
    assert launches == 1, "the backward must be ONE fused kernel (no dequant + dense fallback)"
    assert_exact(gx, round_to(exact_transposed(c, go_np), dtype), what, n_tile=n_tile_of(go_np.shape[0]))
    return need


@gpu
@pytest.mark.parametrize("K,nbits,shape,dtype,batch", _t_cases())
def test_transposed_exact(K, nbits, shape, dtype, batch):
    fin, fout = shape
    c = lattice_case(seed_of("t", K, nbits, shape, batch), fin, fout, K, nbits, batch=1, bias=False, dtype=dtype)
    go = lattice_go(seed_of("t-go", K, nbits, shape, batch), batch, fout)
    _check_transposed(c, go, dtype, f"transposed {K}x{nbits} W {fout}x{fin} bs={batch}")


@gpu
@pytest.mark.parametrize("K,nbits,ksplit,stages,dtype,batch", _t_forced_cases())
def test_transposed_forced_plan_exact(K, nbits, ksplit, stages, dtype, batch):
    fin, fout = T_FORCED_SHAPE
    c = lattice_case(seed_of("t-forced", K, nbits, ksplit, stages), fin, fout, K, nbits, bias=False, dtype=dtype)
    go = lattice_go(seed_of("t-forced-go", K, nbits, ksplit, stages), batch, fout)
    with tunables(gemm_ksplit=ksplit, gemm_stages=stages):
        need = _check_transposed(c, go, dtype, f"transposed {K}x{nbits} bs={batch} ksplit={ksplit} stages={stages}")
    ks = min(ksplit, math.ceil(fout / 64))
    assert need == expected_ws(math.ceil(fin / 128), batch, ks), (need, ks)


# ==== GPU: full size, every row ======================================================================================
@gpu
@pytest.mark.parametrize("K,nbits,shape,dtype,batch", FULL_FWD,
                         ids=[f"{k}x{n}-{s[0]}x{s[1]}-{DT_ID[d]}-bs{b}" for k, n, s, d, b in FULL_FWD])
def test_forward_full_size_exact(K, nbits, shape, dtype, batch):
    fin, fout = shape
    c = lattice_case(seed_of("full", K, nbits, shape, batch), fin, fout, K, nbits, batch=batch, dtype=dtype)
    t = to_torch(c, DEV, dtype)
    y, _, launches = run_forward(t, batch)
    assert launches == 1
    assert_exact(y, round_to(exact_forward(c, dtype=np.float32), dtype), f"{K}x{nbits} {fin}->{fout} bs={batch}",
                 n_tile=n_tile_of(batch))


@gpu
def test_transposed_full_size_exact():
    K, nbits, (fin, fout), dtype, batch = FULL_T
    c = lattice_case(seed_of("full-t"), fin, fout, K, nbits, bias=False, dtype=dtype)
    go = lattice_go(seed_of("full-t-go"), batch, fout)
    t = to_torch(c, DEV, dtype)
    gx, _, launches = run_transposed(t, torch.from_numpy(go).to(dtype).to(DEV))
    assert launches == 1
    assert_exact(gx, round_to(exact_transposed(c, go, dtype=np.float32), dtype), f"transposed W {fout}x{fin} bs={batch}",
                 n_tile=n_tile_of(batch))


# ==== GPU: workspace reuse, the C-ABI without (enough) workspace, and a chain without host sync =======================
@gpu
def test_split_counts_back_to_back_on_one_workspace():
    """ksplit 5 then 3 on the same persistent buffer: the second call never reads the first one's partials."""
    fin, fout, batch = 1152, 456, 100
    bufs = []
    for ks in (5, 3):
        c = lattice_case(seed_of("reuse", ks), fin, fout, 1, 16, batch=batch)
        with tunables(gemm_ksplit=ks, gemm_tile_m=128):
            need, _ = _check_forward(c, batch, torch.float16, f"ksplit={ks} after a larger split")
        assert need == expected_ws(math.ceil(fout / 128), batch, ks)
        bufs.append(_eager_workspace().data_ptr())
    assert bufs[0] == bufs[1], "both calls must share the workspace for this test to mean anything"


@gpu
@pytest.mark.parametrize("transposed", [False, True], ids=["forward", "transposed"])
def test_c_abi_short_or_no_workspace_runs_unsplit(transposed):
    """A workspace one byte smaller than the plan asks for is not used (no split; its partial region is untouched), and
    the entry points without a workspace run unsplit too; every result exact."""
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    fin, fout, batch, dtype = (1088, 1032, 64, torch.bfloat16) if transposed else (1152, 456, 64, torch.float16)
    c = lattice_case(seed_of("cabi", transposed), fin, fout, 1, 16, batch=batch, bias=not transposed, dtype=dtype)
    t = to_torch(c, DEV, dtype)
    w = _weight(t, bias=not transposed)
    st = torch.cuda.current_stream().cuda_stream
    if transposed:
        go_np = lattice_go(seed_of("cabi-go"), batch, fout)
        inp = torch.from_numpy(go_np).to(dtype).to(DEV)
        out = torch.empty((batch, fin), dtype=dtype, device=DEV)
        ref = round_to(exact_transposed(c, go_np), dtype)
        ws_bytes, call = L.aqlm_b200_matmat_dequant_transposed_workspace_bytes, L.aqlm_b200_matmat_dequant_transposed
        calls = [lambda ws, n: call(ctypes.byref(w), inp.data_ptr(), out.data_ptr(), batch, ws, n, st)]
    else:
        inp, out = t["x"], torch.empty((batch, fout), dtype=dtype, device=DEV)
        ref = round_to(exact_forward(c), dtype)
        ws_bytes, call = L.aqlm_b200_matmat_dequant_workspace_bytes, L.aqlm_b200_matmat_dequant_ws
        calls = [lambda ws, n: call(ctypes.byref(w), inp.data_ptr(), out.data_ptr(), batch, ws, n, st),
                 lambda ws, n: L.aqlm_b200_matmat_dequant(ctypes.byref(w), inp.data_ptr(), out.data_ptr(), batch, st)]
    with tunables(gemm_ksplit=5):
        need = ws_bytes(ctypes.byref(w), batch)
        assert need > WS_COUNTERS, "the forced split must ask for a workspace"
        ws = torch.zeros(need - 1, dtype=torch.uint8, device=DEV)
        ws[WS_COUNTERS:] = 0xA5
        for fn in calls:
            out.fill_(float("nan"))
            _cabi.check(fn(ws.data_ptr(), need - 1))
            torch.cuda.synchronize()
            assert_exact(out.float().cpu().numpy(), ref, "short workspace" if fn is calls[0] else "no workspace")
        assert int(torch.count_nonzero(ws[:WS_COUNTERS])) == 0
        assert bool((ws[WS_COUNTERS:] == 0xA5).all()), "a plan that did not fit wrote partials into the workspace"
        if transposed:
            out.fill_(float("nan"))
            _cabi.check(call(ctypes.byref(w), inp.data_ptr(), out.data_ptr(), batch, None, 0, st))
            torch.cuda.synchronize()
            assert_exact(out.float().cpu().numpy(), ref, "transposed, no workspace")


@gpu
def test_chained_layers_without_host_sync():
    """Programmatic dependent launch: layer A's output feeds layer B's GEMM and the transposed GEMM of layer C with no
    host synchronisation in between; checked once against the exact layers applied to A's output read back afterwards."""
    from aqlm_b200.inference_kernels import cuda_kernel

    batch, dtype = 64, torch.float16
    a = lattice_case(seed_of("pdl-a"), *PDL_A, 1, 16, batch=batch, bias=False, unit_scales=True)
    b = lattice_case(seed_of("pdl-b"), *PDL_B, 1, 16, x_max=PDL_X_MAX)
    cc = lattice_case(seed_of("pdl-c"), *PDL_C, 1, 16, bias=False, x_max=PDL_X_MAX)
    ta, tb, tc = (to_torch(v, DEV, dtype) for v in (a, b, cc))
    torch.cuda.synchronize()
    ya = cuda_kernel.matmat_dequant(ta["x"], ta["codes"], ta["codebooks"], ta["scales"], None)
    yb = cuda_kernel.matmat_dequant(ya, tb["codes"], tb["codebooks"], tb["scales"], tb["bias"])
    gc = cuda_kernel.matmat_dequant_transposed(ya, tc["codes"], tc["codebooks"], tc["scales"], None)
    torch.cuda.synchronize()
    ya_np = ya.float().cpu().numpy()
    assert_exact(ya_np, exact_forward(a), "layer A (integer-valued)")
    assert np.abs(ya_np).max() <= PDL_X_MAX
    assert_exact(yb.float().cpu().numpy(), round_to(exact_forward(b, x=ya_np), dtype), "layer B after A",
                 n_tile=n_tile_of(batch))
    assert_exact(gc.float().cpu().numpy(), round_to(exact_transposed(cc, ya_np), dtype), "transposed C after A",
                 n_tile=n_tile_of(batch))


# ==== GPU: GEMV and LUT paths ========================================================================================
@gpu
@pytest.mark.parametrize("shape", GEMV_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits,g", GEMV_SCHEMES)
def test_module_forward_small_batches_exact(K, nbits, g, dtype, shape):
    """QuantizedLinear.forward at batches 1..6 (GEMV, LUT GEMV and the per-row LUT loop), every scheme."""
    fin, fout = shape
    for batch in range(1, 7):
        c = lattice_case(seed_of("module", K, nbits, g, shape, batch), fin, fout, K, nbits, g, batch=batch, dtype=dtype)
        layer, t = make_module(c, DEV, dtype)
        with torch.no_grad():
            y = layer(t["x"]).float().cpu().numpy()
        assert_exact(y, round_to(exact_forward(c), dtype), f"module {K}x{nbits} g={g} {fin}->{fout} bs={batch}")


@gpu
@pytest.mark.parametrize("K,nbits,g", [(1, 16, 8), (2, 8, 8), (8, 8, 8), (1, 8, 8), (2, 12, 8), (1, 16, 16)])
@pytest.mark.parametrize("batch", [1, 2, 3, 6])
def test_partial_f32_is_the_unscaled_exact_sum(K, nbits, g, batch):
    from aqlm_b200.inference_kernels import cuda_kernel

    c = lattice_case(seed_of("partial", K, nbits, g, batch), 1024, 200, K, nbits, g, batch=batch, bias=False)
    t = to_torch(c, DEV)
    p = cuda_kernel.matmat_partial(t["x"], t["codes"], t["codebooks"]).cpu().numpy()
    assert p.dtype == np.float32
    ref = O.dequantize_gemm(c["x"], c["codes"], c["codebooks"], None, None, dtype=np.float64)
    assert_exact(p, ref, f"partial {K}x{nbits} bs={batch}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("batch", [1, 3])
def test_scale_bias_after_shard_sum_exact(dtype, batch):
    from aqlm_b200.inference_kernels import cuda_kernel

    c = lattice_case(seed_of("shards", batch), 2048, 192, 1, 16, batch=batch, dtype=dtype)
    t = to_torch(c, DEV, dtype)
    parts = 0
    for r in range(4):
        parts = parts + cuda_kernel.matmat_partial(t["x"][:, r * 512:(r + 1) * 512].contiguous(),
                                                   t["codes"][:, r * 64:(r + 1) * 64].contiguous(), t["codebooks"])
    y = cuda_kernel.scale_bias(parts, t["scales"], t["bias"], dtype)
    assert_exact(y.float().cpu().numpy(), round_to(exact_forward(c), dtype), f"scale_bias bs={batch}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("batch", [1, 3, 8])
def test_grouped_launch_exact(batch, dtype):
    from aqlm_b200.inference_kernels import cuda_kernel

    outs = [512, 128, 128]
    cases = [lattice_case(seed_of("grouped", i, batch), 1024, o, 1, 16, batch=batch, dtype=dtype) for i, o in enumerate(outs)]
    ts = [to_torch(c, DEV, dtype) for c in cases]
    y = cuda_kernel.matmat_grouped(ts[0]["x"], torch.cat([t["codes"] for t in ts]).contiguous(),
                                   torch.stack([t["codebooks"] for t in ts]).contiguous(),
                                   torch.cat([t["scales"] for t in ts]).contiguous(),
                                   torch.cat([t["bias"] for t in ts]).contiguous(), outs)
    ref = np.concatenate([exact_forward(c, x=cases[0]["x"]) for c in cases], axis=1)
    assert_exact(y.float().cpu().numpy(), round_to(ref, dtype), f"grouped bs={batch}")
