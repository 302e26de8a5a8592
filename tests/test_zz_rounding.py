"""Where every kernel rounds: a per-path rounding model, a lattice on which each rounding point really rounds, and
bit-exact checks of every entry point against the model (runs last: `zz`, it sets AQLM_B200_* switches).

The integer lattice of test_zz_gemm_exact proves indexing, pipelining and split-K, but nothing rounds on it before the
final conversion.  Here the data make every rounding point of a path change results, while every accumulation stays
exact, so the result of a kernel is one value and the model below names each rounding it performs.  rT rounds to the
output type T (fp16 or bf16, nearest even, with subnormals and overflow to +-inf), rf32 to fp32; Wsum = sum_k cb_k is
the K-codebook sum (exact in fp32 on every lattice here); s, b the row scale and bias.

  path                                                          model
  wgmma forward (plain, grouped, routed, any split)             y = rT(rf32(sum_j x * rT(Wsum) * s + b))
                                                                PARTIAL_F32: sum_j x * rT(Wsum)
  GEMV (vector, 1x16, generic, grouped, fused exchange), LUT,   y = rT(rf32(sum_j x * Wsum * s + b))      (W never rounded)
  cluster LUT                                                   PARTIAL_F32: sum_j x * Wsum
  wgmma transposed (plain, grouped, routed)                     gx = rT(sum_o go * rT(rf32(s * Wsum)))
  dequant, apply_scales 1 / 0                                   rT(rf32(s * Wsum)) / rT(Wsum)
  scale_bias, allreduce_scale_bias                              rT(rf32(p * s + b))
  weight gradient                                               grad_scales[r] = sum_j D[r, j] * rT(Wsum)[r, j],
                                                                grad_codebooks = sum s * D,   D = grad_out^T . x
The wgmma kernels feed T operands to the tensor core, so for K >= 2 they round W where the GEMV and LUT kernels do not:
the same row computed on either side of the GEMV / GEMM batch boundary may differ by that rounding.

The rounding lattice (`rounding_case`):
  codebooks  sigma_i * m * 2^cb_exp, m an integer in [2^(p-1), 2^p) (p: T's significand bits), sigma_i = +-1 per element
             position i: every entry is exact in T, the K-sums never cancel, and for K >= 2 they exceed T's significand
  scales     T values with full significands, exponents in [s_lo, s_hi] (neighbouring rows differ)
  bias       T values with full significands, |b| in [2^b_exp, 2^(b_exp + 1)), random signs: rounding the scaled sum
             before adding b changes results
  x          integers in [-x_max, x_max], x_nnz nonzeros per row
  grad_out   go_nnz entries of +-1 / +-2 per row, one of them in the last (ragged) 64-row block of out rows
`rounding_bounds` derives from these windows alone that every accumulation is exact and every output finite (or, for
the overflow variant, that the fp32 value is finite).  A CPU test runs it over every case the GPU tests build, and
`test_model_has_teeth` checks that each rounding point, mutated, changes results of every case it applies to.

GPU tests call the C-ABI with NaN-filled outputs between guard bytes, and with a test-owned workspace whose partial
region is NaN-filled: a partial that a call reads without having written shows up in the result.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from test_zz_gemm_exact import DT_ID, WS_COUNTERS, WS_TICKETS, _neighbours_differ, assert_exact, n_tile_of, seed_of, tunables

from oracle import aqlm_oracle as O

DEV = "cuda:0"
gpu = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
DTYPES = [F16, BF16]
# significand bits, smallest normal exponent, largest finite value
FMT = {F16: (11, -14, 65504.0), BF16: (8, -126, float(torch.finfo(torch.bfloat16).max)),
       torch.float32: (24, -126, float(np.finfo(np.float32).max))}
TEETH = 8        # a mutated rounding point must change at least this many outputs of a case
GUARD = 256      # guard bytes on each side of every output


# ==== the rounding model (CPU, float64) ==============================================================================
def round_to(v, fmt):
    """Round float64 values to nearest even in a binary format (significand bits, subnormals, overflow to +-inf)."""
    p, emin, vmax = FMT[fmt]
    v = np.asarray(v, dtype=np.float64)
    _, ex = np.frexp(v)
    e = np.maximum(ex - 1, emin)                      # exponent of the value's binade (subnormals: emin)
    ulp = np.ldexp(1.0, e - (p - 1))
    r = np.round(v / ulp) * ulp                       # np.round: half to even; v / ulp is exact
    return np.where(np.abs(r) > vmax, np.copysign(np.inf, v), r)


def rT(v, dtype):
    return round_to(v, dtype)


def rf32(v):
    return round_to(v, torch.float32)


def exact_sum(a, b, what):
    """a + b in float64, asserted exact (Fast2Sum: the error term of the larger minus the smaller is zero)."""
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    y = a + b
    big = np.where(np.abs(a) >= np.abs(b), a, b)
    small = np.where(np.abs(a) >= np.abs(b), b, a)
    assert np.all(np.isfinite(y)) and np.all(small - (y - big) == 0), f"{what} is not exact in float64"
    return y


def wsum(c, rounded=False, sum_in_T=False):
    """W [out, in] = sum_k cb_k (exact), rT(sum) (the wgmma operand), or summed in T one codebook at a time."""
    cb, raw, dtype = c["cb"], c["raw"], c["dtype"]
    K = cb.shape[0]
    parts = [cb[k][raw[:, :, k]][:, :, 0, :] for k in range(K)]  # [out, groups, g]
    w = parts[0]
    for k in range(1, K):
        w = rT(w + parts[k], dtype) if sum_in_T else w + parts[k]
    w = w.reshape(raw.shape[0], -1)
    return rT(w, dtype) if rounded else w


def model_forward(c, x=None, w=None, gemm=True, partial=False, bias_after_T=False):
    """wgmma forward (gemm) or GEMV / LUT contract; w overrides W (mutations)."""
    x = c["x"] if x is None else x
    w = wsum(c, rounded=gemm) if w is None else w
    acc = x @ w.T
    assert np.all(np.abs(acc) < 2.0 ** 24 * c["unit"]), "accumulator leaves the exact lattice"
    if partial:
        return acc
    return model_scale_bias(acc, c["s"], c["b"], c["dtype"], bias_after_T)


def model_scale_bias(p, s, b, dtype, bias_after_T=False):
    b = 0.0 if b is None else b
    if bias_after_T:  # the scaled sum rounded to T before the bias is added
        return rT(rf32(rT(rf32(p * s), dtype) + b), dtype)
    # p * s: |p| < 2^24 lattice units times a T value: at most 35 significant bits, exact in float64
    return rT(rf32(exact_sum(p * s, b, "p * s + b")), dtype)


def model_a_operand(c, w=None, scale_in_T=False, unrounded=False):
    """A operand of the transposed kernel: rT(rf32(s * Wsum)) per out row."""
    w = wsum(c) if w is None else w
    s = c["s"][:, None]
    if unrounded:
        return s * w
    if scale_in_T:
        return rT(s * rT(w, c["dtype"]), c["dtype"])
    return rT(rf32(s * w), c["dtype"])


def model_transposed(c, go, a=None):
    exact_a = a is None
    a = model_a_operand(c) if a is None else a
    gx = go @ a
    if exact_a:
        assert np.array_equal(rf32(gx), gx), "transposed sum not exact in fp32"
    return rT(gx, c["dtype"])


def model_dequant(c, apply_scales, scale_in_T=False):
    w = wsum(c)
    if not apply_scales:
        return rT(w, c["dtype"])
    return model_a_operand(c, w, scale_in_T=scale_in_T)


def model_wgrad(c, go, wu_rounded=True):
    D = go.T @ c["x"]                                         # [out, in]
    gs = (D * wsum(c, rounded=wu_rounded)).sum(axis=1)
    K, n, _, g = c["cb"].shape
    gcb = np.zeros((K, n, g))
    sD = (c["s"][:, None] * D).reshape(D.shape[0], -1, g)     # [out, groups, g]
    for k in range(K):
        np.add.at(gcb[k], c["raw"][:, :, k].reshape(-1), sD.reshape(-1, g))
    return gs, gcb


# ==== the rounding lattice (CPU) =====================================================================================
def _windows(fin, K, dtype, variant="plain", transposed=False):
    """Windows of one case: exponents of codebook units, scales and bias, and the activation / grad_out density."""
    p = FMT[dtype][0]
    x_max = 2
    x_nnz = min(fin, 2 ** 23 // (x_max * K * 2 ** p))
    w = dict(cb_exp=0, s_lo=-12, s_hi=-9, x_max=x_max, x_nnz=x_nnz, go_nnz=4, go_max=2, overflow=False)
    if variant == "bf16-huge":       # outputs far above fp16's largest value
        w.update(cb_exp=20, s_lo=-2, s_hi=1)
    elif variant == "bf16-tiny":     # outputs far below fp16's smallest subnormal, far above 2^-126
        w.update(cb_exp=-40, s_lo=-12, s_hi=-9)
    elif variant == "f16-subnormal":  # subnormal scales, subnormal and normal outputs
        w.update(cb_exp=-10, s_lo=-20, s_hi=-17)
    elif variant == "f16-overflow":  # outputs on both sides of 65504
        w.update(s_lo=0, s_hi=0, overflow=True)
        w["s_lo"] = w["s_hi"] = 16 - int(math.log2(math.sqrt(x_nnz) * x_max * K * 2 ** p))
    typ = math.sqrt(w["x_nnz"]) * K * 2 ** (p - 1) * 2.0 ** w["cb_exp"]  # typical |acc|
    w["b_exp"] = int(math.floor(math.log2(typ))) + w["s_lo"]
    return w


def rounding_bounds(fin, fout, K, dtype, w):
    """Assert, from shape, dtype and windows alone, that every accumulation the kernels do is exact in fp32 (inside the
    tensor core too: the data are an integer lattice scaled by a power of two) and that every output is finite."""
    p, emin, vmax = FMT[dtype]
    unit = 2.0 ** w["cb_exp"]
    cb_max = (2 ** p - 1) * unit
    assert cb_max <= vmax and (2 ** (p - 1)) * unit >= 2.0 ** emin, "codebook entries are not normal T values"
    w_max = K * 2 ** p * unit                                    # |Wsum| and |rT(Wsum)|
    acc = w["x_nnz"] * w["x_max"] * w_max
    assert acc < 2.0 ** 24 * unit, f"forward accumulator {acc / unit} units >= 2^24"
    s_max = 2.0 ** (w["s_hi"] + 1)
    assert s_max <= vmax and w["s_lo"] >= emin - (p - 1) + 3, "scales out of T's range"
    y = acc * s_max + 2.0 ** (w["b_exp"] + 1)
    if w["overflow"]:
        assert y < FMT[torch.float32][2] / 2, "overflow variant: fp32 value not finite"
    else:
        assert y <= vmax, f"forward output bound {y} overflows {dtype}"
    # acc * s + b exact in float64: lowest bit of the product vs the bias's, against the top
    lo = min(unit * 2.0 ** (max(w["s_lo"], emin) - (p - 1)), 2.0 ** (max(w["b_exp"], emin) - (p - 1)))
    assert y / lo < 2.0 ** 52, "acc * s + b not exact in float64"
    # transposed: A = rT(s * Wsum) spans [s_lo * K 2^(p-1), s_max * K 2^p] units; a gx element adds go_nnz of them
    a_min = 2.0 ** w["s_lo"] * K * 2 ** (p - 1) * unit
    a_lo = 2.0 ** (max(math.floor(math.log2(a_min)), emin) - (p - 1))
    gx = w["go_nnz"] * w["go_max"] * s_max * w_max
    if not w["overflow"]:
        assert gx <= vmax and s_max * w_max <= vmax, f"transposed bound {gx} overflows {dtype}"
        assert gx / a_lo < 2.0 ** 24, "transposed sum not exact in fp32"
        assert a_min >= 2.0 ** -126, "A operand below fp32's normal range"
    return dict(acc=acc, y=y, gx=gx)


def _full_sig(rng, n, lo, hi, dtype, signed=False):
    """n T values with full significands and exponents in [lo, hi] (neighbours differ when hi > lo)."""
    p = FMT[dtype][0]
    e = _neighbours_differ(rng, n, lo, hi) if hi > lo else np.full(n, lo)
    m = 1.0 + rng.integers(1, 2 ** (p - 1), size=n) / 2.0 ** (p - 1)  # never a power of two
    v = np.ldexp(m, e)
    if signed:
        v *= rng.choice([-1.0, 1.0], size=n)
    return rT(v, dtype)


def rounding_case(seed, fin, fout, K, nbits, dtype, batch=1, g=8, variant="plain", bias=True, transposed=False,
                  n_cb_sets=1):
    """Seeded rounding-lattice inputs (float64 arrays of T values); n_cb_sets: stacked codebooks (grouped / routed)."""
    w = _windows(fin, K, dtype, variant, transposed)
    rounding_bounds(fin, fout, K, dtype, w)
    p = FMT[dtype][0]
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 2 ** nbits, size=(fout, fin // g, K), dtype=np.int64)
    top = 2 ** nbits - 1
    raw[::7, 0, :] = top
    raw[3::11, -1, :] = 0
    unit = 2.0 ** w["cb_exp"]
    sigma = rng.choice([-1.0, 1.0], size=g)
    cb = rng.integers(2 ** (p - 1), 2 ** p, size=(n_cb_sets, K, 2 ** nbits, 1, g)) * sigma * unit
    x = np.zeros((batch, fin))
    for r in range(batch):
        pos = rng.choice(fin, size=w["x_nnz"], replace=False)
        x[r, pos] = rng.integers(-w["x_max"], w["x_max"] + 1, size=w["x_nnz"])
    s = _full_sig(rng, fout, w["s_lo"], w["s_hi"], dtype)
    b = _full_sig(rng, fout, w["b_exp"], w["b_exp"], dtype, signed=True) if bias else None
    c = dict(x=x, raw=raw, cb=cb[0], cbs=cb, s=s, b=b, dtype=dtype, nbits=nbits, g=g, unit=unit, win=w)
    assert all(np.array_equal(rT(a, dtype), a) for a in (cb, x, s) + ((b,) if bias else ()))
    return c


def sparse_go(seed, batch, fout, w):
    """go_nnz entries of +-1 / +-2 per row; row r's first entry sits in the last 64-row block of out rows."""
    rng = np.random.default_rng(seed)
    go = np.zeros((batch, fout))
    last = (fout - 1) // 64 * 64
    for r in range(batch):
        pos = rng.choice(fout, size=w["go_nnz"], replace=False)
        pos[0] = rng.integers(last, fout)
        go[r, pos] = rng.choice([-2.0, -1.0, 1.0, 2.0], size=w["go_nnz"])
    return go


def _segment(c, seg_of_row):
    """A per-row view of W when rows use different codebook sets (grouped: set per segment; routed: per expert)."""
    parts = []
    for i in range(c["cbs"].shape[0]):
        ci = dict(c, cb=c["cbs"][i])
        parts.append(wsum(ci))
    w = np.empty_like(parts[0])
    for o in range(w.shape[0]):
        w[o] = parts[seg_of_row[o]][o]
    return w


# ==== case lists (shared by the GPU tests, the bounds test and the teeth test) ========================================
SCHEMES = [(K, nbits) for nbits in (8, 16) for K in (1, 2, 4, 8)]
FWD_SHAPE = (512, 200)      # 8 k-blocks; out % 8 != 0
FWD_BATCHES = [7, 17, 129, 300]
T_SHAPE = (384, 456)        # 3 in tiles (1x8 code rows must be 16-byte multiples); out = 7 * 64 + 8: a ragged last block
T_BATCHES = [1, 7, 64, 129]
FORCED = [(128, 1), (97, 3), (40, 16), (None, 3)]           # (tile_m, ksplit) of the forward
FORCED_SCHEMES = [(1, 16), (2, 8), (8, 8)]
FORCED_SHAPE = (1024, 200)  # 16 k-blocks: ksplit 16 is one k-block per split
T_KSPLIT = [1, 3, 999]
VARIANTS = {BF16: ["bf16-huge", "bf16-tiny"], F16: ["f16-subnormal", "f16-overflow"]}

# (path, K, nbits, g, fin, batch, switches): each lands on its kernel by the selection rules of capi.cu
GEMV_CASES = [
    ("cluster-lut", 1, 8, 8, 1024, 1, {}), ("cluster-lut", 2, 8, 8, 4096, 1, {}),
    ("ws-lut", 4, 8, 8, 1024, 1, {}), ("ws-lut", 8, 8, 8, 1024, 1, {}), ("ws-lut", 2, 8, 8, 4608, 1, {}),
    ("lut-row-loop", 2, 8, 8, 1024, 3, {}), ("lut-row-loop", 8, 8, 8, 1024, 2, {}),
    ("vec", 2, 8, 8, 1024, 5, {}), ("vec", 4, 8, 8, 1024, 4, {}), ("vec", 8, 8, 8, 1024, 6, {}),
    ("vec", 2, 8, 8, 1024, 1, {"disable_lut": 1}),
    ("1x16", 1, 16, 8, 1024, 1, {}), ("1x16", 1, 16, 8, 1024, 3, {}), ("vec-g16", 1, 16, 16, 1024, 2, {}),
    ("generic", 2, 12, 8, 1024, 2, {}), ("generic", 3, 8, 8, 1024, 3, {}), ("generic", 1, 16, 8, 1032, 1, {}),
    ("generic", 2, 8, 8, 1024, 4, {"force_generic": 1}),
    ("gemv-passes", 2, 8, 8, 1024, 11, {"disable_wgmma": 1}), ("gemv-passes", 4, 16, 8, 1024, 9, {"disable_wgmma": 1}),
]
GEMV_OUT = 200
DEQ_CASES = [(1, 16, 8), (2, 8, 8), (8, 16, 8), (2, 8, 16)]
WGRAD_SCHEMES = [(1, 16), (2, 8), (4, 16), (8, 8)]
WGRAD_SHAPE, WGRAD_BATCH = (256, 136), 64


def _fwd_cases():
    out, i = [], 0
    for K, nbits in SCHEMES:
        for dtype in DTYPES:
            out.append(pytest.param(K, nbits, dtype, FWD_BATCHES[i % 4], None, None,
                                    id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{FWD_BATCHES[i % 4]}"))
            i += 1
    for K, nbits in FORCED_SCHEMES:
        for tm, ks in FORCED:
            dtype, batch = DTYPES[i % 2], FWD_BATCHES[i % 4]
            out.append(pytest.param(K, nbits, dtype, batch, tm, ks, id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}-tm{tm}-ks{ks}"))
            i += 1
    return out


def _t_cases():
    out, i = [], 0
    for K, nbits in SCHEMES:
        for dtype in DTYPES:
            out.append(pytest.param(K, nbits, dtype, T_BATCHES[i % 4], None, id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{T_BATCHES[i % 4]}"))
            i += 1
    for K, nbits in [(1, 16), (8, 8)]:
        for ks in T_KSPLIT:
            dtype, batch = DTYPES[i % 2], T_BATCHES[i % 4]
            out.append(pytest.param(K, nbits, dtype, batch, ks, id=f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}-ks{ks}"))
            i += 1
    return out


def _variant_cases():
    return [pytest.param(v, d, id=v) for d in DTYPES for v in VARIANTS[d]]


def _all_cases():
    """(name, case, go or None, [mutation names]) of every GPU case, built on the CPU."""
    out = []
    for prm in _fwd_cases():
        K, nbits, dtype, batch, tm, ks = prm.values
        fin = FORCED_SHAPE[0] if (tm, ks) != (None, None) else FWD_SHAPE[0]
        out.append(("fwd " + prm.id, rounding_case(seed_of("fwd", prm.id), fin, FWD_SHAPE[1], K, nbits, dtype, batch), None,
                    "gemm"))
    for prm in _t_cases():
        K, nbits, dtype, batch, ks = prm.values
        c = rounding_case(seed_of("t", prm.id), *T_SHAPE, K, nbits, dtype, bias=False, transposed=True)
        out.append(("t " + prm.id, c, sparse_go(seed_of("t-go", prm.id), batch, T_SHAPE[1], c["win"]), "transposed"))
    for path, K, nbits, g, fin, batch, sw in GEMV_CASES:
        for dtype in DTYPES:
            name = f"gemv {path} {K}x{nbits} g{g} in{fin} bs{batch} {DT_ID[dtype]}"
            out.append((name, rounding_case(seed_of("gemv", name), fin, GEMV_OUT, K, nbits, dtype, batch, g), None, "gemv"))
    for v in [v for d in DTYPES for v in VARIANTS[d]]:
        dtype = BF16 if v.startswith("bf16") else F16
        out.append((f"variant {v} gemm", rounding_case(seed_of("var", v), 512, 200, 2, 8, dtype, 17, variant=v), None, "gemm"))
        for batch in (1, 5):
            out.append((f"variant {v} gemv bs{batch}",
                        rounding_case(seed_of("var-gemv", v, batch), 1024, 200, 2, 8, dtype, batch, variant=v), None, "gemv"))
        if v != "f16-overflow":
            c = rounding_case(seed_of("var-t", v), *T_SHAPE, 2, 8, dtype, bias=False, transposed=True, variant=v)
            out.append((f"variant {v} t", c, sparse_go(seed_of("var-t-go", v), 7, T_SHAPE[1], c["win"]), "transposed"))
    return out


# ==== CPU: the model's rounding, the bounds, the teeth ================================================================
def test_round_to_matches_the_hardware_formats():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 20, size=4000),
                        [65504.0, 65519.99, 65520.0, -65520.0, 2.0 ** -25, 3 * 2.0 ** -26, 2049.0, 2051.0]])
    with np.errstate(over="ignore"):  # the values past 65504 become inf, which is the point
        np.testing.assert_array_equal(rT(v, F16), v.astype(np.float16).astype(np.float64))
    np.testing.assert_array_equal(rf32(v), v.astype(np.float32).astype(np.float64))
    v32 = rf32(v * 2.0 ** 60)  # bf16: torch rounds fp32 input once
    np.testing.assert_array_equal(rT(v32, BF16), torch.from_numpy(v32.astype(np.float32)).to(BF16).double().numpy())
    assert rT(np.array([257.0, 259.0]), BF16).tolist() == [256.0, 260.0]


@pytest.mark.parametrize("variant,dtype", [("plain", F16), ("plain", BF16)] + [(v, d) for d in DTYPES for v in VARIANTS[d]])
def test_bounds_hold_for_every_shape(variant, dtype):
    """Every (shape, scheme) the GPU tests build has a lattice whose bounds hold (rounding_case asserts them)."""
    shapes = {FWD_SHAPE, FORCED_SHAPE, T_SHAPE, WGRAD_SHAPE, (512, 200)} | {(fin, GEMV_OUT) for _, _, _, _, fin, _, _ in GEMV_CASES}
    for fin, fout in sorted(shapes):
        for K in (1, 2, 3, 4, 8):
            rounding_bounds(fin, fout, K, dtype, _windows(fin, K, dtype, variant))
            if variant != "f16-overflow":
                rounding_bounds(fin, fout, K, dtype, _windows(fin, K, dtype, variant, transposed=True))


def test_bounds_reject_inexact_windows():
    w = _windows(512, 8, F16)
    with pytest.raises(AssertionError, match="accumulator"):
        rounding_bounds(512, 200, 8, F16, dict(w, x_nnz=512, x_max=3))
    with pytest.raises(AssertionError, match="overflows"):
        rounding_bounds(512, 200, 8, F16, dict(w, s_lo=2, s_hi=5))
    with pytest.raises(AssertionError, match="transposed sum"):
        rounding_bounds(512, 200, 8, F16, dict(w, s_lo=-20, s_hi=-9, go_nnz=64))


def _mutations(c, go, kind):
    """name -> mutated model of the case; only the mutations that change what the path computes for this scheme."""
    K, dtype = c["cb"].shape[0], c["dtype"]
    m = {}
    if kind in ("gemm", "gemv"):
        gemm = kind == "gemm"
        m["bias added after rounding to T"] = lambda: model_forward(c, gemm=gemm, bias_after_T=True)
        if K >= 2:
            m["the other path's W contract"] = lambda: model_forward(c, gemm=not gemm)
        if gemm and K >= 4:
            m["K-sum rounded to T after each add"] = lambda: model_forward(c, w=wsum(c, sum_in_T=True))
    elif kind == "transposed":
        m["A not rounded"] = lambda: model_transposed(c, go, model_a_operand(c, unrounded=True))
        if K >= 2:
            m["rounded before the scale"] = lambda: model_transposed(c, go, model_a_operand(c, scale_in_T=True))
    return m


def _truth(c, go, kind):
    if kind == "transposed":
        return model_transposed(c, go)
    return model_forward(c, gemm=kind == "gemm")


def test_model_has_teeth():
    """Each mutated rounding point changes at least TEETH outputs of every case it applies to, and the overflow and
    subnormal variants really produce +-inf and subnormal outputs."""
    weak = []
    for name, c, go, kind in _all_cases():
        truth = _truth(c, go, kind)
        for mname, f in _mutations(c, go, kind).items():
            n = int(np.sum(f() != truth))
            if n < TEETH:
                weak.append(f"{name}: '{mname}' changes {n} outputs")
        v = c["win"]
        if v["overflow"]:
            assert np.isinf(truth).any() and (np.abs(truth[np.isfinite(truth)]) > 32768).any(), name
        if "subnormal" in name:
            assert ((truth != 0) & (np.abs(truth) < 2.0 ** -14)).any(), name
        if "tiny" in name:
            assert np.abs(truth).max() < 2.0 ** -24 and np.abs(truth[truth != 0]).min() > 2.0 ** -126, name
        if "huge" in name:
            assert np.abs(truth).max() > 65504, name
    assert not weak, "\n".join(weak)


def test_teeth_of_dequant_scale_bias_and_weight_grad():
    for K, nbits, g in DEQ_CASES:
        for dtype in DTYPES:
            c = rounding_case(seed_of("deq", K, nbits, g, DT_ID[dtype]), 512, 136, K, nbits, dtype, g=g, bias=False)
            if K >= 2:
                assert np.sum(model_dequant(c, 1, scale_in_T=True) != model_dequant(c, 1)) >= TEETH
                assert np.sum(model_dequant(c, 0) != wsum(c)) >= TEETH
    for K, nbits in WGRAD_SCHEMES:
        for dtype in DTYPES:
            c, go = _wgrad_case(K, nbits, dtype)
            if K >= 2:
                assert np.sum(model_wgrad(c, go)[0] != model_wgrad(c, go, wu_rounded=False)[0]) >= TEETH
    for dtype in DTYPES:
        c, p = _scale_bias_case(dtype, 3)
        assert np.sum(model_scale_bias(p, c["s"], c["b"], dtype, True) != model_scale_bias(p, c["s"], c["b"], dtype)) >= TEETH


def _wgrad_case(K, nbits, dtype):
    """x in {-1, 0, 1} and one +-1 of grad_out per out row, so |D| <= 1; one scale exponent e, so every s * D of the
    codebook gradient is a multiple of 2^(e - p + 1) below 2^(e + 1)."""
    fin, fout = WGRAD_SHAPE
    c = rounding_case(seed_of("wgrad", K, nbits, DT_ID[dtype]), fin, fout, K, nbits, dtype, WGRAD_BATCH, bias=False)
    rng = np.random.default_rng(seed_of("wgrad-s", K, nbits))
    c["x"] = np.sign(c["x"])
    c["s"] = _full_sig(rng, fout, -4, -4, dtype)
    go = np.zeros((WGRAD_BATCH, fout))
    go[rng.integers(0, WGRAD_BATCH, size=fout), np.arange(fout)] = rng.choice([-1.0, 1.0], size=fout)
    p = FMT[dtype][0]
    assert fin * K * 2 ** p < 2 ** 24, "grad_scales not exact in fp32"
    assert fout * fin // 8 * 2 ** p < 2 ** 24, "grad_codebooks not exact in fp32"
    return c, go


def _scale_bias_case(dtype, batch):
    c = rounding_case(seed_of("sb", DT_ID[dtype]), 1024, 192, 1, 16, dtype, batch)
    return c, model_forward(c, gemm=False, partial=True)


# ==== GPU harness: the C-ABI with poisoned outputs and workspaces ====================================================
def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dtype).to(DEV)


class Out:
    """An output of `shape` between GUARD bytes on each side, all NaN before the call (zeros inside: `zero`)."""

    def __init__(self, shape, dtype, zero=False):
        self.shape, self.dtype = tuple(shape), dtype
        esz = torch.empty((), dtype=dtype).element_size()
        self.g, self.n = GUARD // esz, int(np.prod(shape))
        self.buf = torch.full((self.n + 2 * self.g,), float("nan"), dtype=dtype, device=DEV)
        if zero:
            self.buf[self.g:self.g + self.n] = 0
        self.guards0 = self._guards().clone()

    def _guards(self):
        return torch.cat([self.buf[:self.g], self.buf[self.g + self.n:]]).view(torch.uint8)

    @property
    def ptr(self):
        return self.buf[self.g:].data_ptr()

    def result(self, what):
        torch.cuda.synchronize()
        assert torch.equal(self._guards(), self.guards0), f"{what}: a guard element was written"
        return self.buf[self.g:self.g + self.n].double().cpu().numpy().reshape(self.shape)


class Workspace:
    """Counters zeroed, partial region NaN-filled; the call must leave the ticket words at zero."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.buf = None
        if self.nbytes:
            self.buf = torch.empty(self.nbytes, dtype=torch.uint8, device=DEV)
            self.buf[:WS_COUNTERS] = 0
            self.buf[WS_COUNTERS:].view(torch.float32).fill_(float("nan"))

    @property
    def ptr(self):
        return None if self.buf is None else self.buf.data_ptr()

    def check(self, what):
        if self.buf is not None:
            torch.cuda.synchronize()
            assert int(torch.count_nonzero(self.buf[:WS_TICKETS])) == 0, f"{what}: ticket words left nonzero"


def _lib():
    from aqlm_b200 import _cabi

    return _cabi.lib()


def _check(rc):
    from aqlm_b200 import _cabi

    _cabi.check(rc)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _weight(c, out=None, cbs=False, bias=True):
    """Device tensors and the C-ABI descriptor (out: per-expert rows of a routed call)."""
    from aqlm_b200 import _cabi

    dtype = c["dtype"]
    t = dict(codes=torch.from_numpy(O.pack_int_data(c["raw"], c["nbits"])).to(DEV).contiguous(),
             cb=_dev(c["cbs"] if cbs else c["cb"], dtype), s=_dev(c["s"], dtype),
             b=_dev(c["b"], dtype) if (bias and c["b"] is not None) else None)
    w = _cabi.Weight()
    w.codes, w.codebooks, w.scales = t["codes"].data_ptr(), t["cb"].data_ptr(), t["s"].data_ptr()
    w.bias = t["b"].data_ptr() if t["b"] is not None else None
    w.in_features, w.out_features = c["raw"].shape[1] * c["g"], out or c["raw"].shape[0]
    w.num_codebooks, w.nbits_per_codebook, w.in_group_size, w.out_group_size = c["cb"].shape[0], c["nbits"], c["g"], 1
    w.dtype = _cabi.F16 if dtype == F16 else _cabi.BF16
    return w, t


def _seg_rows(rows):
    return (ctypes.c_int64 * len(rows))(*rows)


def run_forward_gemm(c, partial=False):
    L = _lib()
    w, t = _weight(c)
    x = _dev(c["x"], c["dtype"])
    batch = x.shape[0]
    ws = Workspace(L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), batch))
    out = Out((batch, c["raw"].shape[0]), torch.float32 if partial else c["dtype"])
    _check(L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), x.data_ptr(), out.ptr, batch, 1 if partial else 0, ws.ptr,
                                         ws.nbytes, _stream()))
    y = out.result("forward")
    ws.check("forward")
    return y, ws.nbytes


def run_gemv(c, partial=False):
    """matmat_ws with the LUT's workspace (batch <= 2: the LUT paths), matmat_ex otherwise."""
    L = _lib()
    w, t = _weight(c)
    x = _dev(c["x"], c["dtype"])
    batch = x.shape[0]
    out = Out((batch, c["raw"].shape[0]), torch.float32 if partial else c["dtype"])
    flags = 1 if partial else 0
    ws = Workspace(L.aqlm_b200_matmat_workspace_bytes(ctypes.byref(w), batch))
    if ws.nbytes:
        _check(L.aqlm_b200_matmat_ws(ctypes.byref(w), x.data_ptr(), out.ptr, batch, flags, ws.ptr, ws.nbytes, _stream()))
    else:
        _check(L.aqlm_b200_matmat_ex(ctypes.byref(w), x.data_ptr(), out.ptr, batch, flags, _stream()))
    y = out.result("gemv")
    ws.check("gemv")
    return y


def run_transposed(c, go):
    L = _lib()
    w, t = _weight(c, bias=False)
    g = _dev(go, c["dtype"])
    batch = go.shape[0]
    ws = Workspace(L.aqlm_b200_matmat_dequant_transposed_workspace_bytes(ctypes.byref(w), batch))
    out = Out((batch, c["raw"].shape[1] * c["g"]), c["dtype"])
    _check(L.aqlm_b200_matmat_dequant_transposed(ctypes.byref(w), g.data_ptr(), out.ptr, batch, ws.ptr, ws.nbytes,
                                                 _stream()))
    y = out.result("transposed")
    ws.check("transposed")
    return y, ws.nbytes


# ==== GPU: wgmma forward and transposed ==============================================================================
@gpu
@pytest.mark.parametrize("K,nbits,dtype,batch,tile_m,ksplit", _fwd_cases())
def test_forward_gemm_rounds_as_modelled(K, nbits, dtype, batch, tile_m, ksplit):
    forced = (tile_m, ksplit) != (None, None)
    fin = FORCED_SHAPE[0] if forced else FWD_SHAPE[0]
    pid = f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}" + (f"-tm{tile_m}-ks{ksplit}" if forced else "")
    c = rounding_case(seed_of("fwd", pid), fin, FWD_SHAPE[1], K, nbits, dtype, batch)
    with tunables(gemm_tile_m=tile_m, gemm_ksplit=ksplit):
        y, need = run_forward_gemm(c)
        if ksplit and ksplit > 1:
            assert need > WS_COUNTERS, "the forced split must run through the workspace"
        assert_exact(y, model_forward(c), f"forward {pid}", tile_m=tile_m, n_tile=n_tile_of(batch))
        if forced:  # the same plan with fp32 partials: the unscaled sums of the rounded W
            p, _ = run_forward_gemm(c, partial=True)
            assert_exact(p, model_forward(c, partial=True), f"forward partial {pid}", tile_m=tile_m)


@gpu
@pytest.mark.parametrize("K,nbits,dtype,batch,ksplit", _t_cases())
def test_transposed_gemm_rounds_as_modelled(K, nbits, dtype, batch, ksplit):
    pid = f"{K}x{nbits}-{DT_ID[dtype]}-bs{batch}" + (f"-ks{ksplit}" if ksplit else "")
    c = rounding_case(seed_of("t", pid), *T_SHAPE, K, nbits, dtype, bias=False, transposed=True)
    go = sparse_go(seed_of("t-go", pid), batch, T_SHAPE[1], c["win"])
    with tunables(gemm_ksplit=ksplit):
        gx, need = run_transposed(c, go)
    if ksplit and ksplit > 1:
        assert need > WS_COUNTERS
    assert_exact(gx, model_transposed(c, go), f"transposed {pid}", n_tile=n_tile_of(batch))


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_grouped_gemm_rounds_as_modelled(dtype):
    """Three segments with their own codebooks (ragged segment ends), forward at 17 rows and transposed at 7."""
    L = _lib()
    segs = [72, 64, 64]
    fout = sum(segs)
    seg_of = np.repeat(np.arange(3), segs)
    c = rounding_case(seed_of("grouped", DT_ID[dtype]), 512, fout, 2, 8, dtype, 17, n_cb_sets=3)
    W = _segment(c, seg_of)
    w, t = _weight(c, cbs=True)
    x = _dev(c["x"], dtype)
    ws = Workspace(L.aqlm_b200_matmat_dequant_workspace_bytes(ctypes.byref(w), 17))
    out = Out((17, fout), dtype)
    _check(L.aqlm_b200_matmat_dequant_grouped(ctypes.byref(w), _seg_rows(segs), 3, x.data_ptr(), out.ptr, 17, 0, ws.ptr,
                                              ws.nbytes, _stream()))
    assert_exact(out.result("grouped"), model_forward(c, w=rT(W, dtype)), "grouped forward")
    ws.check("grouped")
    ct = rounding_case(seed_of("grouped-t", DT_ID[dtype]), 512, fout, 2, 8, dtype, bias=False, transposed=True, n_cb_sets=3)
    go = sparse_go(seed_of("grouped-t-go"), 7, fout, ct["win"])
    w, t = _weight(ct, cbs=True, bias=False)
    g = _dev(go, dtype)
    out = Out((7, 512), dtype)
    _check(L.aqlm_b200_matmat_dequant_transposed_grouped(ctypes.byref(w), _seg_rows(segs), 3, g.data_ptr(), out.ptr, 7,
                                                         None, 0, _stream()))
    assert_exact(out.result("grouped transposed"), model_transposed(ct, go, model_a_operand(ct, _segment(ct, seg_of))),
                 "grouped transposed")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_routed_gemm_rounds_as_modelled(dtype):
    """Two experts with their own weights over expert-sorted rows (5 and 18: ragged), forward and transposed."""
    L = _lib()
    out_e, off = 136, [0, 5, 23]
    rows = off[-1]
    expert_of_row = np.repeat(np.arange(2), np.diff(off))
    offs = torch.tensor(off, dtype=torch.int32, device=DEV)
    for transposed in (False, True):
        c = rounding_case(seed_of("routed", DT_ID[dtype], transposed), 512, 2 * out_e, 2, 8, dtype, rows,
                          bias=not transposed, transposed=transposed, n_cb_sets=2)
        W = _segment(c, np.repeat(np.arange(2), out_e))  # [2 * out_e, in]: expert e's rows
        w, t = _weight(c, out=out_e, cbs=True, bias=not transposed)
        ws = Workspace(L.aqlm_b200_matmat_dequant_routed_workspace_bytes(ctypes.byref(w), 2, rows, int(transposed)))
        if not transposed:
            x = _dev(c["x"], dtype)
            out = Out((rows, out_e), dtype)
            _check(L.aqlm_b200_matmat_dequant_routed(ctypes.byref(w), None, 1, 2, offs.data_ptr(), x.data_ptr(), out.ptr,
                                                     rows, ws.ptr, ws.nbytes, _stream()))
            ref = np.empty((rows, out_e))
            for e in range(2):
                sl, ro = slice(off[e], off[e + 1]), slice(e * out_e, (e + 1) * out_e)
                ce = dict(c, s=c["s"][ro], b=c["b"][ro])
                ref[sl] = model_forward(ce, x=c["x"][sl], w=rT(W[ro], dtype))
        else:
            go = np.zeros((rows, out_e))
            for e in range(2):
                go[off[e]:off[e + 1]] = sparse_go(seed_of("routed-go", e), off[e + 1] - off[e], out_e, c["win"])
            g = _dev(go, dtype)
            out = Out((rows, 512), dtype)
            _check(L.aqlm_b200_matmat_dequant_transposed_routed(ctypes.byref(w), None, 1, 2, offs.data_ptr(), g.data_ptr(),
                                                                out.ptr, rows, ws.ptr, ws.nbytes, _stream()))
            a = model_a_operand(c, W)
            ref = np.concatenate([model_transposed(c, go[off[e]:off[e + 1]], a[e * out_e:(e + 1) * out_e])
                                  for e in range(2)])
        assert_exact(out.result("routed"), ref, f"routed {'transposed' if transposed else 'forward'}")
        ws.check("routed")


# ==== GPU: GEMV and LUT paths ========================================================================================
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("path,K,nbits,g,fin,batch,switches", GEMV_CASES,
                         ids=[f"{p}-{k}x{n}-g{g}-in{f}-bs{b}" + "".join(f"-{s}" for s in sw) for p, k, n, g, f, b, sw in GEMV_CASES])
def test_gemv_paths_round_as_modelled(path, K, nbits, g, fin, batch, switches, dtype):
    from aqlm_b200 import _cabi

    name = f"gemv {path} {K}x{nbits} g{g} in{fin} bs{batch} {DT_ID[dtype]}"
    c = rounding_case(seed_of("gemv", name), fin, GEMV_OUT, K, nbits, dtype, batch, g)
    with tunables(**switches):
        before = _cabi.launch_count()
        if path == "gemv-passes":  # the GEMM entry point with the wgmma kernels switched off
            L = _lib()
            w, t = _weight(c)
            x = _dev(c["x"], dtype)
            out = Out((batch, GEMV_OUT), dtype)
            _check(L.aqlm_b200_matmat_dequant_ex(ctypes.byref(w), x.data_ptr(), out.ptr, batch, 0, None, 0, _stream()))
            y = out.result(name)
        else:
            y = run_gemv(c)
        launches = _cabi.launch_count() - before
    assert_exact(y, model_forward(c, gemm=False), name)
    expect = {"lut-row-loop": batch, "gemv-passes": math.ceil(batch / 8)}.get(path, 1)
    assert launches == expect, (path, launches)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_grouped_gemv_and_partial_scale_bias_round_as_modelled(dtype):
    L = _lib()
    segs = [128, 64]
    c = rounding_case(seed_of("grouped-gemv", DT_ID[dtype]), 1024, 192, 1, 16, dtype, 3, n_cb_sets=2)
    w, t = _weight(c, cbs=True)
    x = _dev(c["x"], dtype)
    out = Out((3, 192), dtype)
    _check(L.aqlm_b200_matmat_grouped(ctypes.byref(w), _seg_rows(segs), 2, x.data_ptr(), out.ptr, 3, 0, _stream()))
    assert_exact(out.result("grouped gemv"), model_forward(c, w=_segment(c, np.repeat([0, 1], segs)), gemm=False),
                 "grouped GEMV")
    # PARTIAL_F32 on a 2x8 GEMV (W never rounded), then scale_bias
    c = rounding_case(seed_of("partial", DT_ID[dtype]), 1024, 200, 2, 8, dtype, 2)
    p = run_gemv(c, partial=True)
    assert_exact(p, model_forward(c, gemm=False, partial=True), "GEMV partial")
    c2, p2 = _scale_bias_case(dtype, 3)
    pd = torch.from_numpy(p2.astype(np.float32)).to(DEV)
    assert np.array_equal(pd.double().cpu().numpy(), p2)
    s, b = _dev(c2["s"], dtype), _dev(c2["b"], dtype)
    out = Out(p2.shape, dtype)
    _check(L.aqlm_b200_scale_bias(pd.data_ptr(), s.data_ptr(), b.data_ptr(), out.ptr, 3, 192, 0 if dtype == F16 else 1,
                                  _stream()))
    assert_exact(out.result("scale_bias"), model_scale_bias(p2, c2["s"], c2["b"], dtype), "scale_bias")


# ==== GPU: dequant, weight gradient, exchange epilogues ==============================================================
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits,g", DEQ_CASES)
def test_dequant_rounds_as_modelled(K, nbits, g, dtype):
    L = _lib()
    c = rounding_case(seed_of("deq", K, nbits, g, DT_ID[dtype]), 512, 136, K, nbits, dtype, g=g, bias=False)
    w, t = _weight(c, bias=False)
    for apply in (1, 0):
        out = Out((136, 512), dtype)
        _check(L.aqlm_b200_dequant(ctypes.byref(w), out.ptr, apply, _stream()))
        assert_exact(out.result("dequant"), model_dequant(c, apply), f"dequant {K}x{nbits} g{g} apply_scales={apply}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits", WGRAD_SCHEMES)
def test_weight_grad_sees_the_rounded_w(K, nbits, dtype):
    L = _lib()
    c, go = _wgrad_case(K, nbits, dtype)
    gs_ref, gcb_ref = model_wgrad(c, go)
    w, t = _weight(c, bias=False)
    x, g = _dev(c["x"], dtype), _dev(go, dtype)
    fout = c["raw"].shape[0]
    ws = Workspace(L.aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(w), WGRAD_BATCH))
    gcb = Out(gcb_ref.shape, torch.float32, zero=True)
    gs = Out((fout,), torch.float32)
    _check(L.aqlm_b200_matmat_weight_grad(ctypes.byref(w), x.data_ptr(), g.data_ptr(), WGRAD_BATCH, gcb.ptr, gs.ptr,
                                          ws.ptr, ws.nbytes, _stream()))
    assert_exact(gs.result("grad_scales")[None], gs_ref[None], f"grad_scales {K}x{nbits}")
    assert_exact(gcb.result("grad_codebooks").reshape(1, -1), gcb_ref.reshape(1, -1), f"grad_codebooks {K}x{nbits}")
    ws.check("weight grad")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_exchange_epilogues_round_as_modelled(dtype):
    """allreduce_scale_bias and the GEMV with the exchange fused, on a one-GPU communicator over a buffer of ours."""
    L = _lib()
    max_elems = 4096
    shared = torch.zeros(L.aqlm_b200_comm_shared_bytes(1, max_elems), dtype=torch.uint8, device=DEV)
    comm = ctypes.c_void_p()
    _check(L.aqlm_b200_comm_create(0, 1, (ctypes.c_void_p * 1)(shared.data_ptr()), max_elems, ctypes.byref(comm)))
    try:
        dt = 0 if dtype == F16 else 1
        c, p = _scale_bias_case(dtype, 3)
        pd = torch.from_numpy(p.astype(np.float32)).to(DEV)
        s, b = _dev(c["s"], dtype), _dev(c["b"], dtype)
        out = Out(p.shape, dtype)
        _check(L.aqlm_b200_allreduce_scale_bias(comm, pd.data_ptr(), s.data_ptr(), b.data_ptr(), out.ptr, 3, 192, dt,
                                                _stream()))
        assert_exact(out.result("allreduce_scale_bias"), model_scale_bias(p, c["s"], c["b"], dtype), "allreduce_scale_bias")
        c = rounding_case(seed_of("fused-exchange", DT_ID[dtype]), 1024, 192, 1, 16, dtype, 2)
        w, t = _weight(c)
        x = _dev(c["x"], dtype)
        out = Out((2, 192), dtype)
        _check(L.aqlm_b200_matmat_allreduce(comm, ctypes.byref(w), None, 1, x.data_ptr(), out.ptr, 2, _stream()))
        assert_exact(out.result("matmat_allreduce"), model_forward(c, gemm=False), "matmat_allreduce")
    finally:
        torch.cuda.synchronize()
        L.aqlm_b200_comm_destroy(comm)


# ==== GPU: range variants ============================================================================================
@gpu
@pytest.mark.parametrize("variant,dtype", _variant_cases())
def test_range_variants_round_as_modelled(variant, dtype):
    """Outputs far outside fp16's range (bf16), subnormal scales and outputs, outputs past 65504 (fp16: +-inf), on
    the wgmma forward, the vector GEMV, the cluster LUT, the transposed GEMM, dequant and scale_bias."""
    c = rounding_case(seed_of("var", variant), 512, 200, 2, 8, dtype, 17, variant=variant)
    y, _ = run_forward_gemm(c)
    assert_exact(y, model_forward(c), f"{variant}: wgmma forward")
    for batch in (1, 5):  # cluster LUT, vector Kx8 kernel
        cg = rounding_case(seed_of("var-gemv", variant, batch), 1024, 200, 2, 8, dtype, batch, variant=variant)
        assert_exact(run_gemv(cg), model_forward(cg, gemm=False), f"{variant}: GEMV bs={batch}")
    L = _lib()
    w, t = _weight(c, bias=False)
    out = Out((200, 512), dtype)
    _check(L.aqlm_b200_dequant(ctypes.byref(w), out.ptr, 1, _stream()))
    assert_exact(out.result("dequant"), model_dequant(c, 1), f"{variant}: dequant")
    p = model_forward(c, partial=True)
    pd = torch.from_numpy(p.astype(np.float32)).to(DEV)
    s, b = _dev(c["s"], dtype), _dev(c["b"], dtype)
    out = Out(p.shape, dtype)
    _check(L.aqlm_b200_scale_bias(pd.data_ptr(), s.data_ptr(), b.data_ptr(), out.ptr, p.shape[0], p.shape[1],
                                  0 if dtype == F16 else 1, _stream()))
    assert_exact(out.result("scale_bias"), model_scale_bias(p, c["s"], c["b"], dtype), f"{variant}: scale_bias")
    if variant != "f16-overflow":  # an infinite A operand times a zero of grad_out is NaN in any GEMM
        ct = rounding_case(seed_of("var-t", variant), *T_SHAPE, 2, 8, dtype, bias=False, transposed=True, variant=variant)
        go = sparse_go(seed_of("var-t-go", variant), 7, T_SHAPE[1], ct["win"])
        gx, _ = run_transposed(ct, go)
        assert_exact(gx, model_transposed(ct, go), f"{variant}: transposed")
