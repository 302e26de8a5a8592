"""Grouped and routed weight gradients: one launch for the codebook and scale gradients of a group of linears sharing
their input (q/k/v, gate/up), or of every expert of a mixture-of-experts projection (csrc/gemm_wgrad.cuh).

CPU: the routed plan (`gemm_wgrad_routed_plan`, through a driver compiled against plan.cuh as test_zz_weight_grad.py
compiles one), the expert row ranges of routing.cuh against a brute force, and the argument checks of both C-ABI entry
points, which run before any device query.

GPU: bit-exact on the integer lattice of test_zz_weight_grad.py (every partial sum exact, so the fp32 result equals the
fp64 reference whatever the order of the atomic reductions).  Rows that belong to no expert, and every row outside the
expert under test, hold NaN and inf in both operands.  Then the modules: launch counts, mixed trainability, gradients
against the members run alone and against transformers' dense MixtralExperts, an optimizer step, CUDA-graph replay with
new routing, and deterministic mode.
"""
import copy
import ctypes
import math
import os
import subprocess
import warnings

import numpy as np
import pytest
import torch
from test_zz_routed_gemm import ROUTINGS, SLOT_CASES, effective_offsets
from test_zz_weight_grad import (DT_ID, DTYPES, SCHEMES, WS_COUNTERS, X_MAX, _unfreeze, exact_weight_grad,
                                 expected_plan, lattice_linear, lattice_module, to_dev)

from aqlm_b200 import _cabi

DEV = "cuda:0"
gpu = pytest.mark.gpu
MAX_TILES = 8192  # ticket words of the counter region (plan.cuh kGemmMaxTiles)


# ---- routed plan and expert rows (CPU) -------------------------------------------------------------------------------
DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "plan.cuh"

using namespace aqlm_b200;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    std::string kind;
    is >> kind;
    if (kind == "rows") {  // rows E off[0..E]: every expert's effective row range
      int rows, E;
      is >> rows >> E;
      std::vector<int32_t> off(E + 1);
      for (auto& o : off) is >> o;
      for (int e = 0; e < E; ++e) {
        const RoutedRows r = routed_expert_rows(off.data(), rows, e);
        std::printf("%d %d ", r.first, r.end);
      }
      std::printf("\n");
      continue;
    }
    long long K, nbits, g, fin, fout, off, rows, E;
    is >> K >> nbits >> g >> fin >> fout >> off >> rows >> E;
    Tunables t;
    t.load();
    DeviceInfo di;
    di.max_smem_optin = 232448;
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
    const WgradPlan p = gemm_wgrad_routed_plan(w, (int)E, rows, di, t);
    if (!p.ok) std::printf("0\n");
    else std::printf("1 %d %d %d %d %zu %zu %zu\n", p.out_tiles, p.in_tiles, p.stages, p.total_kblocks, p.smem,
                     p.counters_bytes, p.dots_bytes);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("routed_wgrad")
    src = tmp / "driver.cu"
    src.write_text(DRIVER)
    exe = tmp / "driver"
    flags = [f for f in _cabi.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    subprocess.run(["nvcc", *flags, "-I", _cabi.CSRC, "-o", str(exe), str(src)], check=True, capture_output=True, text=True)
    env = {k: v for k, v in os.environ.items() if not k.startswith("AQLM_B200_")}

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", check=True, capture_output=True, text=True,
                             env=env).stdout.splitlines()
        assert len(out) == len(lines)
        return out
    return run


def expected_routed_plan(K, nbits, g, fin, fout, off, rows, E):
    """The plain plan of `rows` rows, with one ticket word per (expert, out tile) and row dots [in_tiles][E * out]."""
    p = expected_plan(K, nbits, g, fin, fout, off, rows)
    if p == "0" or rows < 1 or not 1 <= E <= 64 or E * -(-fout // 128) > MAX_TILES:
        return "0"
    f = p.split()
    return " ".join(f[:-1] + [str(int(f[-1]) * E)])


def routed_plan_cases():
    """(K, nbits, g, in, out, codes offset, rows, E)"""
    shapes = [(4096, 28672), (14336, 4096), (1152, 256), (1088, 200)]  # Mixtral w1|w3 and w2, small experts
    for K, nbits in SCHEMES:
        for fin, fout in shapes:
            for rows in (1, 63, 300, 4096):
                for E in (1, 8, 64):
                    yield (K, nbits, 8, fin, fout, 0, rows, E)
    for E in (0, -1, 65, 36, 37):  # E * 224 out tiles of 28672 rows: 36 fit the 8192 ticket words, 37 do not
        yield (1, 16, 8, 4096, 28672, 0, 300, E)
    for K, nbits, g, off in [(1, 16, 16, 0), (3, 8, 8, 0), (1, 16, 8, 8)]:
        yield (K, nbits, g, 4096, 4096, off, 300, 8)
    yield (1, 16, 8, 4096, 4100, 0, 300, 8)   # out % 8
    yield (1, 16, 8, 4096, 4096, 0, 0, 8)     # no rows


def test_routed_weight_grad_plan_pins(driver):
    cases = list(routed_plan_cases())
    got = driver([" ".join(map(str, ("plan",) + c)) for c in cases])
    want = [expected_routed_plan(*c) for c in cases]
    diff = [f"{c}: want [{w}] got [{g}]" for c, w, g in zip(cases, want, got) if w != g]
    assert not diff, f"{len(diff)} of {len(cases)} plans differ:\n" + "\n".join(diff[:20])
    by_case = dict(zip(cases, got))
    assert by_case[(1, 16, 8, 4096, 28672, 0, 300, 36)] != "0" and by_case[(1, 16, 8, 4096, 28672, 0, 300, 37)] == "0"
    assert by_case[(1, 16, 8, 4096, 28672, 0, 4096, 64)] == "0"  # 64 x 224 out tiles overflow the counters


def test_expert_rows_match_brute_force(driver):
    offs = [(rows, off) for rows, _, off in SLOT_CASES] + list(ROUTINGS.values())
    rng = np.random.default_rng(5)
    for _ in range(40):  # random malformed tables
        E, rows = int(rng.integers(1, 9)), int(rng.integers(0, 200))
        offs.append((rows, rng.integers(-20, rows + 20, size=E + 1).tolist()))
    got = driver([f"rows {rows} {len(off) - 1} " + " ".join(map(str, off)) for rows, off in offs])
    for (rows, off), line in zip(offs, got):
        c = effective_offsets(off, rows)
        want = [v for e in range(len(off) - 1) for v in (c[e], c[e + 1])]
        assert list(map(int, line.split())) == want, (rows, off)


# ---- C-ABI argument checks (CPU: no device is touched) ---------------------------------------------------------------
def _weight(K=2, nbits=8, g=8, fin=256, fout=64):
    w = _cabi.Weight()
    w.codes, w.codebooks, w.scales = 16, 16, 16  # dummy non-null aligned pointers (never dereferenced)
    w.in_features, w.out_features = fin, fout
    w.num_codebooks, w.nbits_per_codebook, w.in_group_size, w.out_group_size = K, nbits, g, 1
    w.dtype = _cabi.F16
    return w


def _seg(rows):
    return (ctypes.c_int64 * len(rows))(*rows)


def test_grouped_and_routed_weight_grad_checks_without_a_device():
    L = _cabi.lib()
    for name in ("aqlm_b200_matmat_weight_grad_grouped", "aqlm_b200_matmat_weight_grad_routed",
                 "aqlm_b200_matmat_weight_grad_routed_workspace_bytes"):
        assert name in _cabi.header_symbols() and hasattr(ctypes.CDLL(_cabi.LIB_PATH), name)

    def grouped(w, seg=(32, 32), n_seg=None, x=16, go=16, b=64, gcb=16, gs=16):
        return L.aqlm_b200_matmat_weight_grad_grouped(ctypes.byref(w), _seg(seg) if seg is not None else None,
                                                      len(seg) if n_seg is None else n_seg, x, go, b, gcb, gs, None, 0,
                                                      None)

    def routed(w, seg=None, n_seg=1, E=4, off=16, x=16, go=16, rows=64, gcb=16, gs=16):
        return L.aqlm_b200_matmat_weight_grad_routed(ctypes.byref(w), _seg(seg) if seg is not None else None, n_seg, E,
                                                     off, x, go, rows, gcb, gs, None, 0, None)

    S, U = _cabi.ERR_SHAPE, _cabi.ERR_UNSUPPORTED
    def routed2(w, seg=(32, 32), **k):
        return routed(w, seg=seg, n_seg=len(seg), **k)

    for call in (grouped, routed2):
        assert call(_weight(), x=None) == S
        assert call(_weight(), go=None) == S
        assert call(_weight(), gcb=None, gs=None) == S
        assert call(_weight(K=1, nbits=16, g=16)) == U     # in_group 16
        assert call(_weight(K=3)) == U                     # 3 codebooks
        assert call(_weight(fout=60), seg=(30, 30)) == U   # out % 8
        assert call(_weight(), x=24) == U                  # input 8-byte aligned only
        assert call(_weight(), go=8) == U
    # segment tables
    for seg, n_seg in [((32, 31), None), ((64, 0), None), ((80, -16), None), ((16,) * 5, None), ((32, 32), 0)]:
        assert grouped(_weight(), seg=seg, n_seg=n_seg) == S, seg
        assert routed(_weight(), seg=seg, n_seg=len(seg) if n_seg is None else n_seg) == S, seg
    assert grouped(_weight(), seg=None, n_seg=1) == S       # a grouped call needs its table
    assert grouped(_weight(), b=-1) == S
    # expert count, offsets, rows
    for E in (0, 65, -1):
        assert routed(_weight(), E=E) == S, E
    assert routed(_weight(), off=None) == S
    assert routed(_weight(), rows=-1) == S
    assert routed(_weight(), rows=1 << 31) == S
    assert L.aqlm_b200_matmat_weight_grad_routed_workspace_bytes(ctypes.byref(_weight()), 0, 64) == 0
    if not torch.cuda.is_available():
        assert grouped(_weight(), b=0) == _cabi.OK              # no rows: no launch, no device query
        assert routed(_weight(), rows=0) == _cabi.OK
        for rc in (grouped(_weight()), routed(_weight()), routed(_weight(), seg=(32, 32), n_seg=2, E=64)):
            assert rc in (_cabi.ERR_CUDA, _cabi.ERR_ARCH)       # a valid call needs the device, never falls back
        assert L.aqlm_b200_matmat_weight_grad_routed_workspace_bytes(ctypes.byref(_weight()), 4, 64) == 0


# ---- lattice: grouped (GPU) ------------------------------------------------------------------------------------------
GROUP_IN = 384
GROUP_SEGS = [[128, 64, 64], [200, 56], [8, 8, 240]]
GROUP_BATCHES = [1, 7, 64, 129, 300]


def _lattice_group(seed, segs, K, nbits, dtype):
    lins = [lattice_linear(seed + 17 * i, GROUP_IN, n, K, nbits) for i, n in enumerate(segs)]
    t = dict(codes=torch.from_numpy(np.concatenate([lin["codes"] for lin in lins])).to(DEV),
             codebooks=torch.stack([to_dev(lin["codebooks"], dtype) for lin in lins]).contiguous(),
             scales=to_dev(np.concatenate([lin["scales"] for lin in lins]), dtype))
    return lins, t


def _c_grouped(t, segs, x, go, gcb, gs, ws):
    from aqlm_b200.inference_kernels import cuda_kernel

    w = cuda_kernel.make_weight(t["codes"], t["codebooks"][0], t["scales"].reshape(-1), None)
    return _cabi.lib().aqlm_b200_matmat_weight_grad_grouped(
        ctypes.byref(w), _seg(segs), len(segs), x.data_ptr(), go.data_ptr(), x.shape[0],
        gcb.data_ptr() if gcb is not None else None, gs.data_ptr() if gs is not None else None,
        ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0,
        torch.cuda.current_stream().cuda_stream)


@gpu
@pytest.mark.parametrize("segs", GROUP_SEGS, ids=lambda s: "-".join(map(str, s)))
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits", SCHEMES, ids=lambda v: str(v))
def test_lattice_grouped_weight_grad_is_exact(K, nbits, dtype, segs):
    from aqlm_b200.inference_kernels import cuda_kernel

    lins, t = _lattice_group(1000 * K + nbits + len(segs), segs, K, nbits, dtype)
    out = sum(segs)
    w = cuda_kernel.make_weight(t["codes"], t["codebooks"][0], t["scales"].reshape(-1), None)
    for batch in GROUP_BATCHES:
        rng = np.random.default_rng(batch * 13 + len(segs))
        x = rng.integers(-X_MAX, X_MAX + 1, size=(batch, GROUP_IN)).astype(np.float32)
        go = rng.integers(-X_MAX, X_MAX + 1, size=(batch, out)).astype(np.float32)
        refs, off = [], 0
        for lin, n in zip(lins, segs):
            refs.append(exact_weight_grad(lin, x, go[:, off:off + n]))
            off += n
        ref_cb = np.stack([r[0] for r in refs]).astype(np.float32)
        ref_s = np.concatenate([r[1] for r in refs]).astype(np.float32)
        xd, god = to_dev(x, dtype), to_dev(go, dtype)
        what = f"{K}x{nbits} {DT_ID[dtype]} segs {segs} batch {batch}"
        need = _cabi.lib().aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(w), batch)
        assert need == WS_COUNTERS + math.ceil(GROUP_IN / 128) * out * 4
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        gcb = torch.zeros(ref_cb.shape, dtype=torch.float32, device=DEV)
        gs = torch.full((out,), -7.0, dtype=torch.float32, device=DEV)
        before = _cabi.launch_count()
        assert _c_grouped(t, segs, xd, god, gcb, gs, ws) == _cabi.OK
        torch.cuda.synchronize()
        assert _cabi.launch_count() - before == 1
        assert not ws[:WS_COUNTERS].any(), "ticket counters not left at zero"
        assert torch.equal(gcb.cpu(), torch.from_numpy(ref_cb)), what + ": grad_codebooks"
        assert torch.equal(gs.cpu(), torch.from_numpy(ref_s)), what + ": grad_scales"
        # a second call adds into grad_codebooks and rewrites grad_scales
        assert _c_grouped(t, segs, xd, god, gcb, gs, ws) == _cabi.OK
        assert torch.equal(gcb.cpu(), torch.from_numpy(2 * ref_cb)), what + ": accumulation"
        assert torch.equal(gs.cpu(), torch.from_numpy(ref_s))
        # one output requested: the other buffer is untouched
        sentinel = torch.full_like(gcb, 5.0)
        gs2 = torch.full_like(gs, -3.0)
        assert _c_grouped(t, segs, xd, god, None, gs2, ws) == _cabi.OK
        assert _c_grouped(t, segs, xd, god, sentinel, None, None) == _cabi.OK
        assert torch.equal(gs2, gs) and torch.equal(sentinel.cpu(), torch.from_numpy(ref_cb + 5)), what
        assert not ws[:WS_COUNTERS].any()
        # the Python op: the parameters' dtypes, rounded once
        pcb, ps = cuda_kernel.matmat_weight_grad_grouped(xd, god, t["codes"], t["codebooks"], t["scales"], segs)
        assert torch.equal(pcb.float().cpu(), torch.from_numpy(ref_cb).to(dtype).float()), what
        assert torch.equal(ps.float().cpu().reshape(-1), torch.from_numpy(ref_s).to(dtype).float()), what


# ---- lattice: routed (GPU) -------------------------------------------------------------------------------------------
ROUTED_IN = 384
ROUTED_SEGS = {1: [256], 2: [200, 56]}
ROUTED_SCHEMES = [(1, 16), (2, 8), (8, 8), (1, 8)]
POISON = np.array([np.nan, np.inf, -np.inf], dtype=np.float32)
E64 = (300, [0] + sorted(np.random.default_rng(64).integers(0, 300, size=63).tolist()) + [290])  # rows past 290: none


def _lattice_experts(seed, segs, K, nbits, E, dtype):
    experts = [[lattice_linear(seed + 101 * e + 7 * i, ROUTED_IN, n, K, nbits) for i, n in enumerate(segs)]
               for e in range(E)]
    t = dict(codes=torch.stack([torch.from_numpy(np.concatenate([l["codes"] for l in ex])) for ex in experts]).to(DEV),
             codebooks=torch.stack([torch.stack([to_dev(l["codebooks"], dtype) for l in ex]) for ex in experts]).contiguous(),
             scales=torch.stack([to_dev(np.concatenate([l["scales"] for l in ex]), dtype) for ex in experts]).contiguous())
    return experts, t


def _poisoned(a, keep):
    """`a` with every row outside the [lo, hi) ranges of `keep` set to NaN / inf / -inf, cycling."""
    p = np.empty_like(a)
    p[:] = POISON[np.arange(a.shape[0]) % 3][:, None] if a.shape[0] else 0
    for lo, hi in keep:
        p[lo:hi] = a[lo:hi]
    return p


def _c_routed(t, segs, E, off, x, go, gcb, gs, ws):
    from aqlm_b200.inference_kernels import cuda_kernel

    w, seg, n_seg, _ = cuda_kernel._routed_weight(t["codes"], t["codebooks"], t["scales"], segs if len(segs) > 1 else None)
    return _cabi.lib().aqlm_b200_matmat_weight_grad_routed(
        ctypes.byref(w), seg, n_seg, E, off.data_ptr(), x.data_ptr(), go.data_ptr(), x.shape[0],
        gcb.data_ptr() if gcb is not None else None, gs.data_ptr() if gs is not None else None,
        ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0,
        torch.cuda.current_stream().cuda_stream)


def _routed_ref(experts, segs, x, go, c, e):
    refs, off = [], 0
    for lin, n in zip(experts[e], segs):
        refs.append(exact_weight_grad(lin, x[c[e]:c[e + 1]], go[c[e]:c[e + 1], off:off + n]))
        off += n
    return np.stack([r[0] for r in refs]).astype(np.float32), np.concatenate([r[1] for r in refs]).astype(np.float32)


def _routed_params():
    cases = [pytest.param(K, nbits, dtype, n_seg, r, id=f"{K}x{nbits}-{DT_ID[dtype]}-seg{n_seg}-{r}")
             for K, nbits in ROUTED_SCHEMES for dtype in DTYPES for n_seg in (1, 2) for r in ROUTINGS]
    return cases + [pytest.param(K, nbits, torch.float16, 2, "E64", id=f"{K}x{nbits}-f16-seg2-E64")
                    for K, nbits in [(1, 16), (2, 8)]]


@gpu
@pytest.mark.parametrize("K,nbits,dtype,n_seg,routing", _routed_params())
def test_lattice_routed_weight_grad_is_exact(K, nbits, dtype, n_seg, routing):
    segs = ROUTED_SEGS[n_seg]
    rows, off = E64 if routing == "E64" else ROUTINGS[routing]
    E, out = len(off) - 1, sum(segs)
    experts, t = _lattice_experts(1000 * K + nbits + 10 * n_seg + len(routing), segs, K, nbits, E, dtype)
    c = effective_offsets(off, rows)
    rng = np.random.default_rng(rows + E)
    x = rng.integers(-X_MAX, X_MAX + 1, size=(rows, ROUTED_IN)).astype(np.float32)
    go = rng.integers(-X_MAX, X_MAX + 1, size=(rows, out)).astype(np.float32)
    from aqlm_b200.inference_kernels import cuda_kernel

    w = cuda_kernel._routed_weight(t["codes"], t["codebooks"], t["scales"], segs if n_seg > 1 else None)[0]
    need = _cabi.lib().aqlm_b200_matmat_weight_grad_routed_workspace_bytes(ctypes.byref(w), E, rows)
    assert need == WS_COUNTERS + math.ceil(ROUTED_IN / 128) * E * out * 4
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    offs = torch.tensor(off, dtype=torch.int32, device=DEV)
    full = [(c[e], c[e + 1]) for e in range(E)]
    # every expert at once, rows of no expert poisoned; then each non-empty expert alone, every other row poisoned (the
    # neighbour rows of its tail k-block included)
    for keep in [full] + [[r] for r in full if r[1] > r[0]]:
        checked = range(E) if keep is full else [full.index(keep[0])]
        xd, god = to_dev(_poisoned(x, keep), dtype), to_dev(_poisoned(go, keep), dtype)
        gcb = torch.full((E, n_seg, K, 2 ** nbits, 1, 8), 3.0, dtype=torch.float32, device=DEV)
        gs = torch.full((E * out,), -7.0, dtype=torch.float32, device=DEV)
        before = _cabi.launch_count()
        assert _c_routed(t, segs, E, offs, xd, god, gcb, gs, ws) == _cabi.OK
        torch.cuda.synchronize()
        assert _cabi.launch_count() - before == 1
        assert not ws[:WS_COUNTERS].any(), "ticket counters not left at zero"
        gcb, gs = gcb.cpu(), gs.cpu().reshape(E, out)
        for e in checked:
            what = f"{K}x{nbits} {DT_ID[dtype]} seg{n_seg} {routing} expert {e} rows {c[e]}..{c[e + 1]}"
            if c[e + 1] == c[e]:
                assert bool((gs[e] == 0).all()) and bool((gcb[e] == 3.0).all()), what + ": empty expert"
                continue
            ref_cb, ref_s = _routed_ref(experts, segs, x, go, c, e)
            assert torch.equal(gcb[e], torch.from_numpy(ref_cb + 3.0).reshape(gcb[e].shape)), what + ": grad_codebooks"
            assert torch.equal(gs[e], torch.from_numpy(ref_s)), what + ": grad_scales"


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
@pytest.mark.parametrize("rows", [1, 300, 1000])
def test_one_expert_grad_scales_equal_the_plain_call(K, nbits, rows):
    """E = 1 with offsets [0, rows] on random fp16 data: the same k-block partition as the plain call, and grad_scales is
    deterministic, so the two are bitwise equal; so are repeated routed calls."""
    from aqlm_b200.inference_kernels import cuda_kernel

    g = torch.Generator(DEV).manual_seed(rows)
    fin, fout = 1152, 512
    codes = torch.randint(-128, 128, (1, fout, fin // 8, K), dtype=torch.int8 if nbits == 8 else torch.int16, device=DEV,
                          generator=g)
    if nbits == 16:
        codes = torch.randint(-2 ** 15, 2 ** 15, codes.shape, dtype=torch.int16, device=DEV, generator=g)
    cb = (torch.randn((1, 1, K, 2 ** nbits, 1, 8), device=DEV, generator=g) / K ** 0.5).half()
    sc = (0.75 + 0.5 * torch.rand((1, fout, 1, 1, 1), device=DEV, generator=g)).half()
    x = torch.randn((rows, fin), device=DEV, generator=g).half()
    go = torch.randn((rows, fout), device=DEV, generator=g).half()
    off = torch.tensor([0, rows], dtype=torch.int32, device=DEV)
    _, plain = cuda_kernel.matmat_weight_grad(x, go, codes[0], cb[0, 0], sc[0], False, True)
    w = cuda_kernel._routed_weight(codes, cb, sc, None)[0]
    ws = torch.zeros(_cabi.lib().aqlm_b200_matmat_weight_grad_routed_workspace_bytes(ctypes.byref(w), 1, rows),
                     dtype=torch.uint8, device=DEV)
    runs = []
    for _ in range(3):
        gs = torch.empty(fout, dtype=torch.float32, device=DEV)
        assert _c_routed(dict(codes=codes, codebooks=cb, scales=sc), [fout], 1, off, x, go, None, gs, ws) == _cabi.OK
        runs.append(gs)
    ref = torch.zeros(fout, dtype=torch.float32, device=DEV)
    pw = cuda_kernel.make_weight(codes[0], cb[0, 0], sc[0].reshape(-1), None)
    pws = torch.zeros(_cabi.lib().aqlm_b200_matmat_weight_grad_workspace_bytes(ctypes.byref(pw), rows), dtype=torch.uint8,
                      device=DEV)
    assert _cabi.lib().aqlm_b200_matmat_weight_grad(ctypes.byref(pw), x.data_ptr(), go.data_ptr(), rows, None,
                                                    ref.data_ptr(), pws.data_ptr(), pws.numel(),
                                                    torch.cuda.current_stream().cuda_stream) == _cabi.OK
    assert all(torch.equal(r, ref) for r in runs)
    assert torch.equal(plain.reshape(-1), ref.half())


# ---- modules (GPU) ---------------------------------------------------------------------------------------------------
def _lattice_group_modules(K, nbits, outs=(128, 64, 64), fin=256):
    return [lattice_module(K, nbits, fin, o, seed=o + 3 * i) for i, o in enumerate(outs)]


@gpu
@pytest.mark.parametrize("x_grad", [False, True], ids=["weights", "weights+input"])
@pytest.mark.parametrize("rows", [4, 96])
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_group_backward_is_one_weight_grad_launch(K, nbits, rows, x_grad):
    import aqlm_b200

    members = _lattice_group_modules(K, nbits)
    alone = [copy.deepcopy(m) for m in members]
    grp = aqlm_b200.QuantizedLinearGroup(members)
    _unfreeze(grp.members)
    _unfreeze(alone)
    rng = np.random.default_rng(rows)
    x0 = to_dev(rng.integers(-X_MAX, X_MAX + 1, size=(rows, 256)), torch.float16)
    gos = [to_dev(rng.integers(-X_MAX, X_MAX + 1, size=(rows, m.out_features)), torch.float16) for m in members]
    x = x0.clone().requires_grad_(x_grad)
    before = _cabi.launch_count()
    ys = grp(x)
    assert _cabi.launch_count() - before == 1, "one grouped forward launch"
    before = _cabi.launch_count()
    torch.autograd.backward(ys, gos)
    torch.cuda.synchronize()
    assert _cabi.launch_count() - before == 1 + int(x_grad)
    xa = x0.clone().requires_grad_(x_grad)
    for m, go in zip(alone, gos):
        m(xa).backward(go)
    for a, b in zip(grp.members, alone):
        for p, q in ((a.codebooks, b.codebooks), (a.scales, b.scales), (a.bias, b.bias)):
            assert p.grad.dtype == q.grad.dtype and p.grad.shape == q.grad.shape and torch.equal(p.grad, q.grad)
    if x_grad:
        assert torch.equal(x.grad, xa.grad)


@gpu
def test_group_mixed_trainability():
    import aqlm_b200

    members = _lattice_group_modules(2, 8)
    grp = aqlm_b200.QuantizedLinearGroup(members)
    grp.members[0].scales.requires_grad_(True)
    grp.members[2].codebooks.requires_grad_(True)
    grp.members[2].bias.requires_grad_(True)
    x = to_dev(np.random.default_rng(0).integers(-2, 3, size=(40, 256)), torch.float16)
    sum(y.float().sum() for y in grp(x)).backward()
    m0, m1, m2 = grp.members
    assert m0.scales.grad is not None and m0.codebooks.grad is None and m0.bias.grad is None
    assert m1.scales.grad is None and m1.codebooks.grad is None and m1.bias.grad is None
    assert m2.codebooks.grad is not None and m2.scales.grad is None and m2.bias.grad is not None


@gpu
def test_group_optimizer_step_reaches_the_fused_storage():
    import aqlm_b200

    members = _lattice_group_modules(1, 16)
    grp = aqlm_b200.QuantizedLinearGroup(members)
    _unfreeze(grp.members)
    x = to_dev(np.random.default_rng(1).integers(-2, 3, size=(32, 256)), torch.float16)
    with torch.no_grad():
        y0 = torch.cat(grp(x), -1)
    opt = torch.optim.SGD([p for m in grp.members for p in (m.codebooks, m.scales, m.bias)], lr=2.0 ** -16)
    sum(y.float().sum() for y in grp(x)).backward()
    opt.step()
    with torch.no_grad():
        ys = grp(x)
        for m, y in zip(grp.members, ys):
            assert _rel(y, m(x)) < 1e-3
        assert not torch.equal(torch.cat(ys, -1), y0)
    assert grp.members[1].codebooks.data_ptr() == grp._fused_codebooks[1].data_ptr()


@gpu
def test_group_deterministic_mode_refuses_the_codebook_gradient():
    import aqlm_b200

    grp = aqlm_b200.QuantizedLinearGroup(_lattice_group_modules(2, 8))
    grp.members[1].codebooks.requires_grad_(True)
    x = to_dev(np.ones((16, 256)), torch.float16)
    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="not deterministic"):
            sum(y.float().sum() for y in grp(x)).backward()
        grp.members[1].codebooks.requires_grad_(False)
        grp.members[1].scales.requires_grad_(True)
        sum(y.float().sum() for y in grp(x)).backward()  # the scale gradient alone is deterministic
    finally:
        torch.use_deterministic_algorithms(False)
    assert grp.members[1].scales.grad is not None


def _lattice_block(E=4, H=64, I=64, seed=11):
    from aqlm_b200.moe import QuantizedMixtralExperts

    blk = QuantizedMixtralExperts(E, H, I, lambda t: t, 8, 1, 2, 8, device=DEV, dtype=torch.float16)
    with torch.no_grad():
        for e in range(E):
            for name in ("w1", "w3", "w2"):
                m = getattr(blk.expert(e), name)
                lin = lattice_linear(seed + e * 10 + len(name) + m.out_features, m.in_features, m.out_features, 2, 8)
                m.codes.copy_(torch.from_numpy(lin["codes"]))
                m.codebooks.copy_(to_dev(np.clip(lin["codebooks"], -1, 1), torch.float16))
                m.scales.fill_(1.0)
    return blk


def _block_members(b):
    return [getattr(b.expert(e), n) for e in range(b.num_experts) for n in ("w1", "w2", "w3")]


def _trainable(blk, codebooks=True, scales=True):
    for m in _block_members(blk):
        m.codebooks.requires_grad_(codebooks)
        m.scales.requires_grad_(scales)
    return blk


@gpu
@pytest.mark.parametrize("x_grad", [False, True], ids=["weights", "weights+input"])
def test_mixtral_launches_do_not_depend_on_experts_or_routing(x_grad):
    counts = set()
    for E, T, k, skew in [(4, 24, 1, False), (8, 300, 2, False), (8, 300, 2, True), (16, 7, 2, False)]:
        blk = _trainable(_lattice_block(E=E))
        g = torch.Generator().manual_seed(E + T)
        idx = torch.randint(0, E, (T, k), generator=g)
        if skew:
            idx[:, 0] = 3
            idx[::5, 1] = E  # dropped
        x = torch.randint(-1, 2, (T, 64), generator=g).half().to(DEV).requires_grad_(x_grad)
        before = _cabi.launch_count()
        blk(x, idx.to(DEV), torch.ones((T, k), dtype=torch.float16, device=DEV)).float().sum().backward()
        torch.cuda.synchronize()
        counts.add(_cabi.launch_count() - before)
    # forward: 2 routed GEMMs; backward: 2 routed weight gradients, w2's transposed GEMM, and w1|w3's with an input grad
    assert counts == {5 + int(x_grad)}, counts


@gpu
def test_mixtral_mixed_trainability_and_empty_experts_get_zero():
    blk = _lattice_block()
    for e in range(4):
        blk.expert(e).w2.scales.requires_grad_(True)
    blk.expert(1).w3.codebooks.requires_grad_(True)
    T = 12
    idx = torch.tensor([[0], [2], [3]] * 4, device=DEV)  # expert 1 gets no tokens
    x = to_dev(np.random.default_rng(2).integers(-1, 2, size=(T, 64)), torch.float16)
    blk(x, idx, torch.ones((T, 1), dtype=torch.float16, device=DEV)).float().sum().backward()
    for e in range(4):
        m = blk.expert(e)
        assert m.w2.scales.grad is not None and m.w2.codebooks.grad is None
        assert m.w1.codebooks.grad is None and m.w1.scales.grad is None and m.w3.scales.grad is None
        assert (m.w3.codebooks.grad is not None) == (e == 1)
    assert not blk.expert(1).w2.scales.grad.any() and not blk.expert(1).w3.codebooks.grad.any()
    assert blk.expert(0).w2.scales.grad.any()


def _experts_pair(seed, K, nbits, E=4, hidden=128, inter=256):
    """A trainable QuantizedMixtralExperts with random weights and transformers' dense MixtralExperts holding them
    dequantized in fp32."""
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts

    from aqlm_b200.inference_kernels import cuda_kernel
    from aqlm_b200.moe import QuantizedMixtralExperts

    cfg = MixtralConfig(hidden_size=hidden, intermediate_size=inter, num_local_experts=E)
    dense = MixtralExperts(cfg)
    q = QuantizedMixtralExperts(E, hidden, inter, dense.act_fn, 8, 1, K, nbits, device="cpu", dtype=torch.float16)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in _block_members(q):
            lo, hi = (-128, 128) if nbits <= 8 else (-2 ** 15, 2 ** 15)
            m.codes.copy_(torch.randint(lo, hi, m.codes.shape, generator=g, dtype=torch.int32).to(m.codes.dtype))
            m.codebooks.copy_((torch.randn(m.codebooks.shape, generator=g) * (0.3 / K ** 0.5)).half())
            m.scales.copy_((0.75 + 0.5 * torch.rand(m.scales.shape, generator=g)).half())
    q = q.to(DEV)
    deq = lambda m: cuda_kernel.dequant(m.codes, m.codebooks, m.scales).float()  # noqa: E731
    with torch.no_grad():
        dense.gate_up_proj.copy_(torch.stack([torch.cat([deq(q.expert(e).w1), deq(q.expert(e).w3)]) for e in range(E)]))
        dense.down_proj.copy_(torch.stack([deq(q.expert(e).w2) for e in range(E)]))
    return _trainable(q), dense.to(DEV).float()


def _chain(m, dW):
    """The codebook and scale gradients of quantized linear `m` from the dense gradient dW of W = s * Wu."""
    dW = dW.double()
    c = m.codes.long() % m.codebook_size
    Wu = sum(m.codebooks.detach().double()[k, c[:, :, k], 0, :] for k in range(m.num_codebooks))
    gs = (dW.reshape(Wu.shape) * Wu).sum((1, 2))
    sD = (dW * m.scales.detach().double().reshape(-1, 1)).reshape(-1, 8)
    gcb = torch.zeros((m.num_codebooks, m.codebook_size, 8), dtype=torch.float64, device=DEV)
    for k in range(m.num_codebooks):
        gcb[k].index_add_(0, c[:, :, k].reshape(-1), sD)
    return gcb.reshape(m.codebooks.shape), gs.reshape(m.scales.shape)


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_mixtral_weight_grads_match_dense_mixtral_experts(K, nbits):
    q, dense = _experts_pair(5 + K, K, nbits)
    T, k, E = 300, 2, 4
    g = torch.Generator().manual_seed(K)
    idx = torch.randint(0, E, (T, k), generator=g)
    idx[idx == 2] = 1            # expert 2 gets no tokens
    idx[::4, 1] = E              # dropped ids, both kinds
    idx[1::7, 0] = -1
    idx = idx.to(DEV)
    w = torch.softmax(torch.randn((T, k), generator=g), -1).to(DEV)
    x = torch.randn((T, 128), generator=g).half().to(DEV).requires_grad_(True)
    gy = torch.randn((T, 128), generator=g).half().to(DEV)
    q(x, idx, w).backward(gy)
    keep = (idx >= 0) & (idx < E)
    xd = x.detach().float().requires_grad_(True)
    dense(xd, torch.where(keep, idx, 0), w * keep).backward(gy.float())
    I = 256
    for e in range(E):
        ex = q.expert(e)
        for m, dW in ((ex.w1, dense.gate_up_proj.grad[e, :I]), (ex.w3, dense.gate_up_proj.grad[e, I:]),
                      (ex.w2, dense.down_proj.grad[e])):
            rcb, rs = _chain(m, dW)
            if e == 2:
                assert not m.codebooks.grad.any() and not m.scales.grad.any()
                continue
            assert _rel(m.codebooks.grad, rcb) < 1e-2 and _rel(m.scales.grad, rs) < 1e-2, \
                (e, _rel(m.codebooks.grad, rcb), _rel(m.scales.grad, rs))
    assert _rel(x.grad, xd.grad) < 1e-2


@gpu
def test_mixtral_optimizer_step_reaches_the_stacks():
    blk = _trainable(_lattice_block())
    T = 24
    rng = np.random.default_rng(4)
    x = to_dev(rng.integers(-1, 2, size=(T, 64)), torch.float16)
    idx = torch.from_numpy(rng.integers(0, 4, size=(T, 2))).to(DEV)
    wts = torch.ones((T, 2), dtype=torch.float16, device=DEV)
    with torch.no_grad():
        y0 = blk(x, idx, wts)
    opt = torch.optim.SGD([p for m in _block_members(blk) for p in (m.codebooks, m.scales)], lr=2.0 ** -20)
    blk(x, idx, wts).float().sum().backward()
    opt.step()
    assert blk._w13[1].data_ptr() == blk.expert(0).w1.codebooks.data_ptr()
    with torch.no_grad():
        routed = blk(x, idx, wts)
        loop = blk._forward_loop(x, idx, wts)
    assert not torch.equal(routed, y0), "the step did not reach the stacks"
    assert _rel(routed, loop) < 1e-3


@gpu
def test_mixtral_cuda_graph_replays_forward_and_weight_backward_with_new_routing():
    blk = _trainable(_lattice_block())
    T, k, E = 24, 2, 4
    rng = np.random.default_rng(8)
    new_x = lambda: to_dev(rng.integers(-1, 2, size=(T, 64)), torch.float16)  # noqa: E731

    def new_idx(r):
        idx = torch.from_numpy(rng.integers(0, E, size=(T, k))).to(DEV)
        if r == 2:
            idx[:] = 1          # every token to one expert
        if r == 3:
            idx[::3, 1] = E     # dropped ids
        return idx
    sx, sidx, sg = new_x(), new_idx(0), new_x()
    sw = torch.ones((T, k), dtype=torch.float16, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            blk.zero_grad(set_to_none=True)
            blk(sx, sidx, sw).backward(sg)
    torch.cuda.current_stream().wait_stream(s)
    blk.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        blk(sx, sidx, sw).backward(sg)
    for r in range(1, 4):
        x2, i2, g2 = new_x(), new_idx(r), new_x()
        sx.copy_(x2)
        sidx.copy_(i2)
        sg.copy_(g2)
        graph.replay()
        torch.cuda.synchronize()
        eager = copy.deepcopy(blk)
        eager.zero_grad(set_to_none=True)
        eager(x2, i2, sw).backward(g2)
        for a, b in zip(_block_members(blk), _block_members(eager)):
            assert torch.equal(a.codebooks.grad, b.codebooks.grad) and torch.equal(a.scales.grad, b.scales.grad), r


@gpu
def test_mixtral_deterministic_mode_refuses_the_codebook_gradient():
    blk = _trainable(_lattice_block(), codebooks=True, scales=False)
    x = to_dev(np.ones((8, 64)), torch.float16)
    idx = torch.zeros((8, 1), dtype=torch.int64, device=DEV)
    wts = torch.ones((8, 1), dtype=torch.float16, device=DEV)
    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="not deterministic"):
            blk(x, idx, wts).float().sum().backward()
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            blk(x, idx, wts).float().sum().backward()
        assert any("not deterministic" in str(r.message) for r in rec)
    finally:
        torch.use_deterministic_algorithms(False)
