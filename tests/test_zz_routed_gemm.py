"""Routed (mixture-of-experts) wgmma GEMMs and the Mixtral expert block built on them.

A routed call runs E experts of one shape in ONE launch, forward or transposed; expert e applies to rows
[off[e], off[e+1]) of an input sorted by expert, and the offsets live in device memory.  Kernel results are checked
bit-exactly on the integer lattice of test_zz_gemm_exact.py: every expert draws its own lattice weight (codes, scales,
codebooks per segment) of one shape, so the exactness bounds are the shape's, and the exact result of a routed call is
each expert's exact result on its own rows.  Runs after test_zz_gemm_exact.py (`zz`): forced-plan cases set AQLM_B200_*
switches and restore them on the way out.

CPU: argument checks, the routed plans against tests/golden/routed_plans.json (a driver compiled against plan.cuh, as
in test_host_plans.py), the slot resolution of routing.cuh against a brute-force enumeration, the torch routing helper
against numpy, and loading a synthetic AQLM Mixtral checkpoint on the CPU.
"""
import ctypes
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from helpers import TOL_BF16, TOL_NORTH_STAR
from test_zz_gemm_exact import (DEV, DT_ID, DTYPES, WS_COUNTERS, _assert_tickets_clean, assert_exact, exact_forward,
                                exact_transposed, lattice_case, lattice_go, round_to, seed_of, tunables)
from test_zz_sharded_prefill import _descriptor

from oracle import aqlm_oracle as O

gpu = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "routed_plans.json")
SMEM_OPTIN = 232448  # H100 opt-in shared memory per block

# ==== the C++ driver: slot resolution and routed plans ================================================================
DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "plan.cuh"

using namespace aqlm_b200;

int main() {
  Tunables t;
  t.load();
  DeviceInfo di;
  di.max_smem_optin = %(smem)d;
  di.cc_major = 9;
  di.ok = true;
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream is(line);
    std::string op;
    is >> op;
    if (op == "slots") {  // slots rows n_tile E off_0 .. off_E: every slot of the grid, then one past it
      int rows, n, E;
      is >> rows >> n >> E;
      std::vector<int32_t> off(E + 1);
      for (auto& o : off) is >> o;
      const long long count = routed_slot_count(rows, E, n);
      std::printf("%%lld", count);
      for (long long s = 0; s <= count; ++s) {
        const RoutedSlot r = routed_slot(off.data(), E, rows, n, (int)s);
        std::printf(" %%d:%%d:%%d", r.expert, r.row0, r.row1);
      }
      std::printf("\n");
      continue;
    }
    long long K, nbits, g, fin, fout, off, rows;  // plan K nbits g in out codes_offset rows E sm_count split transposed
    int E, split, transposed;
    is >> K >> nbits >> g >> fin >> fout >> off >> rows >> E >> di.sm_count >> split >> transposed;
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
    const GemmPlan p = gemm_plan(w, rows, transposed != 0, E, di, t, split != 0);
    if (!p.ok) std::printf("0\n");
    else std::printf("1 %%d %%d %%d %%d %%d %%d %%d %%zu %%zu\n", p.tile_m, p.m_tiles, p.n_tiles, p.n_tile, p.ksplit, p.stages,
                     p.total_kblocks, p.counters_bytes, p.partials_bytes);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    from aqlm_b200 import _cabi

    d = tmp_path_factory.mktemp("routed_driver")
    src = d / "routed.cu"
    src.write_text(DRIVER % {"smem": SMEM_OPTIN})
    exe = d / "routed"
    flags = [f for f in _cabi.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    subprocess.run(["nvcc", *flags, "-I", _cabi.CSRC, "-o", str(exe), str(src)], check=True, capture_output=True, text=True)
    env = {k: v for k, v in os.environ.items() if not k.startswith("AQLM_B200_")}  # the shipped defaults

    def run(lines):
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", check=True, capture_output=True, text=True,
                             env=env).stdout.splitlines()
        assert len(out) == len(lines)
        return out

    return run


# ---- slot resolution ----------------------------------------------------------------------------------------------
def effective_offsets(off, rows):
    """Clamped into [0, rows], each raised to its predecessor (routing.cuh)."""
    c, prev = [], None
    for o in off:
        v = min(max(int(o), 0), rows)
        if prev is not None and v < prev:
            v = prev
        c.append(v)
        prev = v
    return c


def brute_force_slots(off, rows, n):
    c = effective_offsets(off, rows)
    out = []
    for e in range(len(off) - 1):
        for r0 in range(c[e], c[e + 1], n):
            out.append((e, r0, c[e + 1]))
    return out


SLOT_CASES = [  # (rows, n_tile, offsets)
    (64, 16, [0, 16, 32, 48, 64]),                 # balanced
    (40, 16, [0, 0, 40, 40, 40]),                  # all rows to one expert, empty first and last
    (50, 16, [0, 0, 20, 20, 50]),                  # empty first and middle experts
    (50, 32, [0, 10, 10, 50, 50]),                 # empty middle and last
    (4, 16, [0, 1, 2, 3, 4]),                      # single rows
    (300, 128, [0, 130, 261, 262, 300]),           # runs straddling tiles of N rows
    (77, 16, [0, 33, 77]),                         # rows not a multiple of N
    (40, 16, [0, 10, 5, 30, 40]),                  # a decreasing pair
    (40, 16, [0, 10, 999, 30, 40]),                # an offset past rows
    (40, 16, [-5, 10, -3, 30, 41]),                # negative offsets, a last one past rows
    (40, 16, [7, 10, 20, 30, 33]),                 # rows outside [off[0], off[E])
    (1, 128, [0, 0, 0, 1, 1, 1, 1, 1, 1]),         # one row, 8 experts
    (4096, 128, [0] + sorted(np.random.default_rng(3).integers(0, 4096, size=7).tolist()) + [4096]),
    (4096, 64, [0] * 8 + [4096]),                  # all to the last of 8
    (100, 16, [0] + [100] * 64),                   # 64 experts, all rows to the first
]


def test_slot_resolution_matches_brute_force(driver):
    lines = [f"slots {rows} {n} {len(off) - 1} " + " ".join(map(str, off)) for rows, n, off in SLOT_CASES]
    for (rows, n, off), got in zip(SLOT_CASES, driver(lines)):
        fields = got.split()
        count = int(fields[0])
        slots = [tuple(map(int, f.split(":"))) for f in fields[1:]]
        E = len(off) - 1
        m = min(E, rows)
        assert count == math.ceil((rows + m * (n - 1)) / n), (rows, n, off)
        want = brute_force_slots(off, rows, n)
        assert len(want) <= count, (rows, n, off)
        # slots [0, len(want)) are the tiles in expert order; every later slot (and one past the grid) is empty
        assert slots[:len(want)] == want, (rows, n, off, slots[:len(want)], want)
        assert all(s == (-1, 0, 0) for s in slots[len(want):]), (rows, n, off)
        covered = np.zeros(rows, dtype=np.int64)
        for e, r0, r1 in want:
            assert 0 <= r0 < r1 <= rows
            covered[r0:min(r0 + n, r1)] += 1
        c = effective_offsets(off, rows)
        inside = np.zeros(rows, dtype=bool)
        inside[c[0]:c[-1]] = True
        assert np.array_equal(covered, inside.astype(np.int64)), (rows, n, off)  # every row once, none outside


# ---- routed plans -------------------------------------------------------------------------------------------------
PLAN_SCHEMES = [(K, nbits, 8, 0) for K in (1, 2, 4, 8) for nbits in (8, 16)]
PLAN_SHAPES = [(4096, 28672), (14336, 4096), (1152, 256)]  # Mixtral-8x7B w1|w3 and w2, a small expert
PLAN_ROWS = [1, 2, 7, 8, 16, 64, 256, 1024, 2048, 8192]
PLAN_EXPERTS = [1, 8, 64]


def plan_rows():
    for tr in (0, 1):
        for sc in PLAN_SCHEMES:
            for sh in PLAN_SHAPES:
                K, nbits, g, off = sc
                cases = [f"{K} {nbits} {g} {sh[0]} {sh[1]} {off} {r} {E} 132 1 {tr}" for E in PLAN_EXPERTS
                         for r in PLAN_ROWS]
                cases += [f"{K} {nbits} {g} {sh[0]} {sh[1]} {off} {r} 8 132 0 {tr}" for r in (64, 2048)]
                yield f"{'t' if tr else 'f'} {K}x{nbits} {sh[0]}x{sh[1]}", cases
        # refused: in_group 16, 3 codebooks, 8-byte aligned codes, in % 64 / out % 8, more slots than a grid holds
        odd = [(1, 16, 16, 4096, 4096, 0), (3, 8, 8, 4096, 4096, 0), (1, 16, 8, 4096, 4096, 8), (2, 8, 8, 1032, 512, 0),
               (2, 8, 8, 4096, 4100, 0)]
        yield f"{'t' if tr else 'f'} odd", [f"{K} {nb} {g} {i} {o} {off} 64 8 132 1 {tr}" for K, nb, g, i, o, off in odd] + \
            [f"1 16 8 4096 4096 0 {10 ** 7} 8 132 1 {tr}"]


def run_plans(driver):
    """Every row of plan_rows() through the driver: {label: [result line per case]}."""
    labels = list(plan_rows())
    lines = [f"plan {c}" for _, cs in labels for c in cs]
    out, got, i = driver(lines), {}, 0
    for label, cs in labels:
        got[label] = out[i:i + len(cs)]
        i += len(cs)
    return got


def test_routed_plans_match_golden(driver):
    labels = list(plan_rows())
    got = run_plans(driver)
    with open(GOLDEN) as f:
        want = json.load(f)
    assert want.keys() == got.keys(), "the golden table was made for a different grid"
    cases = dict(labels)
    diff = [f"{label}: {case}: want [{w}] got [{g}]" for label in want
            for case, w, g in zip(cases[label], want[label], got[label]) if w != g]
    assert not diff, f"{len(diff)} routed plans differ from the golden table; first ones:\n" + "\n".join(diff[:20])


def test_routed_plan_properties(driver):
    """Independent of the table: N is the MMA width of the balanced share, the grid covers every routing, the split
    stays within the ticket words, the workspace is [m_tiles][slots][ksplit][N][128] fp32."""
    lines, params = [], []
    for tr in (0, 1):
        for rows in PLAN_ROWS:
            for E in PLAN_EXPERTS:
                lines.append(f"plan 1 16 8 4096 28672 0 {rows} {E} 132 1 {tr}")
                params.append((tr, rows, E))
    for (tr, rows, E), line in zip(params, driver(lines)):
        f = line.split()
        assert f[0] == "1", line
        tile_m, m_tiles, slots, n_tile, ksplit = map(int, f[1:6])
        partials = int(f[9])
        m = min(E, rows)
        n = 16
        while n < 128 and n < math.ceil(rows / m):
            n <<= 1
        assert n_tile == n and slots == math.ceil((rows + m * (n - 1)) / n), line
        assert m_tiles == math.ceil((4096 if tr else 28672) / tile_m)
        assert ksplit == 1 or m_tiles * slots <= 8192
        assert partials == (m_tiles * slots * ksplit * n_tile * 128 * 4 if ksplit > 1 else 0)


# ---- argument checks ----------------------------------------------------------------------------------------------
def _call(L, transposed, w, seg, n_seg, E=4, off=16, b=16, y=16, rows=64):
    seg_arr = None if seg is None else (ctypes.c_int64 * max(len(seg), 1))(*seg)
    fn = L.aqlm_b200_matmat_dequant_transposed_routed if transposed else L.aqlm_b200_matmat_dequant_routed
    return fn(ctypes.byref(w), seg_arr, n_seg, E, off, b, y, rows, None, 0, None)


@pytest.mark.parametrize("transposed", [False, True], ids=["forward", "transposed"])
def test_routed_argument_checks_without_a_device(transposed):
    from aqlm_b200 import _cabi

    L = _cabi.lib()
    S, U = _cabi.ERR_SHAPE, _cabi.ERR_UNSUPPORTED
    w = _descriptor()  # 1024 -> 256, 1x16, in_group 8
    # descriptor first: a bad one wins over every later error
    bad = _descriptor(in_features=1004)
    assert _call(L, transposed, bad, [64], 5, E=0, off=None) == S
    assert b"bad shape" in L.aqlm_b200_last_error()
    nosc = _descriptor()
    nosc.scales = None
    assert _call(L, transposed, nosc, [256], 1) == S
    # segments next (before the expert count and the pointers)
    assert _call(L, transposed, w, [64, 64, 64, 32, 32], 5, E=0, off=None) == S
    assert b"1..4 segments" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, [64] * 4, 0) == S
    assert _call(L, transposed, w, None, 2) == S
    assert _call(L, transposed, w, [128, 64], 2, E=0) == S
    assert b"add up" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, [256, 0], 2) == S
    # then the expert count
    for E in (0, -1, 65):
        assert _call(L, transposed, w, [128, 128], 2, E=E, off=None) == S
        assert b"experts" in L.aqlm_b200_last_error()
    # then NULL offsets / buffers
    assert _call(L, transposed, w, None, 1, off=None, b=None) == S
    assert b"offsets" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, None, 1, b=None) == S
    assert _call(L, transposed, w, None, 1, y=None) == S
    assert _call(L, transposed, w, None, 1, rows=-1) == S
    # layouts the wgmma kernels do not take: ERR_UNSUPPORTED, as for the grouped GEMM
    for kw in (dict(in_group_size=16), dict(num_codebooks=3, nbits_per_codebook=8), dict(nbits_per_codebook=12)):
        assert _call(L, transposed, _descriptor(**kw), [128, 128], 2, E=64) == U, kw
        assert b"routed" in L.aqlm_b200_last_error()
    assert _call(L, transposed, w, None, 1, b=24) == U  # input / grad_output not 16-byte aligned
    assert _call(L, transposed, _descriptor(codes=24), None, 1) == U
    if transposed:
        assert _call(L, transposed, _descriptor(out_features=252), None, 1) == U
        assert b"% 8" in L.aqlm_b200_last_error()
    else:
        assert _call(L, transposed, _descriptor(in_features=1056, num_codebooks=4, nbits_per_codebook=8), None, 1) == U
        assert b"% 64" in L.aqlm_b200_last_error()
    # rows == 0: nothing to do, no device needed (seg_rows NULL with n_seg 1: a plain expert linear)
    assert _call(L, transposed, w, None, 1, rows=0) == _cabi.OK
    assert _call(L, transposed, w, [200, 56], 2, E=64, rows=0) == _cabi.OK
    assert L.aqlm_b200_matmat_dequant_routed_workspace_bytes(ctypes.byref(w), 0, 64, int(transposed)) == 0
    if torch.cuda.is_available():
        return  # the calls below would launch on the dummy pointers
    for seg in ([256], [200, 56], [64, 64, 64, 64]):
        assert _call(L, transposed, w, seg, len(seg)) in (_cabi.ERR_CUDA, _cabi.ERR_ARCH)


# ---- the torch routing helper -------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,k,E", [(1, 2, 8), (7, 2, 4), (300, 2, 8), (64, 3, 5), (33, 1, 64)])
def test_route_matches_numpy(T, k, E):
    from aqlm_b200.moe import route

    rng = np.random.default_rng(T * 100 + k * 10 + E)
    ids = rng.integers(0, E, size=(T, k))
    ids[rng.random((T, k)) < 0.15] = E        # out of range: transformers skips expert_idx == num_experts
    ids[rng.random((T, k)) < 0.05] = -1       # and negative ids are dropped too
    order, offsets, valid = route(torch.from_numpy(ids), E)
    flat = ids.reshape(-1)
    ok = (flat >= 0) & (flat < E)
    key = np.where(ok, flat, E)
    want_order = np.argsort(key, kind="stable")
    want_off = np.searchsorted(key[want_order], np.arange(E + 1), side="left")
    assert np.array_equal(order.numpy(), want_order)
    assert offsets.dtype == torch.int32 and np.array_equal(offsets.numpy(), want_off)
    assert np.array_equal(valid.numpy(), ok)
    assert offsets[-1].item() == ok.sum()


# ---- the Mixtral checkpoint ---------------------------------------------------------------------------------------
def write_synthetic_mixtral(path, K, nbits, seed=0, hidden=128, inter=256, layers=2, experts=4, top_k=2, vocab=96):
    """An AQLM Mixtral checkpoint in the reference's format, with the per-expert names `block_sparse_moe.experts.{e}.
    w{1,2,3}`.  Returns (MixtralConfig, dense state dict with the dequantized weights, the checkpoint's state dict)."""
    from transformers import MixtralConfig, MixtralForCausalLM

    from aqlm_b200 import hf

    cfg = MixtralConfig(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers, num_attention_heads=4,
                        num_key_value_heads=2, num_local_experts=experts, num_experts_per_tok=top_k, vocab_size=vocab,
                        max_position_embeddings=64, tie_word_embeddings=False)
    torch.manual_seed(seed)
    dense = MixtralForCausalLM(cfg).half()
    rng = np.random.default_rng(seed)

    def quantize(prefix, out_f, in_f):
        codes = rng.integers(0, 2 ** nbits, size=(out_f, in_f // 8, K))
        cb = (rng.standard_normal((K, 2 ** nbits, 1, 8)) * (0.08 / K ** 0.5)).astype(np.float16)
        sc = (0.75 + 0.5 * rng.random((out_f, 1, 1, 1))).astype(np.float16)
        ckpt.update(hf.quantized_state_entries(prefix, torch.from_numpy(codes), torch.from_numpy(cb), torch.from_numpy(sc),
                                               nbits))
        return torch.from_numpy(O.dequantize_weight(codes, cb.astype(np.float32), sc.astype(np.float32))).half()

    ckpt, dense_sd, not_quantized = {}, {}, []
    for name, p in dense.state_dict().items():
        if name.endswith("_proj.weight") and ".self_attn." in name:
            dense_sd[name] = quantize(name[: -len(".weight")], *p.shape)
        elif name.endswith("experts.gate_up_proj"):
            pre = name[: -len("mlp.experts.gate_up_proj")] + "block_sparse_moe.experts"
            dense_sd[name] = torch.stack([torch.cat([quantize(f"{pre}.{e}.w1", inter, hidden),
                                                     quantize(f"{pre}.{e}.w3", inter, hidden)]) for e in range(experts)])
        elif name.endswith("experts.down_proj"):
            pre = name[: -len("mlp.experts.down_proj")] + "block_sparse_moe.experts"
            dense_sd[name] = torch.stack([quantize(f"{pre}.{e}.w2", hidden, inter) for e in range(experts)])
        else:
            ckpt[name.replace(".mlp.", ".block_sparse_moe.")] = p.half()
            dense_sd[name] = p.half()
            not_quantized.append(name.replace(".mlp.", ".block_sparse_moe."))
    not_quantized.append("lm_head.weight")  # parameter names only, as the reference converter writes them
    hf.save_quantized_checkpoint(path, cfg.to_dict(), ckpt,
                                 hf.quantization_config_dict(K, nbits, linear_weights_not_to_quantize=not_quantized))
    return cfg, dense_sd, ckpt


@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_load_quantized_mixtral_on_cpu(tmp_path, K, nbits):
    pytest.importorskip("transformers")
    import aqlm_b200
    from aqlm_b200 import hf
    from aqlm_b200.moe import QuantizedMixtralExperts

    cfg, _, ckpt = write_synthetic_mixtral(str(tmp_path / "m"), K, nbits)
    assert any(".block_sparse_moe.experts.3.w2.codes" in k for k in ckpt)
    model = hf.load_quantized_mixtral(str(tmp_path / "m"), torch.float16, "cpu")
    sd = model.state_dict()
    assert not any(t.is_meta for t in sd.values())
    # the strict load left nothing out and nothing over: the model's keys are the checkpoint's, renamed
    assert set(sd) == {k.replace(".block_sparse_moe.", ".mlp.") for k in ckpt}
    n_exp = 0
    for name, mod in model.named_modules():
        if name.endswith("mlp.experts"):
            assert type(mod) is QuantizedMixtralExperts and mod.routed
            n_exp += 1
        if name.endswith(("_proj", ".w1", ".w2", ".w3")):
            assert type(mod) is aqlm_b200.QuantizedLinear, (name, type(mod))
            src = name.replace(".mlp.", ".block_sparse_moe.")
            assert torch.equal(mod.codes, ckpt[f"{src}.codes"]) and mod.codes.dtype == ckpt[f"{src}.codes"].dtype
            assert torch.equal(mod.codebooks, ckpt[f"{src}.codebooks"]) and torch.equal(mod.scales, ckpt[f"{src}.scales"])
    assert n_exp == cfg.num_hidden_layers
    # members are views of the stacked buffers the routed launches read
    ex = model.model.layers[0].mlp.experts
    c13 = ex._w13[0]
    assert ex.expert(1).w3.codes.data_ptr() == c13[1, cfg.intermediate_size:].data_ptr()
    assert ex.expert(2).w2.codebooks.data_ptr() == ex._w2[1][2, 0].data_ptr()
    assert isinstance(model.lm_head, torch.nn.Linear)


def test_replace_mixtral_experts_on_meta():
    """No dense expert tensor: the replacement happens on the meta device, Mixtral-8x7B's shape included."""
    pytest.importorskip("transformers")
    from transformers import MixtralConfig, MixtralForCausalLM

    from aqlm_b200 import hf
    from aqlm_b200.moe import QuantizedMixtralExperts

    cfg = MixtralConfig(num_hidden_layers=2, vocab_size=128)  # 4096 hidden, 14336 intermediate, 8 experts
    cfg.quantization_config = hf.quantization_config_dict(1, 16)
    with torch.device("meta"):
        model = MixtralForCausalLM(cfg)
    assert hf.replace_mixtral_experts(model) == 2
    ex = model.model.layers[1].mlp.experts
    assert type(ex) is QuantizedMixtralExperts and ex._w13[0].is_meta
    assert tuple(ex._w13[0].shape) == (8, 2 * 14336, 4096 // 8, 1) and tuple(ex._w2[1].shape) == (8, 1, 1, 65536, 1, 8)
    assert "model.layers.1.mlp.experts.7.w2.codes" in model.state_dict()


# ==== GPU: the routed kernels, bit-exact ==============================================================================
GEMM_IN = 1152                                 # 18 k-blocks
SEGS = {1: [256], 2: [200, 56]}                # per expert; the 2-segment end lies inside a 128-row tile
ROUTINGS = {                                   # rows, offsets (4 experts)
    "balanced": (64, [0, 16, 32, 48, 64]),
    "all-to-one": (40, [0, 0, 40, 40, 40]),
    "empty": (50, [0, 0, 20, 20, 50]),
    "single-rows": (4, [0, 1, 2, 3, 4]),
    "straddle": (300, [0, 130, 261, 262, 300]),
    "malformed": (40, [-5, 10, 5, 30, 41]),     # clamped: experts [0,10), [10,10), [10,30), [30,40)
}
SCHEMES = [(1, 16), (2, 8), (8, 8), (1, 8)]


def routed_case(seed, fin, segs, K, nbits, E, dtype, rows):
    """E experts of one lattice shape (codebooks per segment), stacked as the routed call takes them."""
    out = sum(segs)
    experts = []
    for e in range(E):
        base = lattice_case(seed_of(seed, "w", e), fin, out, K, nbits, bias=False, dtype=dtype)
        cbs = [lattice_case(seed_of(seed, "cb", e, i), fin, n, K, nbits, dtype=dtype)["codebooks"] for i, n in enumerate(segs)]
        experts.append(dict(base, codebooks_seg=cbs))
    x = lattice_go(seed_of(seed, "x"), rows, fin)
    dev = lambda a, dt: torch.from_numpy(np.asarray(a)).to(dt).to(DEV)  # noqa: E731
    t = dict(x=dev(x, dtype),
             codes=torch.stack([torch.from_numpy(c["codes"]) for c in experts]).to(DEV),
             codebooks=torch.stack([torch.stack([dev(cb, dtype) for cb in c["codebooks_seg"]]) for c in experts]).contiguous(),
             scales=torch.stack([dev(c["scales"], dtype) for c in experts]).contiguous())
    return experts, x, t


def expert_rows(c, segs, x, go=None):
    """Exact forward (go None) or transposed result of one expert on its rows, segment by segment."""
    res, off = [], 0
    for i, n in enumerate(segs):
        seg = dict(codes=c["codes"][off:off + n], codebooks=c["codebooks_seg"][i], scales=c["scales"][off:off + n],
                   bias=None, x=x)
        res.append(exact_forward(seg) if go is None else exact_transposed(seg, go[:, off:off + n]))
        off += n
    return np.concatenate(res, axis=1) if go is None else sum(res)


def _offsets(off):
    return torch.tensor(off, dtype=torch.int32, device=DEV)


def _run(fn, *args, transposed=False, rows=None, E=4):
    """One routed call; returns (result, workspace bytes asked for, launches)."""
    from aqlm_b200 import _cabi
    from aqlm_b200.inference_kernels import cuda_kernel

    before = _cabi.launch_count()
    y = fn(*args)
    launches = _cabi.launch_count() - before
    assert y is not None, "the routed GEMM refused a layout it covers"
    w = cuda_kernel._routed_weight(args[1], args[2], args[3], None if len(args) < 6 else args[5])[0]
    need = _cabi.lib().aqlm_b200_matmat_dequant_routed_workspace_bytes(ctypes.byref(w), E, rows, int(transposed))
    if need:
        _assert_tickets_clean("routed")
    return y, need, launches


def _exact_routed_forward(experts, segs, x, off, rows, fill):
    c = effective_offsets(off, rows)
    ref = np.full((rows, sum(segs)), fill, dtype=np.float64)
    for e, ce in enumerate(experts):
        if c[e + 1] > c[e]:
            ref[c[e]:c[e + 1]] = expert_rows(ce, segs, x[c[e]:c[e + 1]])
    return ref


def _fwd_params():
    return [pytest.param(K, nbits, dtype, n_seg, r, id=f"{K}x{nbits}-{DT_ID[dtype]}-seg{n_seg}-{r}")
            for K, nbits in SCHEMES for dtype in DTYPES for n_seg in (1, 2) for r in ROUTINGS]


@gpu
@pytest.mark.parametrize("K,nbits,dtype,n_seg,routing", _fwd_params())
def test_routed_forward_exact(K, nbits, dtype, n_seg, routing):
    from aqlm_b200.inference_kernels import cuda_kernel

    segs = SEGS[n_seg]
    rows, off = ROUTINGS[routing]
    experts, x, t = routed_case(seed_of("rfwd", K, nbits, n_seg, routing), GEMM_IN, segs, K, nbits, 4, dtype, rows)
    seg_rows = segs if n_seg > 1 else None
    y, _, launches = _run(cuda_kernel.matmat_dequant_routed, t["x"], t["codes"], t["codebooks"], t["scales"],
                          _offsets(off), seg_rows, rows=rows)
    assert launches == 1 and y.shape == (rows, sum(segs))
    c = effective_offsets(off, rows)
    got = y.float().cpu().numpy()[c[0]:c[-1]]  # rows of no expert are left unwritten
    ref = round_to(_exact_routed_forward(experts, segs, x, off, rows, 0.0), dtype)[c[0]:c[-1]]
    assert_exact(got, ref, f"routed {K}x{nbits} {routing} seg{n_seg}")


@gpu
@pytest.mark.parametrize("K,nbits,dtype,n_seg,routing", _fwd_params())
def test_routed_transposed_exact(K, nbits, dtype, n_seg, routing):
    from aqlm_b200.inference_kernels import cuda_kernel

    segs = SEGS[n_seg]
    rows, off = ROUTINGS[routing]
    experts, _, t = routed_case(seed_of("rt", K, nbits, n_seg, routing), GEMM_IN, segs, K, nbits, 4, dtype, 1)
    go = lattice_go(seed_of("rt-go", K, nbits, n_seg, routing), rows, sum(segs))
    gx, _, launches = _run(cuda_kernel.matmat_dequant_transposed_routed, torch.from_numpy(go).to(dtype).to(DEV),
                           t["codes"], t["codebooks"], t["scales"], _offsets(off), segs if n_seg > 1 else None,
                           transposed=True, rows=rows)
    assert launches == 1 and gx.shape == (rows, GEMM_IN)
    c = effective_offsets(off, rows)
    ref = np.zeros((rows, GEMM_IN))
    for e, ce in enumerate(experts):
        if c[e + 1] > c[e]:
            ref[c[e]:c[e + 1]] = expert_rows(ce, segs, None, go[c[e]:c[e + 1]])
    assert_exact(gx.float().cpu().numpy()[c[0]:c[-1]], round_to(ref, dtype)[c[0]:c[-1]],
                 f"routed transposed {K}x{nbits} {routing} seg{n_seg}")


FORCED = [(tm, ks) for tm in (127, 40) for ks in (1, 3, 16)]


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
@pytest.mark.parametrize("tile_m,ksplit", FORCED, ids=[f"tm{tm}-ks{ks}" for tm, ks in FORCED])
def test_routed_forced_plan_exact(K, nbits, tile_m, ksplit):
    """Forced tile heights (straddling the 200-row segment end) and split counts, forward and transposed; the split
    shows in the workspace: counters + [m_tiles][slots][ksplit][N][128] fp32."""
    from aqlm_b200.inference_kernels import cuda_kernel

    segs, (rows, off) = [200, 56], ROUTINGS["straddle"]
    dtype = DTYPES[(tile_m + ksplit) % 2]
    experts, x, t = routed_case(seed_of("rforced", K, nbits, tile_m, ksplit), GEMM_IN, segs, K, nbits, 4, dtype, rows)
    go = lattice_go(seed_of("rforced-go", K, nbits), rows, sum(segs))
    n = 128  # balanced share ceil(300 / 4) = 75 rows
    slots = math.ceil((rows + 4 * (n - 1)) / n)
    with tunables(gemm_tile_m=tile_m, gemm_ksplit=ksplit):
        y, need, launches = _run(cuda_kernel.matmat_dequant_routed, t["x"], t["codes"], t["codebooks"], t["scales"],
                                 _offsets(off), segs, rows=rows)
        gx, need_t, launches_t = _run(cuda_kernel.matmat_dequant_transposed_routed,
                                      torch.from_numpy(go).to(dtype).to(DEV), t["codes"], t["codebooks"], t["scales"],
                                      _offsets(off), segs, transposed=True, rows=rows)
    assert launches == 1 and launches_t == 1
    ks = min(ksplit, GEMM_IN // 64)
    assert need == (WS_COUNTERS + math.ceil(256 / tile_m) * slots * ks * n * 128 * 4 if ks > 1 else 0), need
    ks_t = min(ksplit, 4)
    assert need_t == (WS_COUNTERS + math.ceil(GEMM_IN / 128) * slots * ks_t * n * 128 * 4 if ks_t > 1 else 0), need_t
    assert_exact(y.float().cpu().numpy(), round_to(_exact_routed_forward(experts, segs, x, off, rows, 0.0), dtype),
                 f"routed {K}x{nbits} tile_m={tile_m} ksplit={ksplit}", tile_m=tile_m)
    ref = np.concatenate([expert_rows(ce, segs, None, go[off[e]:off[e + 1]]) for e, ce in enumerate(experts)
                          if off[e + 1] > off[e]])
    assert_exact(gx.float().cpu().numpy(), round_to(ref, dtype), f"routed transposed {K}x{nbits} ksplit={ksplit}")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
@pytest.mark.parametrize("rows", [9, 300])
def test_one_expert_equals_the_plain_gemm(K, nbits, dtype, rows):
    """E = 1 with offsets [0, rows]: the result is the plain GEMM's, bit for bit, in both directions."""
    from aqlm_b200.inference_kernels import cuda_kernel

    experts, x, t = routed_case(seed_of("r1", K, nbits, rows), GEMM_IN, [256], K, nbits, 1, dtype, rows)
    off = _offsets([0, rows])
    y = cuda_kernel.matmat_dequant_routed(t["x"], t["codes"], t["codebooks"], t["scales"], off)
    plain = cuda_kernel.matmat_dequant(t["x"], t["codes"][0], t["codebooks"][0, 0], t["scales"][0])
    assert torch.equal(y, plain)
    go = torch.from_numpy(lattice_go(seed_of("r1-go", rows), rows, 256)).to(dtype).to(DEV)
    gx = cuda_kernel.matmat_dequant_transposed_routed(go, t["codes"], t["codebooks"], t["scales"], off)
    assert torch.equal(gx, cuda_kernel.matmat_dequant_transposed(go, t["codes"][0], t["codebooks"][0, 0], t["scales"][0]))


# ==== GPU: the expert block ===========================================================================================
def _experts_pair(seed, K, nbits, E=4, hidden=128, inter=256, dtype=torch.float16):
    """A QuantizedMixtralExperts with random weights and transformers' dense MixtralExperts holding them dequantized
    (in fp32: the reference of the same arithmetic)."""
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts

    from aqlm_b200.moe import QuantizedMixtralExperts

    cfg = MixtralConfig(hidden_size=hidden, intermediate_size=inter, num_local_experts=E)
    dense = MixtralExperts(cfg)
    q = QuantizedMixtralExperts(E, hidden, inter, dense.act_fn, 8, 1, K, nbits, device="cpu", dtype=dtype)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in [mod for mod in q.modules() if mod.__class__.__name__ == "QuantizedLinear"]:
            lo, hi = (-128, 128) if nbits <= 8 else (-2 ** 15, 2 ** 15)
            m.codes.copy_(torch.randint(lo, hi, m.codes.shape, generator=g, dtype=torch.int32).to(m.codes.dtype))
            m.codebooks.copy_((torch.randn(m.codebooks.shape, generator=g) * (0.3 / K ** 0.5)).to(dtype))
            m.scales.copy_((0.75 + 0.5 * torch.rand(m.scales.shape, generator=g)).to(dtype))
    q = q.to(DEV)

    def deq(m):
        from aqlm_b200.inference_kernels import cuda_kernel

        return cuda_kernel.dequant(m.codes, m.codebooks, m.scales).float()

    with torch.no_grad():
        dense.gate_up_proj.copy_(torch.stack([torch.cat([deq(q.expert(e).w1), deq(q.expert(e).w3)]) for e in range(E)]))
        dense.down_proj.copy_(torch.stack([deq(q.expert(e).w2) for e in range(E)]))
    return q, dense.to(DEV).float()


def _routing(seed, T, k, E, drop=False):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn((T, E), generator=g)
    w, idx = torch.topk(torch.softmax(logits, -1), k, dim=-1)
    w = w / w.sum(-1, keepdim=True)
    if drop:
        idx[::3, -1] = E  # transformers skips expert_idx == num_experts
    return idx.to(DEV), w.to(DEV)


def _rel(a, b):
    return ((a.float() - b.float()).abs().mean() / b.float().abs().mean()).item()


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
@pytest.mark.parametrize("T", [1, 2, 3, 4, 5, 6, 7, 8, 300])
def test_experts_match_dense_mixtral_experts(K, nbits, T):
    from aqlm_b200 import _cabi

    q, dense = _experts_pair(seed_of("moe", K, nbits), K, nbits)
    idx, w = _routing(seed_of("route", T), T, 2, 4, drop=(T == 300))
    x0 = torch.randn((T, 128), generator=torch.Generator().manual_seed(T)).half().to(DEV)
    gy = torch.randn((T, 128), generator=torch.Generator().manual_seed(T + 1)).half().to(DEV)

    x, wq = x0.clone().requires_grad_(True), w.clone().requires_grad_(True)
    before = _cabi.launch_count()
    y = q(x, idx, wq)
    assert _cabi.launch_count() - before == 2, "one routed launch per projection"
    before = _cabi.launch_count()
    y.backward(gy)
    assert _cabi.launch_count() - before == 2, "one routed transposed launch per projection"

    # the dense block gets dropped slots as a valid id with weight 0 (its one_hot takes no out-of-range id)
    keep = idx < 4
    xd, wd = x0.float().clone().requires_grad_(True), w.clone().requires_grad_(True)
    yd = dense(xd, torch.where(keep, idx, 0), wd * keep)
    yd.backward(gy.float())
    assert y.dtype == torch.float16
    assert _rel(y, yd) < TOL_NORTH_STAR, _rel(y, yd)
    assert _rel(x.grad, xd.grad) < TOL_NORTH_STAR, _rel(x.grad, xd.grad)
    # d/dw[t, j] = y[pair(t, j)] . g[t]: a dot product of the fp16-rounded expert output, with cancellation, against
    # the fp32 reference's; bf16-level tolerance
    assert _rel(wq.grad, wd.grad) < TOL_BF16, _rel(wq.grad, wd.grad)
    if T == 300:  # dropped slots contribute nothing and get no gradient
        assert bool((wq.grad[::3, -1] == 0).all())


@gpu
def test_experts_cuda_graph_replays_with_new_routing():
    q, _ = _experts_pair(seed_of("graph"), 1, 16)
    T, k, E = 8, 2, 4
    sx = torch.randn((T, 128), generator=torch.Generator().manual_seed(0)).half().to(DEV)
    sidx, sw = _routing(0, T, k, E)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                q(sx, sidx, sw)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            sy = q(sx, sidx, sw)
        for r in range(1, 6):
            idx, w = _routing(r, T, k, E, drop=(r == 5))
            if r == 3:
                idx[:] = 2  # every token to one expert
            sidx.copy_(idx)
            sw.copy_(w)
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(sy, q(sx, idx, w)), r


@gpu
def test_experts_fallback_for_a_refused_scheme():
    """in_group 16: the routed GEMM does not take it; the block runs the transformers loop over its members."""
    from transformers import MixtralConfig
    from transformers.models.mixtral.modeling_mixtral import MixtralExperts

    from aqlm_b200.moe import QuantizedMixtralExperts

    act = MixtralExperts(MixtralConfig(hidden_size=128, intermediate_size=256, num_local_experts=4)).act_fn
    q = QuantizedMixtralExperts(4, 128, 256, act, 16, 1, 1, 16, device="cpu", dtype=torch.float16)
    assert not q.routed
    with torch.no_grad():
        for p in q.parameters():
            if p.is_floating_point():
                p.copy_(torch.rand(p.shape) * 0.1 + 0.5)
            else:
                p.copy_(torch.randint(-100, 100, p.shape).to(p.dtype))
    q = q.to(DEV)
    idx, w = _routing(1, 16, 2, 4)
    x = torch.randn((16, 128), generator=torch.Generator().manual_seed(1)).half().to(DEV)
    with torch.no_grad():
        y = q(x, idx, w)
        ref = torch.zeros_like(x, dtype=torch.float32)
        for t in range(16):
            for j in range(2):
                m = q.expert(int(idx[t, j]))
                xt = x[t:t + 1]
                ref[t] += (m.w2(act(m.w1(xt)) * m.w3(xt)).float() * w[t, j])[0]
    assert _rel(y, ref) < TOL_NORTH_STAR


@gpu
@pytest.mark.parametrize("K,nbits", [(1, 16), (2, 8)])
def test_mixtral_checkpoint_logits_match_dense(tmp_path, K, nbits):
    from transformers import MixtralForCausalLM

    from aqlm_b200 import hf

    cfg, dense_sd, _ = write_synthetic_mixtral(str(tmp_path / "m"), K, nbits, seed=5)
    model = hf.load_quantized_mixtral(str(tmp_path / "m"), torch.float16, DEV)
    assert hf.fuse_shared_input_linears(model) == cfg.num_hidden_layers  # q/k/v; the experts are already routed
    dense = MixtralForCausalLM(cfg).half()
    dense.load_state_dict(dense_sd)
    dense = dense.to(DEV).eval()
    ids = torch.randint(0, cfg.vocab_size, (4, 5), device=DEV, generator=torch.Generator(DEV).manual_seed(1))
    with torch.no_grad():
        for batch in (ids[:1, :1], ids):  # decode of one token and a 20-row prefill
            lq, ld = model(batch).logits.float(), dense(batch).logits.float()
            assert _rel(lq, ld) < 5e-3, _rel(lq, ld)
