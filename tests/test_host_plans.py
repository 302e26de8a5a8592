"""The host's launch plans, pinned on the CPU against a golden table.

aqlm_b200/csrc/plan.cuh holds the decisions the C-ABI makes before it launches anything: the wgmma GEMM plans (tile
height, split count, stage count, workspace), the Kx8 LUT GEMV plan and the cluster LUT GEMV's row blocking.  They are
pure arithmetic on the weight descriptor, the batch, the device's SM count and opt-in shared memory, and the
AQLM_B200_* switches, so a small C++ driver compiled against plan.cuh runs them here without a GPU.

The driver reads one case per line (`rows()` below; `set NAME VALUE` / `unset NAME` change an AQLM_B200_NAME switch)
and prints one result line per case.  Fields:
  gemm / gemm_t  ok tile_m m_tiles n_tiles n_tile ksplit stages total_kblocks counters_bytes partials_bytes
  lut            ok J n_slabs row_blocks rows_per_block smem partials_bytes
  cluster        eligible rows_per_block row_blocks   (0 0 when the given max-cluster count gives no cluster launch)
A plan that does not apply prints just `0`.

tests/golden/host_plans.json holds, per row label, the results of the same cases as computed by the planners before they
moved into plan.cuh (a harness that included capi.cu and called its planners directly).  Any change of plan -- a retuned cost-model
constant included -- fails here and must come with a regenerated table and a measurement that justifies it.
"""
import json
import os
import subprocess

from aqlm_b200 import _cabi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_plans.json")
SMEM_OPTIN = 232448  # H100 opt-in shared memory per block

# (num_codebooks, nbits, in_group_size, codes pointer offset): the 8 wgmma schemes
SCHEMES = [(K, nbits, 8, 0) for K in (1, 2, 4, 8) for nbits in (8, 16)]
# descriptors that some or all planners reject: in_group 16, K = 3, 12-bit codes, code pointers 8- / 4-byte aligned only
ODD_SCHEMES = [(1, 16, 16, 0), (3, 8, 8, 0), (1, 12, 8, 0), (1, 16, 8, 8), (2, 8, 8, 4)]
S1x16, S2x8 = (1, 16, 8, 0), (2, 8, 8, 0)
# (in_features, out_features); (64, 1) has out % 8 != 0
SHAPES = [(64, 1), (1152, 456), (4096, 4096), (4096, 14336), (14336, 4096), (8192, 28672)]
ODD_SHAPES = [(1032, 512), (4096, 4100)]  # in % 64 != 0; out % 8 != 0
BATCHES = [1, 2, 3, 7, 16, 17, 33, 64, 129, 300, 1024, 4096]
BIG_BATCHES = [6144, 8192, 16384]  # more than kGemmMaxTiles (8192) output tiles at some or every tile height
# a hypothetical 2112-SM device: with 132 SMs, 8192 tiles are 62 waves and no smaller tile height can win, so only a
# device this wide shows whether the forward tile search skips the heights with too many tiles
WIDE_SM_COUNT = 2112
MAX_CLUSTERS = [-1, 1, 7, 16, 66, 132]
# switch settings, each on a smaller grid of the plans it can change
FORCED_GEMM = ([("GEMM_TILE_M", v) for v in (127, 65, 40, 8, 200)] + [("GEMM_KSPLIT", v) for v in (1, 3, 16, 999)]
               + [("GEMM_STAGES", v) for v in (2, 4, 5)] + [("DISABLE_WGMMA", 1)])
FORCED_LUT = [("DISABLE_LUT", 1)] + [("LUT_CTAS_PER_SM", v) for v in (1, 3)]
FORCED_SHAPES = [(1152, 456), (4096, 4096), (8192, 28672)]
FORCED_BATCHES = [1, 17, 300, 4096]


def _w(scheme, shape):
    K, nbits, g, off = scheme
    return f"{K} {nbits} {g} {shape[0]} {shape[1]} {off}"


def _name(scheme, shape=None):
    K, nbits, g, off = scheme
    return f"{K}x{nbits} g{g}" + (f" +{off}" if off else "") + (f" {shape[0]}x{shape[1]}" if shape else "")


def rows():
    """The grid as (label, switch setting or None, driver case lines); the golden table holds one result list per label.

    Case lines: `gemm|gemm_t K nbits g in out codes_offset batch sm_count allow_split`, `lut K nbits g in out codes_offset
    sm_count` and `cluster K nbits g in out codes_offset input_offset batch max_clusters`.
    """
    for op in ("gemm", "gemm_t"):
        for sc in SCHEMES:
            for sh in SHAPES:  # every batch with split-K, then a few without a workspace and on a 114-SM device
                cols = ([f"{b} 132 1" for b in BATCHES] + [f"{b} 132 0" for b in (17, 300)]
                        + [f"{b} 114 1" for b in (17, 300)])
                yield f"{op} {_name(sc, sh)}", None, [f"{op} {_w(sc, sh)} {c}" for c in cols]
        for sc in (S1x16, (1, 8, 8, 0)):
            for sh in [(4096, 14336), (8192, 28672)]:
                cols = [f"{b} {sms} 1" for sms in (132, WIDE_SM_COUNT) for b in BIG_BATCHES]
                yield f"{op} {_name(sc, sh)} big", None, [f"{op} {_w(sc, sh)} {c}" for c in cols]
        for sc, sh in [(sc, (4096, 4096)) for sc in ODD_SCHEMES] + [(sc, sh) for sc in (S1x16, S2x8) for sh in ODD_SHAPES]:
            yield f"{op} {_name(sc, sh)}", None, [f"{op} {_w(sc, sh)} {b} 132 1" for b in (1, 17, 300)]
    for sc in SCHEMES + ODD_SCHEMES:
        yield f"lut {_name(sc)}", None, [f"lut {_w(sc, sh)} {sms}" for sh in SHAPES + ODD_SHAPES for sms in (132, 114)]
    for sc in [(1, 8, 8, 0), S2x8, (4, 8, 8, 0), S1x16, (2, 8, 8, 4)]:
        for sh in [(64, 1), (1152, 456), (4096, 4096), (4096, 14336), (1032, 512)]:
            cols = [f"0 1 {mc}" for mc in MAX_CLUSTERS] + ["2 1 132", "0 2 132"]  # + input 2-byte aligned, batch 2
            yield f"cluster {_name(sc, sh)}", None, [f"cluster {_w(sc, sh)} {c}" for c in cols]
    for name, value in FORCED_GEMM:
        for op in ("gemm", "gemm_t"):
            for sc in (S1x16, S2x8):
                yield (f"{name}={value} {op} {_name(sc)}", (name, value),
                       [f"{op} {_w(sc, sh)} {b} 132 1" for sh in FORCED_SHAPES for b in FORCED_BATCHES])
    for name, value in FORCED_LUT:
        schemes = [(K, 8, 8, 0) for K in (1, 2, 8)]
        yield (f"{name}={value} lut", (name, value),
               [f"lut {_w(sc, sh)} 132" for sc in schemes for sh in FORCED_SHAPES])
        yield (f"{name}={value} cluster", (name, value),
               [f"cluster {_w(sc, sh)} 0 1 132" for sc in schemes[:2] for sh in FORCED_SHAPES])


def run_driver(exe):
    """Run every row through the driver: {label: [result line per case]}."""
    lines, spans = [], []
    for label, setting, cases in rows():
        if setting:
            lines.append("set %s %s" % setting)
        spans.append((label, len(cases)))
        lines += cases
        if setting:
            lines.append(f"unset {setting[0]}")
    out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", check=True, capture_output=True,
                         text=True).stdout.splitlines()
    results, i = {}, 0
    for label, n in spans:
        results[label] = out[i:i + n]
        i += n
    assert i == len(out), f"driver printed {len(out)} lines for {i} cases"
    return results


DRIVER = r"""
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>

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
    std::string op, name, value;
    is >> op;
    if (op == "set" || op == "unset") {
      is >> name >> value;
      name = "AQLM_B200_" + name;
      if (op == "set") setenv(name.c_str(), value.c_str(), 1);
      else unsetenv(name.c_str());
      t.load();
      continue;
    }
    long long K, nbits, g, fin, fout, off;
    is >> K >> nbits >> g >> fin >> fout >> off;
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
    if (op == "lut") {
      is >> di.sm_count;
      const LutPlan L = lut_plan(w, 1, di, t);
      if (!L.ok) std::printf("0\n");
      else std::printf("1 %%d %%d %%d %%d %%zu %%zu\n", L.J, L.n_slabs, L.row_blocks, L.rows_per_block, L.smem, L.partials_bytes);
    } else if (op == "cluster") {
      long long input_off, batch;
      int mc;
      is >> input_off >> batch >> mc;
      const void* x = reinterpret_cast<const void*>(0x7f3000000000ull + input_off);
      if (!lut_cluster_eligible(w, x, batch, t)) {
        std::printf("0\n");
        continue;
      }
      const LutClusterRows r = lut_cluster_rows(w, mc);
      std::printf("1 %%d %%d\n", r.rows_per_block, r.row_blocks);
    } else {
      long long batch;
      int split;
      is >> batch >> di.sm_count >> split;
      const GemmPlan p = gemm_plan(w, batch, op != "gemm", 0, di, t, split != 0);
      if (!p.ok) std::printf("0\n");
      else std::printf("1 %%d %%d %%d %%d %%d %%d %%d %%zu %%zu\n", p.tile_m, p.m_tiles, p.n_tiles, p.n_tile, p.ksplit, p.stages,
                       p.total_kblocks, p.counters_bytes, p.partials_bytes);
    }
  }
  return 0;
}
"""


def test_host_plans_match_golden(tmp_path, monkeypatch):
    for k in list(os.environ):
        if k.startswith("AQLM_B200_"):
            monkeypatch.delenv(k)  # the driver starts from the shipped defaults
    src = tmp_path / "plans.cu"
    src.write_text(DRIVER % {"smem": SMEM_OPTIN})
    exe = tmp_path / "plans"
    # the library's flags without -shared / -fPIC: same language mode, same target
    flags = [f for f in _cabi.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    subprocess.run(["nvcc", *flags, "-I", _cabi.CSRC, "-o", str(exe), str(src)], check=True, capture_output=True,
                   text=True)
    got = run_driver(exe)
    with open(GOLDEN) as f:
        want = json.load(f)
    assert want.keys() == got.keys(), "the golden table was made for a different grid"
    cases = {label: cs for label, _, cs in rows()}
    diff = [f"{label}: {case}: want [{w}] got [{g}]" for label in want
            for case, w, g in zip(cases[label], want[label], got[label]) if w != g]
    n = sum(map(len, want.values()))
    assert not diff, f"{len(diff)} of {n} plans differ from the golden table; first ones:\n" + "\n".join(diff[:20])
