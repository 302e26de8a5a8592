// Launch plans of the C-ABI: which kernel shape serves a call, as pure functions of the weight descriptor, the batch,
// the device (SM count, opt-in shared memory) and the experiment switches.  No globals, no CUDA calls: the planners run
// on a machine without a GPU, which is how tests/test_host_plans.py pins them.
#pragma once

#include <cstdlib>

#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "gemm_wgmma_t.cuh"
#include "gemm_wgrad.cuh"
#include "gemv.cuh"
#include "gemv_lut.cuh"

namespace aqlm_b200 {

inline int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

// Experiment switches (environment variables), read ONCE per process -- not per launch -- and again only when a tool
// calls aqlm_b200_reload_tunables() after changing the environment.  Defaults are the shipped configuration.
struct Tunables {
  int pdl, gemv_ctas_per_sm, force_generic;
  int disable_lut, lut_ctas_per_sm, lut_batch_loop;
  int disable_wgmma, gemm_stages, gemm_ksplit, gemm_gather_mode, gemm_tile_m;
  void load() {
    pdl = env_int("AQLM_B200_PDL", 1);
    gemv_ctas_per_sm = env_int("AQLM_B200_GEMV_CTAS_PER_SM", 1);
    force_generic = env_int("AQLM_B200_FORCE_GENERIC", 0);
    disable_lut = env_int("AQLM_B200_DISABLE_LUT", 0);
    lut_ctas_per_sm = env_int("AQLM_B200_LUT_CTAS_PER_SM", 2);  // 128 regs x 256 threads: registers allow 2
    lut_batch_loop = env_int("AQLM_B200_LUT_BATCH_LOOP", 1);  // batch 2-3 on 256-entry codebooks: one LUT launch per row
    disable_wgmma = env_int("AQLM_B200_DISABLE_WGMMA", 0);
    gemm_stages = env_int("AQLM_B200_GEMM_STAGES", 0);
    gemm_ksplit = env_int("AQLM_B200_GEMM_KSPLIT", 0);
    gemm_gather_mode = env_int("AQLM_B200_GEMM_GATHER_MODE", -1);  // -1: per scheme (1x16: ld.global.cg, no L1 allocation of the 1 MiB codebook's lines; 256-entry codebooks: L1-resident)
    gemm_tile_m = env_int("AQLM_B200_GEMM_TILE_M", 0);            // 0: chosen by the plan
  }
};

constexpr size_t kWsCountersBytes = 65536;  // fixed counter region at the head of every workspace (16384 words)
constexpr int kGemmMaxTiles = 8192;  // split-K / LUT tickets use counter words [0, 8192); the LUT GEMV's generation words follow

// ---- Kx8 LUT GEMV (workspace kernel) ----------------------------------------------------------------------------
struct LutPlan {
  bool ok = false;
  int J = 32, n_slabs = 0, row_blocks = 0, rows_per_block = 0;
  size_t smem = 0, partials_bytes = 0;
};

inline LutPlan lut_plan(const aqlm_b200_weight_t& w, int64_t batch, const DeviceInfo& di, const Tunables& t) {
  LutPlan L;
  const int K = w.num_codebooks;
  if (batch != 1 || w.nbits_per_codebook != 8 || w.in_group_size != 8) return L;
  if (!(K == 1 || K == 2 || K == 4 || K == 8)) return L;
  if (t.disable_lut) return L;
  if ((reinterpret_cast<uintptr_t>(w.codes) & 7) != 0) return L;
  L.J = (K == 8) ? 16 : 32;
  const int in_groups = (int)(w.in_features / 8);
  L.n_slabs = (in_groups + L.J - 1) / L.J;
  L.smem = (size_t)K * 256 * L.J * 4 + 16;  // LUT + the "last CTA" flag word
  if (L.smem + 1024 > (size_t)di.max_smem_optin) return L;
  int per_sm = (int)((size_t)di.max_smem_optin / (L.smem + 1024));
  const int want = t.lut_ctas_per_sm;
  if (per_sm > want) per_sm = want;
  if (per_sm < 1) per_sm = 1;
  // the whole grid must be resident at once (ONE wave): a few CTAs spilling into a second wave double the time
  int rb = (di.sm_count * per_sm) / L.n_slabs;
  if (rb < 1) rb = 1;
  int rpb = (int)((w.out_features + rb - 1) / rb);
  rpb = (rpb + 31) / 32 * 32;
  L.rows_per_block = rpb;
  L.row_blocks = (int)((w.out_features + rpb - 1) / rpb);
  if ((size_t)L.row_blocks > (size_t)kGemmMaxTiles) return L;  // tickets in words [0, 8192), generation words above
  L.partials_bytes = (size_t)L.n_slabs * w.out_features * 4;
  L.ok = true;
  return L;
}

// ---- Kx8 LUT GEMV, cluster / DSMEM variant (K <= 2, at most 8 slabs of 64 groups) ------------------------------
// Batch-1 call on a 1x8 / 2x8 weight whose in_features fit 8 slabs: no workspace needed.
inline bool lut_cluster_eligible(const aqlm_b200_weight_t& w, const void* input, int64_t batch, const Tunables& t) {
  const int K = w.num_codebooks;
  const int in_groups = (int)(w.in_features / 8);
  if (batch != 1 || w.nbits_per_codebook != 8 || w.in_group_size != 8 || (K != 1 && K != 2)) return false;
  if (t.disable_lut) return false;
  if ((in_groups & 1) || in_groups > 8 * kLutCJ) return false;
  return !((reinterpret_cast<uintptr_t>(w.codes) & 3) || (reinterpret_cast<uintptr_t>(input) & 3));
}

inline int lut_cluster_slabs(const aqlm_b200_weight_t& w) {
  const int in_groups = (int)(w.in_features / 8);
  return (in_groups + kLutCJ - 1) / kLutCJ;
}

// Row blocking when `max_clusters` clusters of lut_cluster_slabs() CTAs can be resident at once: the grid must be ONE
// wave (a second wave doubles the time).  rows_per_block == 0: the cluster kernel does not apply (use the workspace one).
struct LutClusterRows {
  int rows_per_block = 0, row_blocks = 0;
};
inline LutClusterRows lut_cluster_rows(const aqlm_b200_weight_t& w, int max_clusters) {
  LutClusterRows r;
  if (max_clusters < 1) return r;
  int rpb = (int)((w.out_features + max_clusters - 1) / max_clusters);
  rpb = (rpb + 31) / 32 * 32;
  if (rpb > 2048) return r;  // per-row partials live in shared memory
  r.rows_per_block = rpb;
  r.row_blocks = (int)((w.out_features + rpb - 1) / rpb);
  return r;
}

// ---- fused dequant + wgmma GEMM, forward and transposed ------------------------------------------------------------
struct GemmPlan {
  bool ok = false;  // tensor-core (wgmma) path applicable
  int m_tiles = 0, n_tiles = 0, n_tile = 0, ksplit = 1, stages = 0, total_kblocks = 0;
  int tile_m = kGemmBlockM;  // output rows per CTA tile (the transposed kernel: always kGemmBlockM)
  size_t counters_bytes = 0, partials_bytes = 0;
};

// MMA width: the smallest wgmma N of {16, 32, 64, 128} covering the batch (larger batches: tiles of 128)
inline void gemm_n_tiles(int64_t batch, int* n_tile, int* n_tiles) {
  int n = 16;
  while (n < kGemmMaxN && n < batch) n <<= 1;
  *n_tile = n;
  *n_tiles = (int)((batch + n - 1) / n);
}

// Cost of one k-block of one CTA in SM clocks: max(gathers, tensor pipe, shared-memory traffic) + a fixed
// synchronisation cost.  Model constants, not measurements: gathers of 16-byte codebook vectors at ~0.6 per clock from
// L2 (the 1 MiB 1x16 codebook) and ~1.1 from L1 (256-entry codebooks); the tensor pipe at 2048 fp16 MACs per clock
// per SM (the data-sheet dense rate); shared memory at 128 bytes per clock.
inline double gemm_kblock_clk(int rows, int K, int nbits, int n_tile, double smem_bytes) {
  const double t_gather = rows * 8.0 * K / (nbits == 16 ? 0.6 : 1.1);
  const double t_mma = 128.0 * n_tile * 64.0 / 2048.0;
  const double t_smem = smem_bytes / 128.0;
  double t = t_gather > t_mma ? t_gather : t_mma;
  return (t > t_smem ? t : t_smem) + 60.0;
}

// Checks both GEMMs share: in_group 8, 8- or 16-bit codes, 1/2/4/8 codebooks, 16-byte aligned code rows.
// TMA needs a 16-byte multiple as the global row stride of the code matrix (1x8: in_features % 128 == 0).
inline bool gemm_scheme_ok(const aqlm_b200_weight_t& w, const Tunables& t) {
  const int K = w.num_codebooks, nbits = w.nbits_per_codebook, cb = nbits <= 8 ? 1 : 2;
  if (w.in_group_size != 8 || (nbits != 8 && nbits != 16) || !(K == 1 || K == 2 || K == 4 || K == 8)) return false;
  if ((reinterpret_cast<uintptr_t>(w.codes) & 15) != 0) return false;
  if (((size_t)(w.in_features / 8) * K * cb) % 16 != 0) return false;
  return !t.disable_wgmma;
}

// Pipeline depth: at most 3 stages (shared memory taken here is L1 taken from the codebook gathers, and outstanding
// misses need L1 lines), fewer when the layout does not fit; AQLM_B200_GEMM_STAGES forces 2..forced_max when it fits.
// 0: not even 2 stages fit.
template <typename SmemTotal>
inline int gemm_stages(SmemTotal smem_total, size_t budget, int forced, int forced_max) {
  int S = 3;
  while (S > 2 && smem_total(S) > budget) --S;
  if (smem_total(S) > budget) return 0;
  if (forced >= 2 && forced <= forced_max && smem_total(forced) <= budget) S = forced;
  return S;
}

// Split-K cost model, in SM clocks, over ksplit = 1..max_ks for one tile height `tm`:
//   per CTA: its k-blocks + a fixed cost (launch ramp, pipeline fill, epilogue: ~5 us);
//   per launch: waves x CTA time + split-K fix-up traffic (partials written and read once through L2).
// Keeps the best (tm, ksplit) so far in *best / *best_tm / *best_ks; full tiles and fewer splits win unless the gain is real.
inline void gemm_split_search(int tm, long long tiles, int K, int nbits, int n_tile, int total_kblocks, int max_ks,
                              int sm_count, double* best, int* best_tm, int* best_ks) {
  const double clk = 1.7e9;
  // smem bytes per k-block: A written once and read once, B written once and read by both consumer warpgroups
  const double t_kb = gemm_kblock_clk(tm, K, nbits, n_tile, 2.0 * 128 * 128 + 3.0 * n_tile * 128);
  for (int c = 1; c <= max_ks; ++c) {
    const double ctas = (double)tiles * c;
    const double waves = (double)((long long)((ctas + sm_count - 1) / sm_count));
    const double kb_cta = (double)((total_kblocks + c - 1) / c);
    const double fix = c > 1 ? ctas * n_tile * kGemmBlockM * 4.0 * 2.0 / 3e12 * clk : 0.0;
    const double t = waves * (kb_cta * t_kb + 5e-6 * clk) + fix;
    if (t < *best * (tm == kGemmBlockM && c == 1 ? 1.0 : 0.97)) {
      *best = t;
      *best_tm = tm;
      *best_ks = c;
    }
  }
}

// The split count the search may try: half the k-blocks, at least 1, at most 16.
inline int gemm_max_ksplit(int total_kblocks) {
  return total_kblocks / 2 < 16 ? (total_kblocks / 2 < 1 ? 1 : total_kblocks / 2) : 16;
}

// AQLM_B200_GEMM_KSPLIT (with a workspace only), clamped to [1, total_kblocks]; then the split-K workspace: a
// fixed-size counter region (the partials of one plan must never overlap the counters of another plan that reuses the
// same persistent workspace) followed by [m_tiles][n_tiles][ksplit][n_tile][128] fp32 partials.
inline void gemm_finish(GemmPlan& g, int ks, bool allow_split, const Tunables& t) {
  if (allow_split && t.gemm_ksplit > 0) ks = t.gemm_ksplit;
  if (ks > g.total_kblocks) ks = g.total_kblocks;
  if (ks < 1) ks = 1;
  g.counters_bytes = kWsCountersBytes;
  if ((size_t)g.m_tiles * g.n_tiles > (size_t)kGemmMaxTiles) ks = 1;
  g.ksplit = ks;
  g.partials_bytes = ks > 1 ? (size_t)g.m_tiles * g.n_tiles * ks * g.n_tile * kGemmBlockM * 4 : 0;
  g.ok = true;
}

// Forward: y[batch][out] = x[batch][in] W^T.  Searches the tile height (128 down to 64 in steps of 1, then to 32 in
// steps of 8) together with the split count; AQLM_B200_GEMM_TILE_M in [8, 128] forces the height.
inline GemmPlan gemm_plan(const aqlm_b200_weight_t& w, int64_t batch, const DeviceInfo& di, const Tunables& t,
                          bool allow_split) {
  GemmPlan g;
  const int K = w.num_codebooks, nbits = w.nbits_per_codebook;
  const int cb = nbits <= 8 ? 1 : 2;
  if (!gemm_scheme_ok(w, t) || 8 * K * cb > kCodeTileBytes || w.in_features % kGemmBlockK != 0) return g;
  g.total_kblocks = (int)(w.in_features / kGemmBlockK);
  gemm_n_tiles(batch, &g.n_tile, &g.n_tiles);
  g.stages = gemm_stages([&](int s) { return gemm_smem_layout(s, g.n_tile, kGemmBlockM * kCodeTileBytes).total; },
                         (size_t)di.max_smem_optin, t.gemm_stages, 4);
  if (!g.stages) return g;
  int best_tm = kGemmBlockM, best_ks = 1;
  double best = 1e30;
  const int max_ks = allow_split ? gemm_max_ksplit(g.total_kblocks) : 1;
  for (int tm = kGemmBlockM; tm >= 32; tm -= (tm > 64 ? 1 : 8)) {
    const long long tiles = ((w.out_features + tm - 1) / tm) * (long long)g.n_tiles;
    if (tiles > kGemmMaxTiles) continue;
    gemm_split_search(tm, tiles, K, nbits, g.n_tile, g.total_kblocks, max_ks, di.sm_count, &best, &best_tm, &best_ks);
  }
  g.tile_m = best_tm;
  if (t.gemm_tile_m >= 8 && t.gemm_tile_m <= kGemmBlockM) g.tile_m = t.gemm_tile_m;
  g.m_tiles = (int)((w.out_features + g.tile_m - 1) / g.tile_m);
  gemm_finish(g, best_ks, allow_split, t);  // more than kGemmMaxTiles tiles: no split
  return g;
}

// Transposed (backward w.r.t. the input): grad_in[batch][in] = grad_out[batch][out] W.  Tiles of kGemmBlockM input
// rows; more than kGemmMaxTiles tiles is not covered.
inline GemmPlan gemm_t_plan(const aqlm_b200_weight_t& w, int64_t batch, const DeviceInfo& di, const Tunables& t,
                            bool allow_split) {
  GemmPlan g;
  const int K = w.num_codebooks, nbits = w.nbits_per_codebook;
  const int cb = nbits <= 8 ? 1 : 2;
  if (!gemm_scheme_ok(w, t) || 16 * K * cb > 256) return g;
  if (w.out_features % 8 != 0) return g;  // TMA row stride of grad_out
  g.total_kblocks = (int)((w.out_features + kGemmBlockK - 1) / kGemmBlockK);
  g.m_tiles = (int)((w.in_features + kGemmBlockM - 1) / kGemmBlockM);
  gemm_n_tiles(batch, &g.n_tile, &g.n_tiles);
  const int ctile_bytes = kGemmTCtileRows * 16 * K * cb;
  // forced stages: 2..3, i.e. never more than the unforced choice
  g.stages = gemm_stages([&](int s) { return gemm_smem_layout(s, g.n_tile, ctile_bytes).total; },
                         (size_t)di.max_smem_optin, t.gemm_stages, 3);
  if (!g.stages) return g;
  if ((size_t)g.m_tiles * g.n_tiles > (size_t)kGemmMaxTiles) return g;
  int best_tm = kGemmBlockM, best_ks = 1;
  double best = 1e30;
  if (allow_split)
    gemm_split_search(kGemmBlockM, (long long)g.m_tiles * g.n_tiles, K, nbits, g.n_tile, g.total_kblocks,
                      gemm_max_ksplit(g.total_kblocks), di.sm_count, &best, &best_tm, &best_ks);
  gemm_finish(g, best_ks, allow_split, t);
  return g;
}

// Routed (mixture-of-experts) GEMM over n_experts experts of descriptor w's shape, forward or transposed, `rows` input
// rows in all.  The routing is on the device, so the plan assumes it balanced: N is the MMA width for ceil(rows / m)
// rows per expert (m = min(E, rows) experts non-empty), and the tile height and split count are searched over m_tiles x
// the slots balanced routing keeps busy.  The grid has routed_slot_count() slots, enough for any routing; the slots
// are the plan's n_tiles (workspace [m_tiles][slots][ksplit][N][128]).  More than kGemmMaxTiles tiles: no split; more
// slots than a grid dimension holds: no plan.
inline GemmPlan gemm_routed_plan(const aqlm_b200_weight_t& w, int64_t rows, int n_experts, const DeviceInfo& di,
                                 const Tunables& t, bool allow_split, bool transposed) {
  GemmPlan g;
  const int K = w.num_codebooks, nbits = w.nbits_per_codebook;
  const int cb = nbits <= 8 ? 1 : 2;
  if (rows < 1 || n_experts < 1 || !gemm_scheme_ok(w, t)) return g;
  if (transposed ? (16 * K * cb > 256 || w.out_features % 8 != 0)
                 : (8 * K * cb > kCodeTileBytes || w.in_features % kGemmBlockK != 0))
    return g;
  const int64_t m = rows < n_experts ? rows : n_experts;
  int per_expert_tiles = 0;
  gemm_n_tiles((rows + m - 1) / m, &g.n_tile, &per_expert_tiles);
  const long long slots = routed_slot_count(rows, n_experts, g.n_tile);
  if (slots > 65535) return g;
  g.n_tiles = (int)slots;
  const long long active = m * (long long)per_expert_tiles;
  const int ctile_bytes = transposed ? kGemmTCtileRows * 16 * K * cb : kGemmBlockM * kCodeTileBytes;
  g.stages = gemm_stages([&](int s) { return gemm_smem_layout(s, g.n_tile, ctile_bytes).total; },
                         (size_t)di.max_smem_optin, t.gemm_stages, transposed ? 3 : 4);
  if (!g.stages) return g;
  g.total_kblocks = (int)(transposed ? (w.out_features + kGemmBlockK - 1) / kGemmBlockK : w.in_features / kGemmBlockK);
  const int max_ks = allow_split ? gemm_max_ksplit(g.total_kblocks) : 1;
  int best_tm = kGemmBlockM, best_ks = 1;
  double best = 1e30;
  if (transposed) {
    gemm_split_search(kGemmBlockM, ((w.in_features + kGemmBlockM - 1) / kGemmBlockM) * active, K, nbits, g.n_tile,
                      g.total_kblocks, max_ks, di.sm_count, &best, &best_tm, &best_ks);
  } else {
    for (int tm = kGemmBlockM; tm >= 32; tm -= (tm > 64 ? 1 : 8)) {
      const long long tiles = ((w.out_features + tm - 1) / tm) * active;
      if (tiles > kGemmMaxTiles) continue;
      gemm_split_search(tm, tiles, K, nbits, g.n_tile, g.total_kblocks, max_ks, di.sm_count, &best, &best_tm, &best_ks);
    }
    g.tile_m = best_tm;
    if (t.gemm_tile_m >= 8 && t.gemm_tile_m <= kGemmBlockM) g.tile_m = t.gemm_tile_m;
  }
  const int64_t m_size = transposed ? w.in_features : w.out_features;
  g.m_tiles = (int)((m_size + g.tile_m - 1) / g.tile_m);
  gemm_finish(g, best_ks, allow_split, t);  // more than kGemmMaxTiles tiles (m_tiles x slots): no split
  return g;
}

// ---- fused weight-gradient GEMM (gradients of codebooks and scales) -------------------------------------------------
struct WgradPlan {
  bool ok = false;
  int out_tiles = 0, in_tiles = 0, stages = 0, total_kblocks = 0;
  size_t smem = 0, counters_bytes = 0, dots_bytes = 0;  // workspace: counters, then [in_tiles][out] fp32 row dots
};

// grad_codebooks / grad_scales from input [batch][in] and grad_output [batch][out]: one CTA per 128 x 128 tile of
// D = grad_output^T input, the batch is the contraction.  The schemes of gemm_scheme_ok, and out % 8 == 0 (TMA row
// stride of grad_output).  Stages as the forward's (at most 4 when forced); the epilogue's memory (the staged D, 64 KiB +
// padding, and for 8-bit codes the CTA's K x 256 x 8 fp32 codebook gradient) reuses the pipeline's.
inline WgradPlan gemm_wgrad_plan(const aqlm_b200_weight_t& w, int64_t batch, const DeviceInfo& di, const Tunables& t) {
  WgradPlan g;
  if (batch < 1 || !gemm_scheme_ok(w, t) || w.out_features % 8 != 0) return g;
  const int64_t out_tiles = (w.out_features + kWgradTile - 1) / kWgradTile;
  const int64_t in_tiles = (w.in_features + kWgradTile - 1) / kWgradTile;
  if (out_tiles > kGemmMaxTiles || in_tiles > 65535) return g;  // one ticket word per out tile; grid.y
  g.out_tiles = (int)out_tiles;
  g.in_tiles = (int)in_tiles;
  g.total_kblocks = (int)((batch + kWgradBlockK - 1) / kWgradBlockK);
  const int cb_bytes = wgrad_cb_smem_bytes(w.num_codebooks, w.nbits_per_codebook);
  g.stages = gemm_stages([&](int s) { return gemm_wgrad_smem_layout(s, cb_bytes).total; }, (size_t)di.max_smem_optin,
                         t.gemm_stages, 4);
  if (!g.stages) return g;
  g.smem = gemm_wgrad_smem_layout(g.stages, cb_bytes).total;
  g.counters_bytes = kWsCountersBytes;
  g.dots_bytes = (size_t)g.in_tiles * w.out_features * 4;
  g.ok = true;
  return g;
}

}  // namespace aqlm_b200
