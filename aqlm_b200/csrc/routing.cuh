// Slot resolution of the routed (mixture-of-experts) GEMMs: pure arithmetic, shared by the kernels and the host tests.
//
// A routed launch covers E experts that share one weight shape.  Its input rows are sorted by expert: expert e owns rows
// [off[e], off[e+1]) of the input (and of the output).  The offsets come from the device (the router ran there), so
// the host sizes the grid from what it knows -- rows, E and the MMA width N -- and every CTA resolves its slot (the
// grid's third index) to an expert and a run of at most N rows of it.
//
// The offsets are input, never trusted: each is clamped into [0, rows] and raised to its predecessor, so the effective
// offsets are non-decreasing.  A decreasing pair is an empty expert, no two experts share a row, and rows outside
// [off[0], off[E]) (after clamping) belong to no expert: they are neither read for output nor written.
#pragma once

#include <cstdint>

namespace aqlm_b200 {

constexpr int kRoutedMaxExperts = 64;  // experts of one routed call

struct RoutedSlot {
  int expert;  // -1: the slot is past the last tile (the CTA has nothing to do)
  int row0;    // first input / output row of the slot's tile
  int row1;    // end of the expert's rows: rows [row0, min(row0 + N, row1)) are the tile's valid rows
};

// Slots a launch needs for `rows` rows among `n_experts` experts in tiles of n_tile rows.  Expert e with c_e rows takes
// ceil(c_e / N) tiles; at most m = min(E, rows) experts are non-empty, so sum ceil(c_e / N) <= (rows + m (N - 1)) / N.
__host__ __device__ inline long long routed_slot_count(long long rows, int n_experts, int n_tile) {
  if (rows <= 0 || n_experts <= 0) return 0;
  const long long m = rows < n_experts ? rows : n_experts;
  return (rows + m * (n_tile - 1) + n_tile - 1) / n_tile;
}

// Expert e's tiles are slots [sum_{i<e} t_i, sum_{i<=e} t_i), t_i = ceil(c_i / N), in expert order.
__host__ __device__ inline RoutedSlot routed_slot(const int32_t* off, int n_experts, int rows, int n_tile, int slot) {
  auto clamp = [rows](int v) { return v < 0 ? 0 : (v > rows ? rows : v); };
  int lo = clamp(off[0]);
  int s = slot;
  for (int e = 0; e < n_experts; ++e) {
    int hi = clamp(off[e + 1]);
    if (hi < lo) hi = lo;
    const int tiles = (hi - lo + n_tile - 1) / n_tile;
    if (s < tiles) return RoutedSlot{e, lo + s * n_tile, hi};
    s -= tiles;
    lo = hi;
  }
  return RoutedSlot{-1, 0, 0};
}

// Expert e's effective rows [first, end) under the same clamping as routed_slot: the running maximum of the clamped
// offsets, so end >= first and the ranges of the experts are disjoint and in expert order.
struct RoutedRows {
  int first, end;
};
__host__ __device__ inline RoutedRows routed_expert_rows(const int32_t* off, int rows, int e) {
  auto clamp = [rows](int v) { return v < 0 ? 0 : (v > rows ? rows : v); };
  int lo = clamp(off[0]);
  for (int i = 1; i <= e; ++i) {
    const int v = clamp(off[i]);
    lo = v > lo ? v : lo;
  }
  const int hi = clamp(off[e + 1]);
  return RoutedRows{lo, hi > lo ? hi : lo};
}

}  // namespace aqlm_b200
