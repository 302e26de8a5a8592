// Fused additive-dequant + TRANSPOSED tensor-core GEMM (the backward w.r.t. the input):
//     grad_in[bs, in] = (grad_out[bs, out] * scales[out]) . W[out, in]          W never touches HBM.
//
// Replaces code{1x16,2x8,1x8}_matmat_dequant_transposed (reference cuda_kernel.cpp:303-354, 486-519, 651-684), which
// materialise W [out,in] in HBM with a Dequant kernel and call cuBLAS on (grad_out * scales); the reference's 2x8/1x8
// variants forget the scaled input (cuda_kernel.cpp:497,518,662,683) -- not reproduced.
//
// The pipeline (warp roles, barrier protocol, epilogue, split-K fix-up) is gemm_pipeline of gemm_wgmma.cuh; this file is
// the transposed direction, with the contraction running over OUT rows:
//   D[128 in-features x N batch] (fp32, registers)  +=  A[128 x 64] . B[N x 64]^T        per k-block of 64 out rows
//   A = W^T tile, produced on chip.  A gathered codebook vector is 8 CONSECUTIVE in-features of ONE out row, i.e. 16
//       contiguous bytes along M: the A stage is therefore kept MN-MAJOR (canonical SWIZZLE_128B MN-major layout,
//       64 x 8 element atoms, wgmma transpose-A), so a gather still lands with ONE 16-byte store;
//       the per-row scale is applied to the vector before it is written (fp32 multiply, one rounding);
//   B = grad_out tile [N x 64 out columns], K-major, TMA-loaded with 128B swizzle (OOB rows/columns zero-filled);
//   code tiles: TMA boxes of 256 out rows x (16 groups * K codes) bytes, un-swizzled.
// Grid = (in/128 tiles, K splits over the out rows, N tiles).  Tiles are always 128 in-features tall and the output is
// always T (no ragged tile_m, no partial_f32).
#pragma once

#include "gemm_wgmma.cuh"

namespace aqlm_b200 {

constexpr int kGemmTCtileRows = 256;  // out rows per code tile (= 4 k-blocks)

// See GemmForward for what a direction describes.
template <int K_, int CODE_BYTES_>
struct GemmTransposed {
  static constexpr int K = K_, CODE_BYTES = CODE_BYTES_;
  static constexpr int CB4 = 4 * K * CODE_BYTES;   // code bytes of one producer thread's 4 adjacent groups
  static constexpr int GBT = 16 * K * CODE_BYTES;  // code bytes per out row per tile (16 groups = 128 in-features)

  // A stage: MN-major SWIZZLE_128B, atoms laid out [k_atom (8)][m_atom (2)][1024 B]: LBO (next MN atom) 1024 B, SBO
  // (next K atom) 2048 B; warpgroup wg owns in-features [64 wg, 64 wg + 64) of the tile = MN atom wg of every K atom
  static constexpr int TA = 1;
  static constexpr uint32_t kALbo = 1024, kASbo = 2048;
  static constexpr uint32_t kAStepK = 256;  // 16 out rows = 2 K atoms: A advances 4096 bytes (+256)
  static constexpr uint32_t kAWarpgroup = 1024;

  // The producer multiplies every vector by the scale of its out row; the epilogue and the fix-up only cast.
  static constexpr bool kScaleInProducer = true;
  static constexpr bool kTransposed = true;
  static __device__ __forceinline__ int tile_m(const GemmParams&) { return kGemmBlockM; }
  // out rows of one expert of a routed call (the contraction's length)
  static __device__ __forceinline__ int out_rows(const GemmParams& p) { return p.k_size; }

  // code tile: 256 out rows x GBT bytes, un-swizzled; covers 4 k-blocks
  static constexpr int kCtileBytes = kGemmTCtileRows * GBT;
  static constexpr int kKbPerCtile = kGemmTCtileRows / kGemmBlockK;
  static __device__ __forceinline__ uint32_t ctile_tx_bytes(int) { return kCtileBytes; }
  static __device__ __forceinline__ int2 ctile_coord(int m_tile, int, int ct) {
    return make_int2(m_tile * GBT, ct * kGemmTCtileRows);
  }

  // producer thread pt -> (out row kk = pt / 4 of the k-block, groups 4 gq .. 4 gq + 3 of the tile's 16, gq = pt % 4)
  static __device__ __forceinline__ bool active(int, int) { return true; }
  // the out row of the thread changes with every k-block: a grouped call resolves its segment's codebooks per k-block
  static constexpr bool kRowPerKblock = true;
  static __device__ __forceinline__ int out_row(int pt, int, int kb) { return kb * kGemmBlockK + (pt >> 2); }
  // e_rows: where a routed call's expert starts in the stacked scales (0 otherwise); o stays relative to the expert
  template <typename T>
  static __device__ __forceinline__ float row_scale(const GemmParams& p, int pt, int kb, size_t e_rows) {
    const int o = out_row(pt, 0, kb);
    return o < p.k_size ? DT<T>::to_float((reinterpret_cast<const T*>(p.scales) + e_rows)[o]) : 0.f;  // rows past the end contribute nothing
  }
  static __device__ __forceinline__ int code_offset(int pt, int st_in, int q) {
    return (st_in * kGemmBlockK + (pt >> 2)) * GBT + (pt & 3) * CB4 + 16 * q;
  }
  // atom (kk >> 3, m_atom) at [(kk >> 3) * 2 + m_atom] * 1024; inside an atom row kk & 7 is 128 bytes of 64 consecutive
  // in-features, its 16-byte chunks XOR-swizzled with kk & 7.  Group j of the tile = 16-byte chunk j along M.
  static __device__ __forceinline__ int a_chunk_offset(int pt, int e) {
    const int kk = pt >> 2, j = (pt & 3) * 4 + e;
    return (kk >> 3) * 2048 + (kk & 7) * 128 + (j >> 3) * 1024 + (((j & 7) ^ (kk & 7)) << 4);
  }
};

template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_t_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_codes, const GemmParams p) {
  gemm_pipeline<T, N, GemmTransposed<K, CODE_BYTES>>(tmap_g, tmap_codes, p);
}

// The backward of a plain linear with a LoRA adapter (LoraArgs, transposed form): grad_in = (grad_out s) W + scaling V A,
// V = grad_out . B computed by the caller, one rounding.
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_t_lora_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_codes,
                           const GemmParams p, const LoraArgs lora) {
  gemm_pipeline<T, N, GemmTransposed<K, CODE_BYTES>, false, false, true>(tmap_g, tmap_codes, p, lora);
}

// The backward of a grouped call: grad_output holds the members' output gradients side by side.
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_t_grouped_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_codes,
                              const GemmParams p) {
  gemm_pipeline<T, N, GemmTransposed<K, CODE_BYTES>, true>(tmap_g, tmap_codes, p);
}

// The backward of a routed call: grad_output rows sorted by expert, as the forward's input was.
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_t_routed_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_codes,
                             const GemmParams p) {
  gemm_pipeline<T, N, GemmTransposed<K, CODE_BYTES>, true, true>(tmap_g, tmap_codes, p);
}

}  // namespace aqlm_b200
