// Fused weight-gradient GEMM of a quantized linear: the gradients of its codebooks and scales, W and dW never in HBM.
//
// The forward computes y[b, r] = s_r * sum_j x[b, j] Wu[r, j] + bias_r, where Wu[r, 8g + i] = sum_k C[k, code(r,g,k), i]
// is the unscaled weight exactly as the forward's producer feeds it to the tensor core (fp32 sum, rounded once to T).
// With G = grad_output [batch, out], X = input [batch, in] and D = G^T X [out, in] (fp32):
//   grad_codebooks[k][c][i] += sum over (r, g) with code(r, g, k) = c of  s_r * D[r, 8g + i]
//   grad_scales[r]           = sum_j D[r, j] * Wu[r, j]
// The reference trains these parameters by dequantizing W into HBM and back-propagating through F.linear, which also
// writes the dense dW [out, in]; here D lives in one CTA's registers and shared memory only.
//
// H100 design (wgmma / TMA / mbarrier, the PTX wrappers of gemm_wgmma_ptx.cuh):
//   Grid = (out / 128 tiles, in / 128 tiles); the contraction runs over the batch in k-blocks of 64 rows.
//   D[128 out x 128 in] (fp32, registers)  +=  A[128 x 64] . B[128 x 64]^T      per k-block
//   A = a G tile, 128 out rows x 64 batch rows, MN-major (out rows contiguous, as G is stored): two TMA boxes of
//       64 out x 64 batch rows, SWIZZLE_128B, i.e. the canonical MN-major layout (64-element atoms 8 KiB apart);
//   B = an X tile, 128 in-columns x 64 batch rows, MN-major the same way: wgmma's transpose-B;
//   out-of-bounds batch rows and columns are zero-filled by TMA, so any batch and ragged tiles work.
// Warp roles: warps 0-7 two consumer warpgroups (64 out rows x 128 columns each), warp 8 TMA.  No dequant producer:
// codes and codebooks are read once per tile, in the epilogue:
//   1. D is staged in the pipeline's freed shared memory (rows padded to 132 floats);
//   2. thread t takes out row t / 2 and 8 of its 16 groups; per (row, group): read the K codes, add s_r * D[r, 8g..+8]
//      into the codebook gradient, gather the K codebook vectors, rebuild Wu rounded as the forward rounds it, and
//      accumulate the row's dot with D in a fixed order.  The codebook gradient of 16-bit codes goes straight to
//      grad_codebooks, two red.global.add.v4.f32 per codebook; with 8-bit codes every reduction of every CTA would land
//      on the same 2 * K * 256 16-byte addresses, so the CTA first adds into a shared-memory copy of the K x 256 x 8
//      gradient (shared-memory atomics) and then adds that copy to grad_codebooks once, two vector reductions per
//      entry it touched;
//   3. the two halves of a row are added in a fixed order and written to workspace slot [in_tile][row];
//   4. the last-arriving CTA of each out tile adds the slots in in_tile order and writes grad_scales (the ticket pattern
//      of gemm_splitk_fixup; counters are left at zero).
// grad_scales is deterministic.  grad_codebooks is not: the reductions land in atomic arrival order, so on real data
// its fp32 sums can differ in the last bits from run to run (on an integer lattice every partial sum is exact and the
// result is order-independent).  red.global.add.v4.f32 (REDG.E.ADD.F32x4.FTZ.RN) flushes fp32 denormals to zero.
#pragma once

#include "gemm_wgmma_ptx.cuh"

namespace aqlm_b200 {

constexpr int kWgradConsumerWarps = 8;                    // two warpgroups
constexpr int kWgradThreads = 32 * (kWgradConsumerWarps + 1);  // + the TMA warp
constexpr int kWgradTile = 128;                           // out rows and in columns of a CTA tile
constexpr int kWgradBlockK = 64;                          // batch rows per k-block (= one TMA box height)
constexpr int kWgradBoxBytes = 64 * 128;                  // one TMA box: 64 batch rows x 64 elements
constexpr int kWgradStageBytes = 4 * kWgradBoxBytes;      // A (2 boxes) + B (2 boxes)
constexpr int kWgradDStride = kWgradTile + 4;             // floats per staged D row (padding against bank conflicts)
constexpr int kWgradDBytes = kWgradTile * kWgradDStride * 4;

// bytes of the per-CTA codebook-gradient copy: K x 256 x 8 fp32 for 8-bit codes, none for 16-bit codes
__host__ __device__ constexpr int wgrad_cb_smem_bytes(int K, int nbits) { return nbits <= 8 ? K * 256 * 8 * 4 : 0; }

struct WgradParams {
  const void* codes;       // [out][in / 8][K] codes of CODE_BYTES
  const void* codebooks;   // [K][2^nbits][8] in T
  const void* scales;      // [out] in T; read only with grad_codebooks
  float* grad_codebooks;   // [K][2^nbits][8] fp32, added into; null: not wanted
  float* grad_scales;      // [out] fp32, written; null: not wanted
  float* ws_dots;          // [in_tiles][out] fp32: the row dots of every in tile (grad_scales only)
  unsigned int* ws_counters;  // [out_tiles], zero on entry and on exit (grad_scales only)
  int out_features, in_features, nbits, total_kblocks, stages;
};

// shared-memory carve-up (offsets from a 1024-byte aligned base): the pipeline's stages, reused by the staged D and,
// after it, the codebook-gradient copy of cb_bytes (wgrad_cb_smem_bytes)
struct WgradSmem {
  uint32_t cb, full, empty, flag;
  size_t total;
};
__host__ __device__ inline WgradSmem gemm_wgrad_smem_layout(int stages, int cb_bytes) {
  WgradSmem L;
  const size_t pipe = (size_t)stages * kWgradStageBytes, epi = (size_t)kWgradDBytes + cb_bytes;
  L.cb = (uint32_t)kWgradDBytes;
  size_t off = pipe > epi ? pipe : epi;
  L.full = (uint32_t)off; off += 8 * 8;
  L.empty = (uint32_t)off; off += 8 * 8;
  L.flag = (uint32_t)off; off += 4;
  L.total = off + 1024;  // slack for manual 1024-byte alignment of the dynamic smem base
  return L;
}

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// K codes of one (row, group) position, K * CODE_BYTES contiguous bytes aligned to their size
template <int K, int CODE_BYTES>
struct WgradCodes {
  static constexpr int BYTES = K * CODE_BYTES, WORDS = (BYTES + 3) / 4;
  uint32_t w[WORDS];
  __device__ __forceinline__ void load(const uint8_t* p) {
    if constexpr (BYTES == 16) { const uint4 v = *reinterpret_cast<const uint4*>(p); w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; }
    else if constexpr (BYTES == 8) { const uint2 v = *reinterpret_cast<const uint2*>(p); w[0] = v.x; w[1] = v.y; }
    else if constexpr (BYTES == 4) w[0] = *reinterpret_cast<const uint32_t*>(p);
    else if constexpr (BYTES == 2) w[0] = *reinterpret_cast<const uint16_t*>(p);
    else w[0] = *p;
  }
  __device__ __forceinline__ uint32_t at(int k) const {
    if constexpr (CODE_BYTES == 2) return (w[k >> 1] >> ((k & 1) * 16)) & 0xffffu;
    else return (w[k >> 2] >> ((k & 3) * 8)) & 0xffu;
  }
};

template <typename T, int K, int CODE_BYTES>
__global__ void __launch_bounds__(kWgradThreads, 1)
gemm_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_x, const WgradParams p) {
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* gbase = smem_dyn + (base - smem_u32(smem_dyn));
  constexpr bool CB_SMEM = CODE_BYTES == 1;  // 8-bit codes: pre-reduce the codebook gradient in shared memory
  constexpr int CB_FLOATS = wgrad_cb_smem_bytes(K, 8) / 4;
  const WgradSmem L = gemm_wgrad_smem_layout(p.stages, CB_SMEM ? wgrad_cb_smem_bytes(K, 8) : 0);
  const int S = p.stages, nkb = p.total_kblocks;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, n_tile = blockIdx.y;
  const int m0 = m_tile * kWgradTile, n0 = n_tile * kWgradTile;
  auto full_bar = [&](int s) { return base + L.full + 8 * s; };
  auto empty_bar = [&](int s) { return base + L.empty + 8 * s; };

  griddep_launch_dependents();
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);                     // the TMA thread's expect_tx arrival
      mbar_init(empty_bar(s), kWgradConsumerWarps);  // every consumer warp, after its wgmma group completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  griddep_wait();  // G and X are the previous kernels' outputs; grad_codebooks may have just been zeroed

  float acc[kWgradTile / 2];
#pragma unroll
  for (int i = 0; i < kWgradTile / 2; ++i) acc[i] = 0.f;
  if (warp < kWgradConsumerWarps) {
    // ===== consumers: warpgroup wg owns out rows [64 wg, 64 wg + 64) of the tile = A's MN atom wg =====
    const int wg = warp >> 2;
    int s = 0, prev = -1;
    uint32_t ph = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(full_bar(s), ph);
      const uint32_t st = base + s * kWgradStageBytes;
      // MN-major SWIZZLE_128B: LBO = next 64-element MN atom (the second TMA box), SBO = next 8 batch rows
      const uint64_t ad = wgmma_desc(st + wg * kWgradBoxBytes, kWgradBoxBytes, 1024);
      const uint64_t bd = wgmma_desc(st + 2 * kWgradBoxBytes, kWgradBoxBytes, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kWgradBlockK / 16; ++k)  // 16 batch rows = 2048 bytes = +128 in the descriptors' address field
        wgmma_tile<T, kWgradTile, 1, 1>(acc, ad + (uint64_t)(128 * k), bd + (uint64_t)(128 * k));
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = s;
      if (++s == S) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
  } else if (nkb > 0) {
    // ===== TMA warp: per k-block two G boxes (out rows m0, m0 + 64) and two X boxes (in columns n0, n0 + 64) =====
    int s = 0, it = 0;
    for (int i = 0; i < nkb; ++i) {
      if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
      if (elect_one()) {
        const uint32_t st = base + s * kWgradStageBytes;
        const int b0 = i * kWgradBlockK;
        mbar_expect_tx(full_bar(s), kWgradStageBytes);
        tma_load_2d(st, &tmap_g, m0, b0, full_bar(s));
        tma_load_2d(st + kWgradBoxBytes, &tmap_g, m0 + 64, b0, full_bar(s));
        tma_load_2d(st + 2 * kWgradBoxBytes, &tmap_x, n0, b0, full_bar(s));
        tma_load_2d(st + 3 * kWgradBoxBytes, &tmap_x, n0 + 64, b0, full_bar(s));
      }
      __syncwarp();
      if (++s == S) { s = 0; ++it; }
    }
  }
  // every stage has been filled and read: the pipeline's memory takes D (and the codebook-gradient copy, zeroed)
  __syncthreads();
  float* Ds = reinterpret_cast<float*>(gbase);
  // codebook-gradient copy, [k][i][code]: the 32 lanes of a warp add to their own codes' element i, so the banks they
  // hit follow the codes, not i
  float* cbs = reinterpret_cast<float*>(gbase + L.cb);
  const bool want_cb = p.grad_codebooks != nullptr;
  if constexpr (CB_SMEM) {
    if (want_cb)
      for (int e = threadIdx.x; e < CB_FLOATS / 4; e += kWgradThreads) reinterpret_cast<float4*>(cbs)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (warp < kWgradConsumerWarps) {
    // accumulator fragment: register 4i + 2j + c holds (row 16 (warp % 4) + lane / 4 + 8 j, column 8 i + 2 (lane % 4) + c)
    const int wg = warp >> 2;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * j;
#pragma unroll
      for (int i = 0; i < kWgradTile / 8; ++i)
        *reinterpret_cast<float2*>(Ds + row * kWgradDStride + 8 * i + 2 * (lane & 3)) =
            make_float2(acc[4 * i + 2 * j], acc[4 * i + 2 * j + 1]);
    }
  }
  __syncthreads();

  const bool want_scales = p.grad_scales != nullptr;
  if (warp < kWgradConsumerWarps) {
    // ===== epilogue: thread t -> tile row t / 2, groups (t % 2) * 8 .. + 8 of the tile's 16 =====
    const int rr = threadIdx.x >> 1, half = threadIdx.x & 1;
    const int row = m0 + rr;
    const int in_groups = p.in_features / 8;
    const int groups = min(kWgradTile, p.in_features - n0) / 8;  // groups of this (ragged) tile
    const uint4* cb = reinterpret_cast<const uint4*>(p.codebooks);
    float dot = 0.f;
    if (row < p.out_features) {
      const float sc = p.grad_codebooks ? DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]) : 0.f;
      const uint8_t* crow = reinterpret_cast<const uint8_t*>(p.codes) + ((size_t)row * in_groups + n0 / 8) * (K * CODE_BYTES);
#pragma unroll 2
      for (int gi = 0; gi < 8; ++gi) {
        const int lg = half * 8 + gi;
        if (lg >= groups) break;
        WgradCodes<K, CODE_BYTES> c;
        c.load(crow + lg * (K * CODE_BYTES));
        const float4 d0 = *reinterpret_cast<const float4*>(Ds + rr * kWgradDStride + 8 * lg);
        const float4 d1 = *reinterpret_cast<const float4*>(Ds + rr * kWgradDStride + 8 * lg + 4);
        if (want_cb) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            if constexpr (CB_SMEM) {
              float* sp = cbs + k * (8 * 256) + c.at(k);
              const float v[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
              for (int i = 0; i < 8; ++i) atomicAdd(sp + i * 256, sc * v[i]);
            } else {
              float* gp = p.grad_codebooks + ((((size_t)k << p.nbits) + c.at(k)) << 3);
              red_add_v4(gp, sc * d0.x, sc * d0.y, sc * d0.z, sc * d0.w);
              red_add_v4(gp + 4, sc * d1.x, sc * d1.y, sc * d1.z, sc * d1.w);
            }
          }
        }
        if (want_scales) {
          float f[8];
          unpack8<T>(ld_gather_v4<CODE_BYTES == 2 ? 1 : 0>(cb + c.at(0)), f);
#pragma unroll
          for (int k = 1; k < K; ++k) accum8<T>(ld_gather_v4<CODE_BYTES == 2 ? 1 : 0>(cb + (((size_t)k << p.nbits) + c.at(k))), f);
          // Wu as the forward's producer writes it: the fp32 sum rounded once to T (exact for K = 1)
          const uint4 wu = make_uint4(DT<T>::pack2(f[0], f[1]), DT<T>::pack2(f[2], f[3]), DT<T>::pack2(f[4], f[5]),
                                      DT<T>::pack2(f[6], f[7]));
          unpack8<T>(wu, f);
          const float d[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
          for (int q = 0; q < 8; ++q) dot = fmaf(d[q], f[q], dot);
        }
      }
    }
    if (want_scales) {
      // the row's two halves, added in a fixed order
      const float other = __shfl_xor_sync(0xffffffffu, dot, 1);
      if (half == 0 && row < p.out_features) p.ws_dots[(size_t)n_tile * p.out_features + row] = dot + other;
    }
  }
  if constexpr (CB_SMEM) {
    if (want_cb) {
      // the CTA's codebook gradient into grad_codebooks: entries (k, code, half) it never touched stay out of L2
      __syncthreads();
      for (int e = threadIdx.x; e < CB_FLOATS / 4; e += kWgradThreads) {
        const int k = e >> 9, code = (e >> 1) & 255, i0 = (e & 1) * 4;
        const float* sp = cbs + k * (8 * 256) + code;
        const float a = sp[i0 * 256], b = sp[(i0 + 1) * 256], c = sp[(i0 + 2) * 256], d = sp[(i0 + 3) * 256];
        if (a != 0.f || b != 0.f || c != 0.f || d != 0.f) red_add_v4(p.grad_codebooks + (size_t)e * 4, a, b, c, d);
      }
    }
  }
  if (!want_scales) return;

  // ===== the last-arriving in tile of this out tile adds the row dots in in_tile order =====
  uint32_t* flag = reinterpret_cast<uint32_t*>(gbase + L.flag);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int old = atomicAdd(p.ws_counters + m_tile, 1u);
    const bool last = old == gridDim.y - 1;
    *flag = last ? 1u : 0u;
    if (last) p.ws_counters[m_tile] = 0u;  // leave the counter clean for the next call
  }
  __syncthreads();
  if (*flag && threadIdx.x < kWgradTile && m0 + (int)threadIdx.x < p.out_features) {
    __threadfence();
    const int row = m0 + threadIdx.x;
    float v = 0.f;
    for (unsigned int t = 0; t < gridDim.y; ++t) v += __ldcg(p.ws_dots + (size_t)t * p.out_features + row);
    p.grad_scales[row] = v;
  }
}

}  // namespace aqlm_b200
