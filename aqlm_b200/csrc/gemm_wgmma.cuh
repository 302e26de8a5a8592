// Fused additive-dequant + tensor-core GEMM for batch > 6:  Y[bs, out] = X[bs, in] . W^T, W never touches HBM.
//
// Replaces code{1x16,2x8,1x8}_matmat_dequant (reference cuda_kernel.cpp:249-301, 450-484, 615-649), which
// materialise W [out,in] in HBM with a Dequant kernel (cuda_kernel.cu:98-142) and then call cuBLAS.
//
// H100 design (wgmma / TMA / mbarrier, hand-written PTX):
//   D[128 x N] (fp32, registers)  +=  A[128 x 64] (smem, K-major, SWIZZLE_128B)  x  B[N x 64]^T (smem, K-major, SWIZZLE_128B)
//   A = a 128-row tile of W, produced ON CHIP: producer warps read packed codes from a TMA-staged code tile,
//       gather the codebook vectors (L2/L1) and write them straight into the swizzled wgmma layout;
//   B = the activation tile X[n0:n0+N, k0:k0+64], TMA-loaded (OOB rows zero-filled, so any batch works);
//   two consumer warpgroups (rows 0-63 and 64-127 of the tile) issue wgmma.mma_async (64 x N x 16, fp16 or bf16
//   operands, fp32 accumulate in registers), release the smem stage through an mbarrier once their wgmma group has
//   completed, and apply scale + bias in the epilogue (or, with partial_f32, store the unscaled fp32 sums that an
//   in_features-sharded linear all-reduces).
// Warp roles: warps 0-7 consumers, warp 8 TMA (X tiles and code tiles), warps 9-16 dequant producers.
// Grid = (M tiles, K splits, N tiles).  The kernel is bound by the per-SM codebook-gather rate, so the K dimension is
// split to put every SM to work; split partials go through an fp32 workspace and the LAST-arriving CTA of each tile
// reduces them in a fixed order (deterministic).
#pragma once

#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace aqlm_b200 {

constexpr int kGemmConsumerWarps = 8;   // two warpgroups
constexpr int kGemmTmaWarp = kGemmConsumerWarps;
constexpr int kGemmProducerWarps = 8;
constexpr int kGemmProducerThreads = 32 * kGemmProducerWarps;
constexpr int kGemmProducer0 = 32 * (kGemmConsumerWarps + 1);  // first producer thread
constexpr int kGemmThreads = kGemmProducer0 + kGemmProducerThreads;
constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;          // 64 halves = 128 bytes = one swizzle row
constexpr int kGemmMaxN = 128;           // accumulator of one consumer thread: N / 2 fp32 registers
constexpr int kCodeTileBytes = 128;      // bytes of codes per row per code tile (TMA box inner extent)
constexpr int kCodeTileStages = 2;

struct GemmParams {
  const void* codebooks;
  const void* scales;
  const void* bias;
  void* y;              // [batch, out_features]
  float* ws_partials;   // [m_tiles][n_tiles][ksplit][N][128] fp32 (ksplit > 1)
  unsigned int* ws_counters;  // [m_tiles * n_tiles], zero on entry
  int out_features;
  int batch;
  int nbits;
  int total_kblocks;    // in_features / 64
  int ksplit;
  int stages;
  int tile_m;           // output rows per CTA tile (<= 128): ragged tile heights balance the grid
  int gather_mode;      // 0: ld.global.nc (L1 allocate), 1: ld.global.cg
  int partial_f32;      // 1: y is fp32 and gets the UNSCALED sums (no scale, no bias; scales / bias may be null)
};

// ---- PTX wrappers -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
// one lane of a converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, SWIZZLE_128B: start>>4 | LBO>>4 << 16 | SBO>>4 << 32 | swizzle mode 1 << 62.
// K-major: SBO = 1024 (8-row atoms), LBO unused.  MN-major: LBO = distance of 64-element atoms along MN, SBO =
// distance of 8-row atoms along K.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) |
         ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// waits until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 16] . B[N x 16]^T; TA = 1: A is MN-major (transposed), B is K-major
template <int TA>
__device__ __forceinline__ void wgmma_m64n16_f16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, %11, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n16_bf16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, %11, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n32_f16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, %19, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n32_bf16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1, %19, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n64_f16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n64_bf16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n128_f16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}

template <int TA>
__device__ __forceinline__ void wgmma_m64n128_bf16(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1), "n"(TA));
}
template <typename T, int N, int TA>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t a, uint64_t b) {
  static_assert(N == 16 || N == 32 || N == 64 || N == 128, "wgmma tile width");
  if constexpr (DT<T>::is_bf16) {
    if constexpr (N == 16) wgmma_m64n16_bf16<TA>(d, a, b);
    else if constexpr (N == 32) wgmma_m64n32_bf16<TA>(d, a, b);
    else if constexpr (N == 64) wgmma_m64n64_bf16<TA>(d, a, b);
    else wgmma_m64n128_bf16<TA>(d, a, b);
  } else {
    if constexpr (N == 16) wgmma_m64n16_f16<TA>(d, a, b);
    else if constexpr (N == 32) wgmma_m64n32_f16<TA>(d, a, b);
    else if constexpr (N == 64) wgmma_m64n64_f16<TA>(d, a, b);
    else wgmma_m64n128_f16<TA>(d, a, b);
  }
}

// shared-memory carve-up (all offsets from a 1024-byte aligned base)
struct GemmSmem {
  uint32_t a, b, codes, full, empty, cfull, cempty, flag;
  size_t total;
};
__host__ __device__ inline GemmSmem gemm_smem_layout(int stages, int n_tile) {
  GemmSmem L;
  size_t off = 0;
  L.a = (uint32_t)off; off += (size_t)stages * kGemmBlockM * 128;
  L.b = (uint32_t)off; off += (size_t)stages * n_tile * 128;
  off = (off + 1023) & ~(size_t)1023;
  L.codes = (uint32_t)off; off += (size_t)kCodeTileStages * kGemmBlockM * kCodeTileBytes;
  L.full = (uint32_t)off; off += 8 * 8;
  L.empty = (uint32_t)off; off += 8 * 8;
  L.cfull = (uint32_t)off; off += 8 * kCodeTileStages;
  L.cempty = (uint32_t)off; off += 8 * kCodeTileStages;
  L.flag = (uint32_t)off; off += 4;
  L.total = off + 1024;  // slack for manual 1024-byte alignment of the dynamic smem base
  return L;
}

// Split-K fix-up shared by both GEMM kernels: the LAST-arriving split of a tile adds all partials in split order
// (deterministic) with the whole CTA; partials are [split][column][128 rows].  Writes y[n * ld + row0 + r] =
// v * scale[row] + bias[row] (scales == nullptr: no scale / bias); an fp32 output (OutT = float) gets the sum v itself.
template <typename T, typename OutT = T>
__device__ __forceinline__ void gemm_splitk_fixup(uint32_t* flag, unsigned int* counter, const float* parts, int ksplit, int N,
                                                  int ncols, OutT* y, long long ld, int n0, int row0, int rows,
                                                  const T* scales, const T* bias) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int old = atomicAdd(counter, 1u);
    const bool last = (old == (unsigned int)ksplit - 1);
    *flag = last ? 1u : 0u;
    if (last) *counter = 0u;  // leave the counter clean for the next call
  }
  __syncthreads();
  constexpr int kPhases = kGemmThreads / kGemmBlockM;  // column phases of 128 threads each
  if (*flag && threadIdx.x < kPhases * kGemmBlockM) {
    __threadfence();
    const int rrow = threadIdx.x & (kGemmBlockM - 1);
    const int cphase = threadIdx.x >> 7;
    if (rrow < rows) {
      const int row = row0 + rrow;
      const float sc = scales ? DT<T>::to_float(scales[row]) : 1.f;
      const float bi = bias ? DT<T>::to_float(bias[row]) : 0.f;
      for (int c = cphase; c < ncols; c += kPhases * 4) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (int sp = 0; sp < ksplit; ++sp) {
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int cc = c + u * kPhases;
            if (cc < ncols) v[u] += __ldcg(parts + ((size_t)sp * N + cc) * kGemmBlockM + rrow);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int cc = c + u * kPhases;
          if (cc >= ncols) continue;
          if constexpr (std::is_same<OutT, float>::value) y[(size_t)(n0 + cc) * ld + row] = v[u];
          else y[(size_t)(n0 + cc) * ld + row] = DT<T>::from_float(fmaf(v[u], sc, bi));
        }
      }
    }
  }
}

// K = codebooks per group, CODE_BYTES = 1|2 ; in_group_size == 8.  N = MMA width (columns of the batch tile).
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_codes, const GemmParams p) {
  constexpr int GB = 8 * K * CODE_BYTES;             // code bytes per row per k-block
  constexpr int KB_PER_CTILE = kCodeTileBytes / GB;  // k-blocks covered by one code tile
  static_assert(KB_PER_CTILE >= 1, "scheme too wide for the code tile");
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* gbase = smem_dyn + (base - smem_u32(smem_dyn));
  const GemmSmem L = gemm_smem_layout(p.stages, N);
  const int S = p.stages;
  const int TM = p.tile_m;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, split = blockIdx.y, n_blk = blockIdx.z;
  const int m0 = m_tile * TM, n0 = n_blk * N;
  // PDL: the next kernel of the stream may be dispatched as soon as SM resources free up (no launch gap).  Everything this
  // kernel does before griddep_wait() touches WEIGHTS only (code tiles, codebook gathers); the X tiles are read and y /
  // the workspace written after it.
  griddep_launch_dependents();
  // k-block range of this split (balanced, contiguous)
  const int kb0 = (int)(((long long)p.total_kblocks * split) / p.ksplit);
  const int kb1 = (int)(((long long)p.total_kblocks * (split + 1)) / p.ksplit);
  const int nkb = kb1 - kb0;
  // code tiles: aligned to KB_PER_CTILE boundaries in absolute k-block index
  const int ct0 = kb0 / KB_PER_CTILE;
  const int ct1 = (kb1 + KB_PER_CTILE - 1) / KB_PER_CTILE;

  auto full_bar = [&](int s) { return base + L.full + 8 * s; };
  auto empty_bar = [&](int s) { return base + L.empty + 8 * s; };
  auto cfull_bar = [&](int s) { return base + L.cfull + 8 * s; };
  auto cempty_bar = [&](int s) { return base + L.cempty + 8 * s; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), kGemmProducerWarps + 1);  // producer warps + the TMA thread's expect_tx arrival
      mbar_init(empty_bar(s), kGemmConsumerWarps);     // every consumer warp, after its wgmma group completed
    }
    for (int s = 0; s < kCodeTileStages; ++s) {
      mbar_init(cfull_bar(s), 1);
      mbar_init(cempty_bar(s), kGemmProducerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const size_t tile_id = (size_t)m_tile * gridDim.z + n_blk;
  T* y = reinterpret_cast<T*>(p.y);
  if (warp < kGemmConsumerWarps) {
    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    // one wgmma group stays in flight: k-block i's MMAs run while the warpgroup waits for k-block i+1, and the stage of
    // k-block i is released once k-block i+1's group is committed and i's has completed (S >= 2 keeps this deadlock-free)
    int s = 0, prev = -1;
    uint32_t ph = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(full_bar(s), ph);
      const uint64_t ad = wgmma_desc(base + L.a + s * kGemmBlockM * 128 + wg * 64 * 128, 16, 1024);
      const uint64_t bd = wgmma_desc(base + L.b + s * N * 128, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kGemmBlockK / 16; ++k)  // 16 K-elements = 32 bytes = +2 in the descriptor's address field
        wgmma_tile<T, N, 0>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k));
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(prev));  // this warp's reads of the previous stage are complete
      }
      prev = s;
      if (++s == S) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
    }
    griddep_wait();  // before any global write (y, split-K partials): the previous kernel has completed
    // accumulator fragment: register 4i + 2j + c holds (row 16 (warp % 4) + lane / 4 + 8 j, column 8 i + 2 (lane % 4) + c)
    float* my_part = p.ws_partials ? p.ws_partials + ((tile_id * p.ksplit + split) * (size_t)N) * kGemmBlockM : nullptr;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * j;
      const int row = m0 + row_in_tile;
      const bool row_ok = row_in_tile < TM && row < p.out_features;
      float sc = 1.f, bi = 0.f;
      if (row_ok && p.ksplit == 1 && !p.partial_f32) {
        sc = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        if (p.bias) bi = DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]);
      }
#pragma unroll
      for (int i = 0; i < N / 8; ++i) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int col = 8 * i + 2 * (lane & 3) + c;
          const float v = acc[4 * i + 2 * j + c];
          if (p.ksplit == 1) {
            if (row_ok && n0 + col < p.batch) {
              const size_t o = (size_t)(n0 + col) * p.out_features + row;
              if (p.partial_f32) reinterpret_cast<float*>(p.y)[o] = v;
              else y[o] = DT<T>::from_float(fmaf(v, sc, bi));
            }
          } else {
            my_part[(size_t)col * kGemmBlockM + row_in_tile] = v;
          }
        }
      }
    }
  } else if (warp == kGemmTmaWarp) {
    if (nkb > 0) {
      // ===== TMA producer (whole warp, one elected lane issues): code tiles (one per KB_PER_CTILE k-blocks) and one X
      //       tile per k-block =====
      int ct_loaded = ct0;
      auto load_ctile = [&](int ct) {
        const int cs = (ct - ct0) % kCodeTileStages;
        const int it = (ct - ct0) / kCodeTileStages;
        if (it > 0) mbar_wait(cempty_bar(cs), (it - 1) & 1);  // every producer warp released the previous tenant
        if (elect_one()) {
          mbar_expect_tx(cfull_bar(cs), (uint32_t)TM * kCodeTileBytes);  // the TMA box is tile_m rows tall
          tma_load_2d(base + L.codes + cs * kGemmBlockM * kCodeTileBytes, &tmap_codes, ct * kCodeTileBytes, m0, cfull_bar(cs));
        }
        __syncwarp();
      };
      load_ctile(ct_loaded++);
      griddep_wait();  // X is produced by the previous kernel
      int s = 0, it = 0;  // X stage and its use count (no runtime division in this loop)
      for (int i = 0; i < nkb; ++i) {
        if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
        if (elect_one()) {
          mbar_expect_tx(full_bar(s), (uint32_t)N * 128);
          tma_load_2d(base + L.b + s * N * 128, &tmap_x, (kb0 + i) * kGemmBlockK, n0, full_bar(s));
        }
        __syncwarp();
        // prefetch the NEXT code tile while the producers work on the current one
        const int ct_cur = (kb0 + i) / KB_PER_CTILE;
        if (ct_loaded < ct1 && ct_loaded <= ct_cur + 1) load_ctile(ct_loaded++);
        if (++s == S) { s = 0; ++it; }
      }
    }
  } else if (nkb > 0) {
    // ===== dequant producers: 256 threads, thread -> (row, half of the 8 groups of a k-block) =====
    // Software-pipelined for K <= 2: the gathers of the next D k-blocks are in flight while k-block i is written to smem
    // (the kernel is bound by gather latency unless several gathers per thread are outstanding).  K >= 4 gathers and
    // sums group by group (the 256-entry codebooks of those schemes are L1-resident).
    const int pt = threadIdx.x - kGemmProducer0;
    const int row = pt >> 1, half = pt & 1;
    const bool active = row < TM;  // rows past the (ragged) tile height: no gathers, nothing to write
    const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);
    constexpr int CB4 = 4 * K * CODE_BYTES;  // code bytes of this thread's 4 groups
    constexpr int CW = (CB4 + 3) / 4;        // 32-bit words holding them
    constexpr bool INREG = K <= 2;           // hold the raw gathered vectors in registers until the write
    constexpr int KR = INREG ? K : 1;
    constexpr int D = (K == 1) ? 2 : 1;      // k-blocks of gathers held in registers ahead of the writes
    auto gather = [&](const uint4* gp) -> uint4 {
      return p.gather_mode == 1 ? ld_gather_v4<1>(gp) : ld_gather_v4<0>(gp);
    };

    // codes of k-block index i (relative) -> the 4 groups' gathers (K <= 2) or their dequantized sums (K >= 4)
    auto issue = [&](int i, uint4 (&wv)[4][KR]) {
      const int kb = kb0 + i;
      const int ct = kb / KB_PER_CTILE, st_in = kb % KB_PER_CTILE;
      const int cs = (ct - ct0) % kCodeTileStages, cit = (ct - ct0) / kCodeTileStages;
      mbar_wait(cfull_bar(cs), cit & 1);
      uint32_t cw[CW];
      // logical byte offset inside the 128-byte code row -> physical (SWIZZLE_128B: 16-byte chunk ^= row & 7)
      const int lbyte = st_in * GB + half * CB4;
      const uint8_t* crow = gbase + L.codes + cs * kGemmBlockM * kCodeTileBytes + row * 128;
      if (!active) {
#pragma unroll
        for (int q = 0; q < CW; ++q) cw[q] = 0u;
      } else if constexpr (CB4 >= 16) {
#pragma unroll
        for (int q = 0; q < CB4 / 16; ++q) {
          const int chunk = ((lbyte >> 4) + q) ^ (row & 7);
          const uint4 v = *reinterpret_cast<const uint4*>(crow + (chunk << 4));
          cw[4 * q + 0] = v.x; cw[4 * q + 1] = v.y; cw[4 * q + 2] = v.z; cw[4 * q + 3] = v.w;
        }
      } else {
        const uint8_t* src = crow + ((((lbyte >> 4) ^ (row & 7))) << 4) + (lbyte & 15);
        if constexpr (CB4 == 8) { const uint2 v = *reinterpret_cast<const uint2*>(src); cw[0] = v.x; cw[1] = v.y; }
        else cw[0] = *reinterpret_cast<const uint32_t*>(src);
      }
      auto code_at = [&](int idx) -> uint32_t {
        if constexpr (CODE_BYTES == 2) return (cw[idx >> 1] >> ((idx & 1) * 16)) & 0xffffu;
        else return (cw[idx >> 2] >> ((idx & 3) * 8)) & 0xffu;
      };
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if constexpr (INREG) {
#pragma unroll
          for (int k = 0; k < K; ++k)
            wv[e][k] = active ? gather(gcb + (((size_t)k << p.nbits) + code_at(e * K + k))) : make_uint4(0u, 0u, 0u, 0u);
        } else {
          float f[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) f[q] = 0.f;
          if (active) {
#pragma unroll
            for (int k = 0; k < K; ++k) accum8<T>(gather(gcb + (((size_t)k << p.nbits) + code_at(e * K + k))), f);
          }
          wv[e][0].x = DT<T>::pack2(f[0], f[1]); wv[e][0].y = DT<T>::pack2(f[2], f[3]);
          wv[e][0].z = DT<T>::pack2(f[4], f[5]); wv[e][0].w = DT<T>::pack2(f[6], f[7]);
        }
      }
      // Release the code tile after its last k-block.  This MUST come after the gathers above were issued: their
      // addresses depend on the code registers, so the shared-memory loads of the codes have completed by now.
      if (st_in == KB_PER_CTILE - 1 || i == nkb - 1) {
        __syncwarp();
        if (lane == 0) mbar_arrive(cempty_bar(cs));
      }
    };
    int st_next = 0, it_next = 0;  // commit() runs for k-blocks 0, 1, 2, ... in order
    // additive dequant + write the 4 groups of k-block i into the swizzled A stage, then signal the consumers
    auto commit = [&](uint4 (&wv)[4][KR]) {
      const int s = st_next, it = it_next;
      if (++st_next == S) { st_next = 0; ++it_next; }
      if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
      uint8_t* arow = gbase + L.a + s * kGemmBlockM * 128 + row * 128;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        uint4 v = wv[e][0];
        if constexpr (K == 2) {
          float f[8];
          unpack8<T>(wv[e][0], f);
          accum8<T>(wv[e][1], f);
          v.x = DT<T>::pack2(f[0], f[1]); v.y = DT<T>::pack2(f[2], f[3]);
          v.z = DT<T>::pack2(f[4], f[5]); v.w = DT<T>::pack2(f[6], f[7]);
        }
        const int j = half * 4 + e;  // 16-byte chunk (= group) index inside the 128-byte K row
        if (active) *reinterpret_cast<uint4*>(arow + ((j ^ (row & 7)) << 4)) = v;
      }
      fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(s));
    };
    uint4 w[D][4][KR];
#pragma unroll
    for (int d = 0; d < D; ++d)
      if (d < nkb) issue(d, w[d]);
    for (int i = 0; i < nkb; i += D) {
#pragma unroll
      for (int d = 0; d < D; ++d) {
        if (i + d < nkb) {
          commit(w[d]);
          if (i + d + D < nkb) issue(i + d + D, w[d]);
        }
      }
    }
  }

  if (p.ksplit > 1) {
    griddep_wait();
    uint32_t* flag = reinterpret_cast<uint32_t*>(gbase + L.flag);
    const float* parts = p.ws_partials + (tile_id * p.ksplit) * (size_t)N * kGemmBlockM;
    const int ncols = min(N, p.batch - n0), rows = min(TM, p.out_features - m0);
    if (p.partial_f32)
      gemm_splitk_fixup<T, float>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, reinterpret_cast<float*>(p.y),
                                  p.out_features, n0, m0, rows, nullptr, nullptr);
    else
      gemm_splitk_fixup<T>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, y, p.out_features, n0, m0, rows,
                           reinterpret_cast<const T*>(p.scales), reinterpret_cast<const T*>(p.bias));
  }
}

}  // namespace aqlm_b200
