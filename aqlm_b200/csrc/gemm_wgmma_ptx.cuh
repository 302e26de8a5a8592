// Hand-written PTX of the wgmma GEMM pipeline (gemm_wgmma.cuh): mbarrier, TMA tensor loads, the async-proxy fence and
// wgmma.mma_async with its shared-memory matrix descriptors.
#pragma once

#include <cuda.h>

#include "common.cuh"

namespace aqlm_b200 {

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

// One wgmma.mma_async m64nNk16 statement per width, over the names d, a, b, TA of wgmma_tile below; TY is the
// instruction's operand type token ("f16" or "bf16"), the only thing the two data types differ in.  N / 2 accumulator
// registers, then the A and B descriptors, the scale-d predicate and the transpose-A and transpose-B immediates.
#define AQLM_WGMMA_D8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define AQLM_WGMMA_D16(o) AQLM_WGMMA_D8(o), AQLM_WGMMA_D8(o + 8)
#define AQLM_WGMMA_D32(o) AQLM_WGMMA_D16(o), AQLM_WGMMA_D16(o + 16)
#define AQLM_WGMMA_R0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define AQLM_WGMMA_R8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define AQLM_WGMMA_R16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define AQLM_WGMMA_R32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define AQLM_WGMMA_R48 ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
// SHAPE "m64nNk16"; DREGS the accumulator placeholders; A, B, P, TAI, TBI the placeholders that follow them
#define AQLM_WGMMA(SHAPE, TY, DREGS, A, B, P, TAI, TBI, ...)                              \
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, " P ", 0;\n"                              \
               "wgmma.mma_async.sync.aligned." SHAPE ".f32." TY "." TY " "                 \
               "{" DREGS "}, " A ", " B ", p, 1, 1, " TAI ", " TBI ";\n}\n"                \
               : __VA_ARGS__                                                               \
               : "l"(a), "l"(b), "r"(1), "n"(TA), "n"(TB))
#define AQLM_WGMMA_N16(TY) AQLM_WGMMA("m64n16k16", TY, AQLM_WGMMA_R0, "%8", "%9", "%10", "%11", "%12", AQLM_WGMMA_D8(0))
#define AQLM_WGMMA_N32(TY) \
  AQLM_WGMMA("m64n32k16", TY, AQLM_WGMMA_R0 AQLM_WGMMA_R8, "%16", "%17", "%18", "%19", "%20", AQLM_WGMMA_D16(0))
#define AQLM_WGMMA_N64(TY)                                                                                             \
  AQLM_WGMMA("m64n64k16", TY, AQLM_WGMMA_R0 AQLM_WGMMA_R8 AQLM_WGMMA_R16, "%32", "%33", "%34", "%35", "%36", \
             AQLM_WGMMA_D32(0))
#define AQLM_WGMMA_N128(TY)                                                                                          \
  AQLM_WGMMA("m64n128k16", TY, AQLM_WGMMA_R0 AQLM_WGMMA_R8 AQLM_WGMMA_R16 AQLM_WGMMA_R32 AQLM_WGMMA_R48, "%64", "%65", \
             "%66", "%67", "%68", AQLM_WGMMA_D32(0), AQLM_WGMMA_D32(32))

// D[64 x N] += A[64 x 16] . B[N x 16]^T in T (fp16 or bf16), fp32 accumulate; TA = 1: A is MN-major (transposed);
// TB = 1: B is MN-major (transposed); 0: K-major
template <typename T, int N, int TA, int TB = 0>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t a, uint64_t b) {
  static_assert(N == 16 || N == 32 || N == 64 || N == 128, "wgmma tile width");
  if constexpr (DT<T>::is_bf16) {
    if constexpr (N == 16) AQLM_WGMMA_N16("bf16");
    else if constexpr (N == 32) AQLM_WGMMA_N32("bf16");
    else if constexpr (N == 64) AQLM_WGMMA_N64("bf16");
    else AQLM_WGMMA_N128("bf16");
  } else {
    if constexpr (N == 16) AQLM_WGMMA_N16("f16");
    else if constexpr (N == 32) AQLM_WGMMA_N32("f16");
    else if constexpr (N == 64) AQLM_WGMMA_N64("f16");
    else AQLM_WGMMA_N128("f16");
  }
}

}  // namespace aqlm_b200
