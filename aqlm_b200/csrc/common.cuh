// Common device/host helpers for the aqlm_b200 kernels (sm_90a only).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/aqlm_b200.h"

namespace aqlm_b200 {

// ---- error plumbing -------------------------------------------------------------------------------
inline char* tls_error_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}
inline int fail(int status, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(tls_error_buf(), 512, fmt, ap);
  va_end(ap);
  return status;
}
#define AQLM_CUDA_CHECK(expr)                                                                                  \
  do {                                                                                                         \
    cudaError_t _e = (expr);                                                                                   \
    if (_e != cudaSuccess) {                                                                                   \
      (void)cudaGetLastError(); /* clear the sticky-less error so the caller's next launch check is not poisoned */ \
      return ::aqlm_b200::fail(AQLM_B200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),    \
                               __FILE__, __LINE__);                                                            \
    }                                                                                                          \
  } while (0)

extern std::atomic<uint64_t> g_launch_count;
inline void count_launch() { g_launch_count.fetch_add(1, std::memory_order_relaxed); }

// Per-device constants, queried ONCE per device (the reference queries device 0 twice per call,
// cuda_kernel.cu:486,497).
constexpr int kMaxDevices = 64;
struct DeviceInfo {
  int index = 0;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  int max_smem_optin = 0;
  // Set (release) after the fields above are written; a reader that sees it (acquire) sees them too.
  std::atomic<bool> ok{false};
};
const DeviceInfo* device_info();  // for the current device; nullptr on failure (error set)

// ---- dtype traits ---------------------------------------------------------------------------------
template <typename T>
struct DT;
template <>
struct DT<__half> {
  static constexpr bool is_bf16 = false;
  static __device__ __forceinline__ float2 unpack2(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
  }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float to_float(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
};
template <>
struct DT<__nv_bfloat16> {
  static constexpr bool is_bf16 = true;
  static __device__ __forceinline__ float2 unpack2(uint32_t v) {
    // bf16 -> f32 is a 16-bit shift: exact and cheaper than the cvt path
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
  }
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
};

// ---- memory access flavours -----------------------------------------------------------------------
// Streaming read of packed codes: read exactly once, keep out of L1.
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// Codebook gathers. MODE 0: read-only path with L1 allocation (LDG.CONSTANT); 1: L2 only (ld.cg, the
// reference's choice, cuda_kernel.cu:46-57).
template <int MODE>
__device__ __forceinline__ uint4 ld_gather_v4(const void* p) {
  static_assert(MODE == 0 || MODE == 1, "gather mode");
  uint4 r;
  if constexpr (MODE == 0) {
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  } else {
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  }
  return r;
}

// 32-byte gather (in_group_size = 16: one codebook entry = one 32-byte L2 sector).  sm_90 has no 256-bit load, so
// the entry is read as two 128-bit requests to the same sector, issued back to back.
__device__ __forceinline__ void ld_gather_v8(const void* p, uint4& lo, uint4& hi) {
  lo = ld_gather_v4<0>(p);
  hi = ld_gather_v4<0>(reinterpret_cast<const uint4*>(p) + 1);
}

// Programmatic dependent launch (PDL).  Both are no-ops when the kernel was launched without the
// programmatic-stream-serialization attribute.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// XOR swizzle of 16-byte units so that lanes reading units 8 apart hit different bank groups.
__device__ __forceinline__ int swz16(int u) { return u ^ ((u >> 3) & 7); }

template <typename T>
__device__ __forceinline__ float dot8(const uint4& w, const uint4& x, float acc) {
  float2 a, b;
  a = DT<T>::unpack2(w.x); b = DT<T>::unpack2(x.x); acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
  a = DT<T>::unpack2(w.y); b = DT<T>::unpack2(x.y); acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
  a = DT<T>::unpack2(w.z); b = DT<T>::unpack2(x.z); acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
  a = DT<T>::unpack2(w.w); b = DT<T>::unpack2(x.w); acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc);
  return acc;
}

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& w, float* f) {
  float2 a;
  a = DT<T>::unpack2(w.x); f[0] = a.x; f[1] = a.y;
  a = DT<T>::unpack2(w.y); f[2] = a.x; f[3] = a.y;
  a = DT<T>::unpack2(w.z); f[4] = a.x; f[5] = a.y;
  a = DT<T>::unpack2(w.w); f[6] = a.x; f[7] = a.y;
}
template <typename T>
__device__ __forceinline__ void accum8(const uint4& w, float* f) {
  float2 a;
  a = DT<T>::unpack2(w.x); f[0] += a.x; f[1] += a.y;
  a = DT<T>::unpack2(w.y); f[2] += a.x; f[3] += a.y;
  a = DT<T>::unpack2(w.z); f[4] += a.x; f[5] += a.y;
  a = DT<T>::unpack2(w.w); f[6] += a.x; f[7] += a.y;
}
template <typename T>
__device__ __forceinline__ float dot8f(const float* w, const uint4& x, float acc) {
  float2 b;
  b = DT<T>::unpack2(x.x); acc = fmaf(w[0], b.x, acc); acc = fmaf(w[1], b.y, acc);
  b = DT<T>::unpack2(x.y); acc = fmaf(w[2], b.x, acc); acc = fmaf(w[3], b.y, acc);
  b = DT<T>::unpack2(x.z); acc = fmaf(w[4], b.x, acc); acc = fmaf(w[5], b.y, acc);
  b = DT<T>::unpack2(x.w); acc = fmaf(w[6], b.x, acc); acc = fmaf(w[7], b.y, acc);
  return acc;
}

// LoRA adapter of a linear, as the fused kernels take it (aqlm_b200_lora_t on the device side).  The kernel adds
// scaling * sum_j lin[t][j] * w(m, j), summed in fp32, to output element (t, m) before its one rounding to T:
//   forward:    lin = U = dropout(x) . A^T [batch][rank],  w(o, j) = B[o][j]   (B = up,   [out][rank])
//   transposed: lin = V = grad_out . B     [batch][rank],  w(i, j) = A[j][i]   (A = down, [rank][in])
// All of it is read after griddep_wait(): lin comes from the previous kernel, A and B from the optimizer step.
struct LoraArgs {
  const void* lin;
  const void* w;
  int rank;     // 8..64, a multiple of 8
  int f32;      // 1: adapter operands are fp32, 0: T
  float scaling;
};

// Elements idx .. idx + 3 (idx % 4 == 0, 16-byte aligned rows) of an adapter operand, as fp32
template <typename T>
__device__ __forceinline__ float4 lora_load4(const void* base, size_t idx, int f32) {
  if (f32) return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + idx);
  const uint2 v = *reinterpret_cast<const uint2*>(reinterpret_cast<const T*>(base) + idx);
  const float2 a = DT<T>::unpack2(v.x), b = DT<T>::unpack2(v.y);
  return make_float4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ float dot4(const float4& a, const float4& b, float acc) {
  acc = fmaf(a.x, b.x, acc);
  acc = fmaf(a.y, b.y, acc);
  acc = fmaf(a.z, b.z, acc);
  return fmaf(a.w, b.w, acc);
}

// Extract element `idx` (compile-time after unrolling) of CODE_BYTES-wide unsigned codes from a 16-byte chunk.
template <int CODE_BYTES>
__device__ __forceinline__ uint32_t chunk_code(const uint4& c, int idx) {
  const uint32_t w[4] = {c.x, c.y, c.z, c.w};
  if constexpr (CODE_BYTES == 2) {
    return (w[idx >> 1] >> ((idx & 1) * 16)) & 0xffffu;
  } else {
    return (w[idx >> 2] >> ((idx & 3) * 8)) & 0xffu;
  }
}

}  // namespace aqlm_b200
