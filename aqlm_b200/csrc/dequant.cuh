// Materialise W [out_features, in_features] from codes/codebooks(/scales).
// Replaces Code1x16Dequant / Code2x8Dequant / CodeKx8Dequant (reference cuda_kernel.cu:98-142, 235-294,
// 392-468) and the `weight *= scales` launch behind code*_dequant (cuda_kernel.cpp:184-227): one thread
// per weight group, additive sum in fp32 (exact for codebook entries of one binade), optional scale fused as an fp32
// multiply (rounded to fp32), then ONE rounding to T: W = rT(rf32(s * sum)), or rT(sum) without scales; 16-byte
// coalesced stores.
#pragma once

#include "common.cuh"

namespace aqlm_b200 {

template <typename T, int CODE_BYTES, int G>
__global__ void __launch_bounds__(256) dequant_kernel(const void* __restrict__ codes, const void* __restrict__ codebooks,
                                                      const T* __restrict__ scales, void* __restrict__ W,
                                                      int64_t out_features, int in_groups, int K, int nbits) {
  constexpr int UPG = G / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= out_features * in_groups) return;
  const int64_t row = idx / in_groups;
  const uint32_t mask = (1u << nbits) - 1u;
  const uint4* gcb = reinterpret_cast<const uint4*>(codebooks);
  float wf[UPG][8];
  for (int k = 0; k < K; ++k) {
    uint32_t code;
    if constexpr (CODE_BYTES == 2) code = reinterpret_cast<const uint16_t*>(codes)[idx * K + k];
    else code = reinterpret_cast<const uint8_t*>(codes)[idx * K + k];
    code &= mask;
    const size_t off = (((size_t)k << nbits) + code) * UPG;
#pragma unroll
    for (int h = 0; h < UPG; ++h) {
      const uint4 v = ld_gather_v4<0>(gcb + off + h);
      if (k == 0) unpack8<T>(v, wf[h]);
      else accum8<T>(v, wf[h]);
    }
  }
  const float s = scales ? DT<T>::to_float(scales[row]) : 1.f;
  uint4* out = reinterpret_cast<uint4*>(W) + idx * UPG;
#pragma unroll
  for (int h = 0; h < UPG; ++h) {
    uint4 o;
    o.x = DT<T>::pack2(wf[h][0] * s, wf[h][1] * s);
    o.y = DT<T>::pack2(wf[h][2] * s, wf[h][3] * s);
    o.z = DT<T>::pack2(wf[h][4] * s, wf[h][5] * s);
    o.w = DT<T>::pack2(wf[h][6] * s, wf[h][7] * s);
    out[h] = o;
  }
}

}  // namespace aqlm_b200
