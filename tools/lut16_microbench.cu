// Go / no-go microbenchmark for a dot-product-LUT formulation of the 1x16 matvec (VERDICT r1 item 9b).
//
// Idea under test:  y[o] = sum_j LUT_j[code[o,j]],  LUT_j[c] = codebook[c] . x_j  (65536 fp16 entries = 128 KiB per
// in-group j, held in shared memory; one SM owns one j at a time and streams that group's codes for all rows).  It
// replaces a random 16-byte L2 gather per code (chip cap ~250 G/s) by a random 2-byte shared-memory lookup, but every
// (SM, j) pair must ingest the whole 1 MiB codebook to build its LUT.  Two rates decide whether it can win:
//   (1) random 2-byte shared-memory lookups per clock per SM (128 KiB table)     -- needs >= 6 / clk / SM
//   (2) codebook ingest per SM in bytes/clk when a cluster shares the stream by TMA multicast -- needs >= 100 B/clk/SM
// One JSON line per variant.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/bin/lut16_microbench tools/lut16_microbench.cu
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e = (x);                                                                   \
    if (e != cudaSuccess) {                                                                \
      printf("{\"error\": \"%s at %s:%d\"}\n", cudaGetErrorString(e), __FILE__, __LINE__); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

// ---- (1) random 2-byte lookups in a 128 KiB shared-memory table; U code chunks (8 codes each) in flight per lane ----
template <int U>
__global__ void __launch_bounds__(1024, 1) k_lds16(const uint4* __restrict__ codes, size_t nchunks, float* out) {
  extern __shared__ uint16_t tab[];
  for (int i = threadIdx.x; i < 65536; i += blockDim.x) tab[i] = (uint16_t)(i * 2654435761u >> 16);
  __syncthreads();
  float acc = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += stride * U) {
    uint4 cw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) cw[u] = (c + u * stride < nchunks) ? ld_stream(codes + c + u * stride) : make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t w[4] = {cw[u].x, cw[u].y, cw[u].z, cw[u].w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t code = (w[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
        acc += __half2float(__ushort_as_half(tab[code]));
      }
    }
  }
  if (acc == 123.456f) out[0] = acc;
}

// ---- (2) codebook ingest through TMA bulk copies multicast over a cluster of CS CTAs ------------------------------
// Every CTA ends up with every chunk of the stream in its own shared memory; CTA r issues the r-th 1/CS of each chunk
// with a multicast mask covering the whole cluster.  Two 32 KiB buffers; a split cluster barrier guards buffer reuse.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
template <int CS>
__global__ void __launch_bounds__(128, 1) k_ingest(const uint8_t* __restrict__ src, size_t total_bytes, int reps, float* out) {
  constexpr int CH = 32768;
  extern __shared__ __align__(128) uint8_t buf[];  // [2][CH]
  __shared__ __align__(8) uint64_t bars[2];
  uint32_t rank = 0;
  if (CS > 1) asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const uint32_t b0 = smem_u32(&bars[0]);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b0));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b0 + 8));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CS > 1) asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  const size_t nchunks = total_bytes / CH;
  const size_t iters = nchunks * reps;
  const uint16_t mask = (uint16_t)((1u << CS) - 1u);
  auto issue = [&](size_t it) {
    const int b = (int)(it & 1);
    const uint8_t* g = src + (it % nchunks) * CH + rank * (CH / CS);
    const uint32_t dst = smem_u32(buf) + b * CH + rank * (CH / CS);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b0 + 8 * b), "r"(CH) : "memory");
    if (CS > 1)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                   ::"r"(dst), "l"(g), "r"(CH / CS), "r"(b0 + 8 * b), "h"(mask) : "memory");
    else
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(dst), "l"(g), "r"(CH), "r"(b0 + 8 * b) : "memory");
  };
  float acc = 0.f;
  if (threadIdx.x == 0) {
    issue(0);
    if (iters > 1) issue(1);
  }
  for (size_t it = 0; it < iters; ++it) {
    const int b = (int)(it & 1);
    mbar_wait(b0 + 8 * b, (uint32_t)((it >> 1) & 1));
    acc += (float)buf[b * CH + threadIdx.x * 16];  // touch the data
    // all CTAs of the cluster must be done with buffer b before anyone multicasts into it again
    if (CS > 1) asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    else __syncthreads();
    if (threadIdx.x == 0 && it + 2 < iters) issue(it + 2);
  }
  if (acc == 123.456f) out[0] = acc;
}

int main() {
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  int khz = 0;
  CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0));
  const double clk = khz * 1e3;
  float* out;
  CK(cudaMalloc(&out, 64));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  {  // (1)
    const size_t ncodes = (size_t)28672 * 512 * 4;  // 58.7 M codes per launch
    const size_t nchunks = ncodes / 8;
    uint4* codes;
    CK(cudaMalloc(&codes, nchunks * sizeof(uint4)));
    std::vector<uint32_t> h(nchunks * 4);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    for (auto& w : h) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; w = (uint32_t)(s >> 16); }
    CK(cudaMemcpy(codes, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
    auto run = [&](auto kernel, const char* name) {
      CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 131072));
      for (int i = 0; i < 2; ++i) kernel<<<sms, 1024, 131072>>>(codes, nchunks, out);
      CK(cudaDeviceSynchronize());
      CK(cudaEventRecord(a));
      for (int i = 0; i < 5; ++i) kernel<<<sms, 1024, 131072>>>(codes, nchunks, out);
      CK(cudaEventRecord(b));
      CK(cudaEventSynchronize(b));
      float ms;
      CK(cudaEventElapsedTime(&ms, a, b));
      ms /= 5;
      const double per_s = ncodes / (ms * 1e-3);
      printf("{\"test\": \"smem_random_2byte_lookups\", \"variant\": \"%s\", \"ms\": %.4f, \"Glookups_s\": %.1f, "
             "\"lookups_per_clk_per_sm\": %.2f, \"equiv_code_GBps\": %.1f, \"need\": \">= 6 /clk/SM\"}\n",
             name, ms, per_s / 1e9, per_s / sms / clk, per_s * 2 / 1e9);
      fflush(stdout);
    };
    run(k_lds16<1>, "1024 threads, 8 lookups in flight per lane");
    run(k_lds16<2>, "1024 threads, 16 lookups in flight per lane");
    run(k_lds16<4>, "1024 threads, 32 lookups in flight per lane");
    CK(cudaFree(codes));
  }
  {  // (2)
    const size_t total = 1 << 20;  // the 1 MiB codebook, streamed `reps` times
    uint8_t* src;
    CK(cudaMalloc(&src, total));
    CK(cudaMemset(src, 1, total));
    const int reps = 64;
    auto run = [&](auto kernel, int cs, const char* name) {
      CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
      if (cs > 8) CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      cfg.gridDim = dim3((sms / cs) * cs); cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = 65536;
      cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, (const uint8_t*)src, total, 2, out);
      if (e != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
        cudaGetLastError();
        printf("{\"test\": \"codebook_ingest\", \"variant\": \"%s\", \"skipped\": \"%s\"}\n", name, cudaGetErrorString(e));
        return;
      }
      CK(cudaEventRecord(a));
      CK(cudaLaunchKernelEx(&cfg, kernel, (const uint8_t*)src, total, reps, out));
      CK(cudaEventRecord(b));
      CK(cudaEventSynchronize(b));
      float ms;
      CK(cudaEventElapsedTime(&ms, a, b));
      const double bytes_per_sm = (double)total * reps;
      printf("{\"test\": \"codebook_ingest\", \"variant\": \"%s\", \"ctas\": %d, \"ms\": %.4f, \"ingest_B_per_clk_per_sm\": %.1f, "
             "\"chip_TBps_landed\": %.2f, \"need\": \">= 100 B/clk/SM\"}\n",
             name, (sms / cs) * cs, ms, bytes_per_sm / (ms * 1e-3) / clk, bytes_per_sm * ((sms / cs) * cs) / (ms * 1e-3) / 1e12);
      fflush(stdout);
    };
    run(k_ingest<1>, 1, "unicast bulk copies (no cluster)");
    run(k_ingest<2>, 2, "multicast, cluster of 2");
    run(k_ingest<4>, 4, "multicast, cluster of 4");
    run(k_ingest<8>, 8, "multicast, cluster of 8");
    run(k_ingest<16>, 16, "multicast, cluster of 16 (non-portable)");
  }
  return 0;
}
