// Microbenchmark: how fast can an H100 do the random 16-byte codebook gathers of the 1x16 AQLM scheme?
//
// Every variant streams the same packed uint16 codes (coalesced 16-byte loads, 8 codes per lane per step,
// exactly like the GEMV kernel) and gathers one 16-byte vector per code from a 65536-entry (1 MiB) table
// through a different path.  Output: one JSON line per variant with G gathers/s and the equivalent
// code-bytes GB/s (2 B per gather), to be compared with the HBM roofline of the code stream.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/bin/gather_microbench tools/gather_microbench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#define CK(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e = (x);                                                                        \
    if (e != cudaSuccess) {                                                                     \
      printf("{\"error\": \"%s at %s:%d\"}\n", cudaGetErrorString(e), __FILE__, __LINE__);      \
      exit(1);                                                                                  \
    }                                                                                           \
  } while (0)

__device__ __forceinline__ uint4 ld_stream(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
template <int MODE>
__device__ __forceinline__ uint4 ld_g(const uint4* p) {
  uint4 r;
  if (MODE == 0) asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  if (MODE == 1) asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  if (MODE == 2) asm volatile("ld.global.ca.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  if (MODE == 3) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  if (MODE == 4) asm volatile("ld.global.nc.L1::evict_last.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t code_of(const uint4& c, int e) {
  const uint32_t w[4] = {c.x, c.y, c.z, c.w};
  return (w[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
}
#define ACC(v) { acc.x ^= (v).x; acc.y += (v).y; acc.z ^= (v).z; acc.w += (v).w; }

// ---- 0. code stream only (HBM/L2 stream reference) -------------------------------------------------
__global__ void k_stream(const uint4* __restrict__ codes, size_t nchunks, uint4* out) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)gridDim.x * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    ACC(cw);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 1. global gathers, MODE = load flavour, U = chunks in flight per lane -------------------------
template <int MODE, int U>
__global__ void k_ldg(const uint4* __restrict__ codes, size_t nchunks, const uint4* __restrict__ table, uint4* out) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += stride * U) {
    uint4 cw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) cw[u] = (c + u * stride < nchunks) ? ld_stream(codes + c + u * stride) : make_uint4(0, 0, 0, 0);
    uint4 v[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int e = 0; e < 8; ++e) v[u][e] = ld_g<MODE>(table + code_of(cw[u], e));
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int e = 0; e < 8; ++e) ACC(v[u][e]);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 2. texture gathers ----------------------------------------------------------------------------
__global__ void k_tex(const uint4* __restrict__ codes, size_t nchunks, cudaTextureObject_t tex, uint4* out) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)gridDim.x * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    uint4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = tex1Dfetch<uint4>(tex, (int)code_of(cw, e));
#pragma unroll
    for (int e = 0; e < 8; ++e) ACC(v[e]);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 3. shared-memory gathers: NE-entry slice of the table in smem, codes masked into it ------------
template <int LOG_NE>
__global__ void k_lds(const uint4* __restrict__ codes, size_t nchunks, const uint4* __restrict__ table, uint4* out) {
  extern __shared__ uint4 stab[];
  for (int i = threadIdx.x; i < (1 << LOG_NE); i += blockDim.x) stab[i] = table[i];
  __syncthreads();
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)gridDim.x * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    uint4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = stab[code_of(cw, e) & ((1 << LOG_NE) - 1)];
#pragma unroll
    for (int e = 0; e < 8; ++e) ACC(v[e]);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 4. distributed shared memory: cluster of CS CTAs, each holds 65536/CS entries ------------------
template <int CS>
__global__ void k_dsmem(const uint4* __restrict__ codes, size_t nchunks, const uint4* __restrict__ table, uint4* out) {
  extern __shared__ uint4 stab[];
  constexpr int PER = 65536 / CS;
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  for (int i = threadIdx.x; i < PER; i += blockDim.x) stab[i] = table[rank * PER + i];
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;\n" ::: "memory");
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(stab);
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)gridDim.x * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    uint4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const uint32_t code = code_of(cw, e);
      const uint32_t local = base + (code % PER) * 16;
      uint32_t remote;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(code / PER));
      asm volatile("ld.shared::cluster.v4.u32 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v[e].x), "=r"(v[e].y), "=r"(v[e].z), "=r"(v[e].w) : "r"(remote));
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) ACC(v[e]);
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;\n" ::: "memory");
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 5. hybrid: entries < NE from local smem, the rest from L2 --------------------------------------
template <int NE, int MODE>
__global__ void k_hybrid(const uint4* __restrict__ codes, size_t nchunks, const uint4* __restrict__ table, uint4* out) {
  extern __shared__ uint4 stab[];
  for (int i = threadIdx.x; i < NE; i += blockDim.x) stab[i] = table[i];
  __syncthreads();
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)gridDim.x * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    uint4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const uint32_t code = code_of(cw, e);
      if (code < NE) v[e] = stab[code];
      else v[e] = ld_g<MODE>(table + code);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) ACC(v[e]);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

// ---- 6. range-split: each CTA owns table slice [lo, lo+NE) in smem, scans ALL codes of its share and
//         gathers only matching ones (others read a zero slot).  `nsplit` CTAs cover one code range, so
//         every code chunk is visited by nsplit CTAs (reads beyond the first come from L2). ------------
template <int NE>
__global__ void k_split(const uint4* __restrict__ codes, size_t nchunks, const uint4* __restrict__ table, int nsplit, uint4* out) {
  extern __shared__ uint4 stab[];
  const int slice = blockIdx.x % nsplit;
  const int lo = slice * NE;
  for (int i = threadIdx.x; i < NE; i += blockDim.x) stab[i] = (lo + i < 65536) ? table[lo + i] : make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0) stab[NE] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const int group = blockIdx.x / nsplit, ngroups = gridDim.x / nsplit;
  uint4 acc = make_uint4(0, 0, 0, 0);
  for (size_t c = (size_t)group * blockDim.x + threadIdx.x; c < nchunks; c += (size_t)ngroups * blockDim.x) {
    uint4 cw = ld_stream(codes + c);
    uint4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      uint32_t idx = code_of(cw, e) - lo;  // wraps to huge when below lo
      idx = min(idx, (uint32_t)NE);
      v[e] = stab[idx];
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) ACC(v[e]);
  }
  if (acc.x == 0x12345 && acc.y == 0x777) out[0] = acc;
}

template <typename F>
static float time_ms(F launch, int iters) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) launch(i);
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(a));
  for (int i = 0; i < iters; ++i) launch(i);
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float ms;
  CK(cudaEventElapsedTime(&ms, a, b));
  return ms / iters;
}

int main(int argc, char** argv) {
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  // NBUF distinct code buffers of 14336x4096 1x16 (14.7 MB each) rotated so the stream comes from HBM
  const size_t ncodes = (size_t)14336 * 512;
  const size_t nchunks = ncodes / 8;
  const int NBUF = 12;  // 176 MB > L2
  uint4* codes;
  CK(cudaMalloc(&codes, NBUF * nchunks * sizeof(uint4)));
  {
    std::vector<uint32_t> h(NBUF * nchunks * 4);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    for (auto& w : h) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; w = (uint32_t)(s >> 16); }
    CK(cudaMemcpy(codes, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
  }
  uint4* table;
  CK(cudaMalloc(&table, 65536 * sizeof(uint4)));
  CK(cudaMemset(table, 1, 65536 * sizeof(uint4)));
  uint4* out;
  CK(cudaMalloc(&out, 64));
  cudaResourceDesc rd = {};
  rd.resType = cudaResourceTypeLinear;
  rd.res.linear.devPtr = table;
  rd.res.linear.desc = cudaCreateChannelDesc<uint4>();
  rd.res.linear.sizeInBytes = 65536 * sizeof(uint4);
  cudaTextureDesc td = {};
  td.readMode = cudaReadModeElementType;
  cudaTextureObject_t tex;
  CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));

  const int iters = 24;
  printf("{\"device\": \"%s\", \"sms\": %d, \"codes_per_launch\": %zu, \"rotating_buffers\": %d}\n", prop.name, sms, ncodes, NBUF);
  auto report = [&](const char* name, int ctas_per_sm, int threads, float ms) {
    const double g = ncodes / (ms * 1e-3) / 1e9;
    printf("{\"variant\": \"%s\", \"ctas_per_sm\": %d, \"threads\": %d, \"ms\": %.4f, \"Ggather_s\": %.1f, \"code_GBps\": %.1f, "
           "\"gather_per_clk_per_sm_at_1.9GHz\": %.3f}\n", name, ctas_per_sm, threads, ms, g, 2 * g, g / sms / 1.9);
    fflush(stdout);
  };
#define BUF(i) (codes + (size_t)((i) % NBUF) * nchunks)

  if (argc > 1 && std::string(argv[1]) == "ncu") {
    // One launch of each representative variant, for `ncu --set full` (names the unit behind the gather cap):
    // best LDG variant, the 2-chunk variant, pure shared-memory gathers and the smem/global hybrid.
    CK(cudaFuncSetAttribute(k_lds<13>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16));
    CK(cudaFuncSetAttribute(k_hybrid<12288, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 16));
    for (int i = 0; i < 2; ++i) {
      k_ldg<0, 1><<<sms * 4, 256>>>(BUF(i), nchunks, table, out);
      k_ldg<1, 1><<<sms * 4, 256>>>(BUF(i), nchunks, table, out);
      k_ldg<0, 2><<<sms * 4, 256>>>(BUF(i), nchunks, table, out);
      k_lds<13><<<sms, 1024, 8192 * 16>>>(BUF(i), nchunks, table, out);
      k_hybrid<12288, 0><<<sms, 1024, 12288 * 16>>>(BUF(i), nchunks, table, out);
    }
    CK(cudaDeviceSynchronize());
    return 0;
  }
  report("stream_only", 8, 256, time_ms([&](int i) { k_stream<<<sms * 8, 256>>>(BUF(i), nchunks, out); }, iters));

  const int cfgs[][2] = {{2, 256}, {4, 256}, {8, 256}, {2, 1024}, {1, 1024}};
  for (auto& cf : cfgs) {
    const int cps = cf[0], th = cf[1];
    report("ldg_nc_u1", cps, th, time_ms([&](int i) { k_ldg<0, 1><<<sms * cps, th>>>(BUF(i), nchunks, table, out); }, iters));
    report("ldg_cg_u1", cps, th, time_ms([&](int i) { k_ldg<1, 1><<<sms * cps, th>>>(BUF(i), nchunks, table, out); }, iters));
  }
  report("ldg_ca_u1", 8, 256, time_ms([&](int i) { k_ldg<2, 1><<<sms * 8, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("ldg_nc_noalloc_u1", 8, 256, time_ms([&](int i) { k_ldg<3, 1><<<sms * 8, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("ldg_nc_evictlast_u1", 8, 256, time_ms([&](int i) { k_ldg<4, 1><<<sms * 8, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("ldg_nc_u2", 4, 256, time_ms([&](int i) { k_ldg<0, 2><<<sms * 4, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("ldg_cg_u2", 4, 256, time_ms([&](int i) { k_ldg<1, 2><<<sms * 4, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("ldg_nc_u2", 8, 256, time_ms([&](int i) { k_ldg<0, 2><<<sms * 8, 256>>>(BUF(i), nchunks, table, out); }, iters));
  report("tex", 8, 256, time_ms([&](int i) { k_tex<<<sms * 8, 256>>>(BUF(i), nchunks, tex, out); }, iters));
  report("tex", 2, 1024, time_ms([&](int i) { k_tex<<<sms * 2, 1024>>>(BUF(i), nchunks, tex, out); }, iters));

  CK(cudaFuncSetAttribute(k_lds<13>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16));
  report("lds_8192entries", 1, 1024, time_ms([&](int i) { k_lds<13><<<sms, 1024, 8192 * 16>>>(BUF(i), nchunks, table, out); }, iters));
  report("lds_8192entries", 1, 512, time_ms([&](int i) { k_lds<13><<<sms, 512, 8192 * 16>>>(BUF(i), nchunks, table, out); }, iters));
  CK(cudaFuncSetAttribute(k_lds<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16));
  report("lds_4096entries", 2, 1024, time_ms([&](int i) { k_lds<12><<<sms * 2, 1024, 4096 * 16>>>(BUF(i), nchunks, table, out); }, iters));

  {  // DSMEM, cluster of 8 (128 KB per CTA) and 16 (64 KB per CTA; non-portable)
    CK(cudaFuncSetAttribute(k_dsmem<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16));
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 8; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cfg.gridDim = dim3((sms / 8) * 8); cfg.blockDim = dim3(1024); cfg.dynamicSmemBytes = 8192 * 16;
    report("dsmem_cluster8", 1, 1024, time_ms([&](int i) { CK(cudaLaunchKernelEx(&cfg, k_dsmem<8>, (const uint4*)BUF(i), nchunks, (const uint4*)table, out)); }, iters));
    CK(cudaFuncSetAttribute(k_dsmem<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16));
    if (cudaFuncSetAttribute(k_dsmem<16>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
      at[0].val.clusterDim.x = 16;
      cfg.gridDim = dim3((sms / 16) * 16); cfg.dynamicSmemBytes = 4096 * 16;
      cudaError_t e = cudaLaunchKernelEx(&cfg, k_dsmem<16>, (const uint4*)BUF(0), nchunks, (const uint4*)table, out);
      if (e == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess)
        report("dsmem_cluster16", 1, 1024, time_ms([&](int i) { CK(cudaLaunchKernelEx(&cfg, k_dsmem<16>, (const uint4*)BUF(i), nchunks, (const uint4*)table, out)); }, iters));
      else { cudaGetLastError(); printf("{\"variant\": \"dsmem_cluster16\", \"skipped\": \"%s\"}\n", cudaGetErrorString(e)); }
    }
  }
  CK(cudaFuncSetAttribute(k_hybrid<12288, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 16));
  report("hybrid_12288smem_nc", 1, 1024, time_ms([&](int i) { k_hybrid<12288, 0><<<sms, 1024, 12288 * 16>>>(BUF(i), nchunks, table, out); }, iters));
  CK(cudaFuncSetAttribute(k_hybrid<12288, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 16));
  report("hybrid_12288smem_cg", 1, 1024, time_ms([&](int i) { k_hybrid<12288, 1><<<sms, 1024, 12288 * 16>>>(BUF(i), nchunks, table, out); }, iters));

  CK(cudaFuncSetAttribute(k_split<13108>, cudaFuncAttributeMaxDynamicSharedMemorySize, 13109 * 16));
  report("split5_smem_zero_slot", 1, 1024, time_ms([&](int i) { k_split<13108><<<(sms / 5) * 5, 1024, 13109 * 16>>>(BUF(i), nchunks, table, 5, out); }, iters));
  CK(cudaFuncSetAttribute(k_split<6554>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6555 * 16));
  report("split10_smem_zero_slot", 2, 1024, time_ms([&](int i) { k_split<6554><<<(sms * 2 / 10) * 10, 1024, 6555 * 16>>>(BUF(i), nchunks, table, 10, out); }, iters));
  CK(cudaDeviceSynchronize());
  return 0;
}
