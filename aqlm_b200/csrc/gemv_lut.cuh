// Batch-1 GEMV for 256-entry codebooks (Kx8 schemes: 1x8, 2x8, 4x8, 8x8), dot-product LUT formulation.
//
//   y[o] = scale[o] * sum_j sum_k L[j][k][code[o,j,k]],     L[j][k][c] = codebook[k][c] . x_j   (fp32)
//
// Replaces Code2x8MatVec / CodeKx8MatVec (reference cuda_kernel.cu:144-233, 296-390) and the Triton kernel the
// reference uses for 8x8 (kernel_selector.py:91-94).  The reference's direct kernels gather a 16-byte codebook
// vector per code from shared memory (8x replicated to dodge bank conflicts, cuda_kernel.cu:168-173) and do 8
// FMAs per code; its CPU kernel (numba_kernel.py:37-48) uses the LUT idea.  Here every code byte costs ONE
// conflict-free 4-byte shared-memory read and one add:
//   * a CTA owns a slab of J in-groups (J = 32, or 16 for K = 8) and a block of output rows;
//   * the LUT [K][256][J] fp32 is built in shared memory by tensor cores (mma.sync m16n8k8, exact fp16/bf16
//     products, fp32 accumulate) and stored so that lane <-> group <-> bank: lookups never conflict for J = 32;
//   * each lane streams the K code bytes of ITS group for 32 rows (coalesced 64-byte row segments, all loads in
//     flight), looks them up, and a 31-shuffle transpose-reduce leaves lane l with the total of row l;
//   * per-slab partial rows go to an fp32 workspace; the LAST CTA of a row block (atomic ticket) adds the slabs
//     in a fixed order and applies scale + bias (deterministic, no float atomics).
#pragma once

#include <type_traits>

#include "common.cuh"

namespace aqlm_b200 {

struct LutParams {
  const void* codes;
  const void* codebooks;
  const void* scales;
  const void* bias;
  const void* x;       // [in_features]
  void* y;             // [out_features] T, or float when partial_f32
  float* ws_partials;  // [n_slabs][out_features]
  unsigned int* ws_counters;  // [row_blocks] arrival tickets, zero on entry, left zero
  unsigned int* ws_gen;       // [row_blocks] generation words (monotonic; any value on entry)
  int out_features;
  int in_groups;
  int n_slabs;
  int rows_per_block;  // multiple of 32
  int partial_f32;
};


__device__ __forceinline__ void mma_m16n8k8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0, bool bf16) {
  if (bf16) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(b0));
  } else {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(b0));
  }
}

// K codebooks, J groups per slab (32 -> one row per warp step, 16 -> two rows per warp step)
template <typename T, int K, int J, int kLutThreads>
__global__ void __launch_bounds__(kLutThreads, (kLutThreads == 256) ? 2 : 1) gemv_lut_kernel(const LutParams p) {
  // [K][256][J] fp32 LUT at shared-memory offset 0 (the kernel has NO static shared memory), so a lookup address is
  // just (code << log2(4J)) | lane_constant; one extra word after the LUT holds the "last CTA" flag
  extern __shared__ __align__(16) float lut[];
  constexpr int NT = J / 8;                     // n-tiles (8 groups each) per slab
  constexpr int RPW = 32 / J;                   // rows per warp step
  constexpr int kWarps = kLutThreads / 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slab = blockIdx.x, rb = blockIdx.y;
  const int j0 = slab * J;
  griddep_launch_dependents();

  // lane <-> group mapping of the lookup phase
  const int jj = lane & (J - 1);
  const int rsub = lane / J;  // 0 for J == 32; 0/1 for J == 16
  const int g = j0 + jj;
  const bool g_ok = g < p.in_groups;
  const size_t row_bytes = (size_t)p.in_groups * K;
  const uint8_t* cbase = reinterpret_cast<const uint8_t*>(p.codes) + (size_t)g * K;
  const uint32_t lane_off = (uint32_t)jj * 4u;
  const int row_begin = rb * p.rows_per_block;
  const int row_end = min(p.out_features, row_begin + p.rows_per_block);
  constexpr int RB = J;  // values per lane per batch; the butterfly leaves one row total per lane
  constexpr int CWN = (K + 3) / 4;
  float* part = p.ws_partials + (size_t)slab * p.out_features;

  auto load_one = [&](const uint8_t* src, uint32_t (&c)[CWN]) {
    if constexpr (K == 1) c[0] = (uint32_t)__ldg(src);
    else if constexpr (K == 2) c[0] = (uint32_t)__ldg(reinterpret_cast<const uint16_t*>(src));
    else if constexpr (K == 4) c[0] = __ldg(reinterpret_cast<const uint32_t*>(src));
    else {
      const uint2 t2 = __ldg(reinterpret_cast<const uint2*>(src));
      c[0] = t2.x; c[1] = t2.y;
    }
  };
  auto load_codes = [&](int r0, uint32_t (&cw)[RB][CWN]) {
    const uint8_t* src = cbase + (size_t)(r0 + rsub) * row_bytes;
    const size_t stride = (size_t)RPW * row_bytes;
    if (g_ok && r0 + RB * RPW <= row_end) {  // fast path: whole batch in range, no per-row predicates
#pragma unroll
      for (int i = 0; i < RB; ++i, src += stride) load_one(src, cw[i]);
    } else {
#pragma unroll
      for (int i = 0; i < RB; ++i, src += stride) {
#pragma unroll
        for (int q = 0; q < CWN; ++q) cw[i][q] = 0u;
        if (g_ok && r0 + i * RPW + rsub < row_end) load_one(src, cw[i]);
      }
    }
  };

  // ---- prologue (weights only, overlaps the previous kernel under PDL): first batch of codes (HBM) and this warp's
  //      codebook fragments (L2) go in flight before anything waits ----
  constexpr int kBatchStride = kWarps * RB * RPW;
  uint32_t cwa[RB][CWN], cwb[RB][CWN];
  int r0 = row_begin + warp * (RB * RPW);
  load_codes(r0, cwa);
  if (r0 + kBatchStride < row_end) load_codes(r0 + kBatchStride, cwb);
  constexpr int MT = (K * 16) / kWarps;  // 16-entry tiles per warp (K*16 tiles, 8 warps)
  static_assert((K * 16) % kWarps == 0, "tiles must divide evenly");
  const int q = lane >> 2, m = lane & 3;
  uint32_t afrag[MT][2];
  {
    const uint32_t* cb32 = reinterpret_cast<const uint32_t*>(p.codebooks);
#pragma unroll
    for (int u = 0; u < MT; ++u) {
      const int e0 = (warp + u * kWarps) * 16;  // global entry index (k*256 + c)
      afrag[u][0] = __ldg(cb32 + (size_t)(e0 + q) * 4 + m);
      afrag[u][1] = __ldg(cb32 + (size_t)(e0 + q + 8) * 4 + m);
    }
  }
  griddep_wait();  // x is produced by the previous kernel

  // ---------------- LUT build: D[16 entries x 8 groups] = CB[16 x 8] . X^T[8 x 8], tensor cores ----------------
  // The host launches no empty slab, so the guard always holds.  It keeps ptxas from scheduling the build together with
  // the lookups: for K = 8 that costs one extra instruction per lookup and ~3% of the 8x8 GEMV's time on an H100.
  if (j0 < p.in_groups) {
    // column (2m'+i) of n-tile t holds group (2*NT)*m' + 2t + i, so a lane ends up with 2*NT consecutive groups
    uint32_t bfrag[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int gg = j0 + (2 * NT) * (q >> 1) + 2 * t + (q & 1);
      uint32_t v = 0;
      if (gg < p.in_groups) v = reinterpret_cast<const uint32_t*>(p.x)[gg * 4 + m];
      bfrag[t] = v;
    }
#pragma unroll
    for (int u = 0; u < MT; ++u) {
      const int e0 = (warp + u * kWarps) * 16;
      float d[NT][4];
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        d[t][0] = d[t][1] = d[t][2] = d[t][3] = 0.f;
        mma_m16n8k8(d[t], afrag[u][0], afrag[u][1], bfrag[t], DT<T>::is_bf16);
      }
      // lane holds, for entry e0+q, groups (2NT)m .. (2NT)m + 2NT-1 in d[t][0..1]; for entry e0+q+8 in d[t][2..3]
      float* ra = lut + (size_t)(e0 + q) * J + (2 * NT) * m;
      float* rb8 = lut + (size_t)(e0 + q + 8) * J + (2 * NT) * m;
      if constexpr (NT == 4) {
        // two 16-byte stores per entry; odd rows store the upper half first so that a quarter-warp hits 32 distinct banks
        const bool odd = q & 1;
        const float4 lo0 = make_float4(d[0][0], d[0][1], d[1][0], d[1][1]), hi0 = make_float4(d[2][0], d[2][1], d[3][0], d[3][1]);
        const float4 lo1 = make_float4(d[0][2], d[0][3], d[1][2], d[1][3]), hi1 = make_float4(d[2][2], d[2][3], d[3][2], d[3][3]);
        *reinterpret_cast<float4*>(ra + (odd ? 4 : 0)) = odd ? hi0 : lo0;
        *reinterpret_cast<float4*>(ra + (odd ? 0 : 4)) = odd ? lo0 : hi0;
        *reinterpret_cast<float4*>(rb8 + (odd ? 4 : 0)) = odd ? hi1 : lo1;
        *reinterpret_cast<float4*>(rb8 + (odd ? 0 : 4)) = odd ? lo1 : hi1;
      } else {
        // J = 16: one 16-byte store per entry; consecutive entries alternate bank halves
        *reinterpret_cast<float4*>(ra) = make_float4(d[0][0], d[0][1], d[1][0], d[1][1]);
        *reinterpret_cast<float4*>(rb8) = make_float4(d[0][2], d[0][3], d[1][2], d[1][3]);
      }
    }
  }
  __syncthreads();

  // ---------------- lookups: lane <-> group <-> bank; two batches of code loads are always in flight ----------------
  auto process = [&](int rbase, uint32_t (&cw)[RB][CWN]) {
    float v[RB];
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        // address = (code * 4J) | lane_off + k * 256 * 4J : shift + (and|or) + LDS with an immediate offset
        constexpr int SH = (J == 32) ? 7 : 6;  // log2(4 * J)
        const int bit = (k & 3) * 8;
        const uint32_t w = cw[i][k >> 2];
        const uint32_t sh = bit >= SH ? (w >> (bit - SH)) : (w << (SH - bit));
        const uint32_t off = (sh & (0xffu << SH)) | lane_off;  // byte offset inside codebook k's LUT
        acc += *reinterpret_cast<const float*>(reinterpret_cast<const char*>(lut) + (size_t)k * 256 * 4 * J + off);
        // (rows/groups out of range hold code 0: harmless, never stored)
      }
      v[i] = acc;
    }
    // refill this buffer with the batch after next before the shuffle phase
    if (rbase + 2 * kBatchStride < row_end) load_codes(rbase + 2 * kBatchStride, cw);
    // transpose-reduce over the J lanes of a row group: lane jj ends with the total of row index jj of the batch
#pragma unroll
    for (int d = J / 2, n = RB; d >= 1; d >>= 1, n >>= 1) {
      const bool up = (lane & d) != 0;
#pragma unroll
      for (int i = 0; i < n / 2; ++i) {
        const float send = up ? v[i] : v[i + n / 2];
        const float keep = up ? v[i + n / 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, d);
      }
    }
    const int row = rbase + jj * RPW + rsub;
    if (row < row_end) part[row] = v[0];
  };
  for (; r0 < row_end; r0 += 2 * kBatchStride) {
    process(r0, cwa);
    if (r0 + kBatchStride < row_end) process(r0 + kBatchStride, cwb);
  }

  // ---------------- fix-up: ALL slab CTAs of this row block share the cross-slab sum ----------------
  // The grid is one resident wave (host side guarantees it), so the n_slabs CTAs of a row block can rendezvous: each
  // publishes its partials, takes a ticket, and the last arrival bumps the block's generation word; everybody then adds
  // the slabs IN SLAB ORDER (deterministic) for its own 1/n_slabs share of the rows (32-row chunks dealt round-robin).
  // (Letting only the last-arriving CTA do the whole block puts n_slabs x rows loads behind one L2 round trip each.)
  unsigned int* s_gen = reinterpret_cast<unsigned int*>(lut + (size_t)K * 256 * J);
  if (tid == 0) *s_gen = *reinterpret_cast<volatile unsigned int*>(p.ws_gen + rb);  // cannot advance before I arrive
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int g0 = *s_gen;
    const unsigned int old = atomicAdd(p.ws_counters + rb, 1u);
    if (old == (unsigned int)p.n_slabs - 1) {
      p.ws_counters[rb] = 0u;  // leave the ticket clean for the next call
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p.ws_gen + rb), "r"(g0 + 1u) : "memory");
    } else {
      unsigned int g;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(g) : "l"(p.ws_gen + rb) : "memory");
      } while (g == g0);
    }
  }
  __syncthreads();
  {
    const int chunks = (row_end - row_begin + 31) >> 5;
    for (int c = slab + warp * p.n_slabs; c < chunks; c += kWarps * p.n_slabs) {
      const int row = row_begin + (c << 5) + lane;
      if (row >= row_end) continue;
      float acc = 0.f;
      int sidx = 0;
      for (; sidx + 8 <= p.n_slabs; sidx += 8) {  // 8 independent L2 loads in flight, added in slab order
        float t8[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) t8[u] = __ldcg(p.ws_partials + (size_t)(sidx + u) * p.out_features + row);
#pragma unroll
        for (int u = 0; u < 8; ++u) acc += t8[u];
      }
      for (; sidx < p.n_slabs; ++sidx) acc += __ldcg(p.ws_partials + (size_t)sidx * p.out_features + row);
      if (p.partial_f32) {
        reinterpret_cast<float*>(p.y)[row] = acc;
      } else {
        const float sc = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        const float bi = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
        reinterpret_cast<T*>(p.y)[row] = DT<T>::from_float(fmaf(acc, sc, bi));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Cluster variant for K = 1, 2 and in_features <= 8 slabs of 64 groups (4096 for g = 8): the slab CTAs of a row block form
// ONE thread-block cluster and reduce their partial rows through DISTRIBUTED SHARED MEMORY -- no workspace, no global
// partials, no fence/atomic/poll round trips through global memory.  One CTA per SM.
//   * slab = 64 in-groups, LUT [K][256][64] fp32 (64/128 KiB), built by tensor cores as in gemv_lut_kernel.  A LUT row
//     (one entry, 64 groups) is 256 bytes.
//   * a lane owns the ADJACENT groups 2l, 2l+1: one aligned code word per row (K=2: 4 bytes, K=1: 2 bytes) = a fully
//     coalesced 128/64-byte row segment per warp.  Group 2l sits at LUT position l and group 2l+1 at position 32+l, so
//     both lookups of a lane hit bank l: the lookups never conflict.
//   * ONE instruction of address arithmetic per lookup.  The LUT is placed at the first 64 KiB boundary of the CTA's
//     shared window above the receive buffers (window offset 0x10000; codebook k at 0x10000 * (1 + k)), so the address of
//     entry `code` for the lane's even group is  {byte3, byte2, byte1, byte0} = {base.hi, base.lo + k, code, 4 * lane}:
//     one PRMT takes the code byte straight out of the packed code word and the other three bytes from a per-lane
//     constant; the odd group is the immediate offset +128 of the LDS.  The ~63 KiB below 0x10000 are not wasted on this
//     1-CTA/SM kernel: they hold the receive buffers of the cross-slab sum.
//   * every warp owns ONE batch of 16 rows: the CTA is launched with as many warps as its row block has batches (8 to 32,
//     MAXT = 768 or 1024 threads), so there is no second, mostly empty, round and nothing is double-buffered.  16 rows
//     over 32 lanes: the two half-warps are folded first, then a 15-shuffle transpose-reduce over 16 lanes leaves lane l
//     with the slab total of row l of the batch.
//   * the cross-slab sum is PUSH-based: a lane that holds the slab total of a row stores it (st.shared::cluster) into the
//     receive buffer of the CTA that owns the row's share; after ONE cluster barrier every CTA adds the n_slabs values of
//     its rows from its OWN shared memory, in slab order (deterministic).  No remote loads, no second barrier (nobody
//     touches a peer's memory after the barrier).
// ---------------------------------------------------------------------------------------------------
struct LutClusterParams {
  const void* codes;
  const void* codebooks;
  const void* scales;
  const void* bias;
  const void* x;
  void* y;
  int out_features;
  int in_groups;
  int n_slabs;         // = cluster size along x
  int rows_per_block;  // multiple of 32
  int partial_f32;
};

constexpr int kLutCJ = 64;
constexpr uint32_t kLutAbs = 0x10000u;  // absolute shared-memory address of LUT 0

template <typename T, int K, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) gemv_lut_cluster_kernel(const LutClusterParams p) {
  static_assert(K == 1 || K == 2, "cluster LUT kernel: one or two 256-entry codebooks");
  constexpr int RB = 16;  // rows per warp batch
  extern __shared__ __align__(16) uint8_t smem_dyn[];
  constexpr int J = kLutCJ, NT = J / 8;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_warps = (int)blockDim.x >> 5;
  const int slab = blockIdx.x, rb = blockIdx.y;
  const int j0 = slab * J;
  griddep_launch_dependents();
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");  // "I have started" (waited for before the pushes)
  // The shared-window address of this CTA's dynamic shared memory.  Only its low 16 bits are assumed small: inside a
  // cluster the upper bits of a shared::cta address may carry the CTA's position in the shared::cluster window, so the LUT
  // base is "the next 64 KiB boundary above the receive buffers", whatever those upper bits are.
  const uint32_t dyn_base = (uint32_t)__cvta_generic_to_shared(smem_dyn);
  const uint32_t lut_base = (dyn_base & 0xffff0000u) + kLutAbs;                      // absolute address of LUT 0
  float* recv = reinterpret_cast<float*>(smem_dyn);                                 // [n_slabs][per], below the LUT
  float* lut = reinterpret_cast<float*>(smem_dyn + (lut_base - dyn_base));          // [K][256][64] fp32
  const int row_begin = rb * p.rows_per_block;
  const int row_end = min(p.out_features, row_begin + p.rows_per_block);
  const int per = (p.rows_per_block + p.n_slabs - 1) / p.n_slabs;  // rows of a block that one CTA finishes
  // (the host sizes the window as 64 KiB + the LUT; the dynamic area starts ~1 KiB into a 64 KiB-aligned window)
  if ((dyn_base & 0xffffu) + 4u * (uint32_t)(p.n_slabs * per) > kLutAbs) __trap();
  const size_t row_bytes = (size_t)p.in_groups * K;
  using CodeWord = typename std::conditional<K == 2, uint32_t, uint16_t>::type;
  const bool g_ok = j0 + 2 * lane + 1 < p.in_groups;
  const uint8_t* cbase = reinterpret_cast<const uint8_t*>(p.codes) + (size_t)(j0 + 2 * lane) * K;
  const int batch_stride = n_warps * RB;
  auto load_codes = [&](int r0, uint32_t (&cw)[RB]) {
    const uint8_t* src = cbase + (size_t)r0 * row_bytes;
    if (g_ok && r0 + RB <= row_end) {
#pragma unroll
      for (int i = 0; i < RB; ++i, src += row_bytes) cw[i] = (uint32_t)__ldg(reinterpret_cast<const CodeWord*>(src));
    } else {
#pragma unroll
      for (int i = 0; i < RB; ++i, src += row_bytes) {
        cw[i] = 0u;
        if (g_ok && r0 + i < row_end) cw[i] = (uint32_t)__ldg(reinterpret_cast<const CodeWord*>(src));
      }
    }
  };
  // ---- prologue (weights only; overlaps the previous kernel under PDL) ----
  uint32_t cw[RB];
  int r0 = row_begin + warp * RB;
  if (r0 < row_end) load_codes(r0, cw);
  const int q = lane >> 2, m = lane & 3;
  const uint32_t* cb32 = reinterpret_cast<const uint32_t*>(p.codebooks);
  uint32_t a0 = 0, a1 = 0;
  if (warp < K * 16) {
    a0 = __ldg(cb32 + (size_t)(warp * 16 + q) * 4 + m);
    a1 = __ldg(cb32 + (size_t)(warp * 16 + q + 8) * 4 + m);
  }
  griddep_wait();  // x is produced by the previous kernel
  // ---- LUT build (tensor cores), 16-entry tiles dealt to the warps ----
  {
    uint32_t bfrag[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      const int gg = j0 + 16 * (q >> 1) + 2 * t + (q & 1);
      bfrag[t] = gg < p.in_groups ? reinterpret_cast<const uint32_t*>(p.x)[gg * 4 + m] : 0u;
    }
    for (int tile = warp; tile < K * 16; tile += n_warps) {
      if (tile != warp) {
        a0 = __ldg(cb32 + (size_t)(tile * 16 + q) * 4 + m);
        a1 = __ldg(cb32 + (size_t)(tile * 16 + q + 8) * 4 + m);
      }
      const int e0 = tile * 16;
      float* ra = lut + (size_t)(e0 + q) * J + 8 * m;
      float* rb8 = lut + (size_t)(e0 + q + 8) * J + 8 * m;
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // two passes of 4 n-tiles (keeps the accumulators at 16 registers).  Every lane of a
                                     // pass holds the SAME half, so the even and the odd entry row of a quarter-warp store
                                     // to the same banks: a 2-way conflict on the build stores, the price of those registers
        float d[4][4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          d[t][0] = d[t][1] = d[t][2] = d[t][3] = 0.f;
          mma_m16n8k8(d[t], a0, a1, bfrag[4 * h + t], DT<T>::is_bf16);
        }
        const int off = h * 4;  // n-tiles 4h .. 4h+3 live at positions 8m + 4h + t
        // accumulator column c: 0/1 = entry e0+q, even/odd groups; 2/3 = entry e0+q+8
        *reinterpret_cast<float4*>(ra + off) = make_float4(d[0][0], d[1][0], d[2][0], d[3][0]);
        *reinterpret_cast<float4*>(ra + 32 + off) = make_float4(d[0][1], d[1][1], d[2][1], d[3][1]);
        *reinterpret_cast<float4*>(rb8 + off) = make_float4(d[0][2], d[1][2], d[2][2], d[3][2]);
        *reinterpret_cast<float4*>(rb8 + 32 + off) = make_float4(d[0][3], d[1][3], d[2][3], d[3][3]);
      }
    }
  }
  __syncthreads();
  asm volatile("barrier.cluster.wait.aligned;" ::: "memory");  // every CTA of the cluster runs: its shared memory may be written
  // ---- lookups: PRMT -> LDS -> FADD per code byte ----
  const uint32_t c0 = lut_base | ((uint32_t)lane << 2);
  const uint32_t c1 = (lut_base + kLutAbs) | ((uint32_t)lane << 2);
  const uint32_t recv_s = dyn_base;
  for (; r0 < row_end; r0 += batch_stride) {
    if (r0 != row_begin + warp * RB) load_codes(r0, cw);  // (row blocks of more than 32 batches: later rounds, not prefetched)
    float v[RB];
#pragma unroll
    for (int i = 0; i < RB; ++i) {
      const uint32_t w = cw[i];
      float t0, t1, t2, t3;
      if constexpr (K == 2) {  // bytes: [g0 k0][g0 k1][g1 k0][g1 k1]
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t0) : "r"(__byte_perm(w, c0, 0x7604)));
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t1) : "r"(__byte_perm(w, c1, 0x7614)));
        asm volatile("ld.shared.f32 %0, [%1+128];" : "=f"(t2) : "r"(__byte_perm(w, c0, 0x7624)));
        asm volatile("ld.shared.f32 %0, [%1+128];" : "=f"(t3) : "r"(__byte_perm(w, c1, 0x7634)));
        v[i] = (t0 + t1) + (t2 + t3);
      } else {                 // bytes: [g0][g1]
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t0) : "r"(__byte_perm(w, c0, 0x7604)));
        asm volatile("ld.shared.f32 %0, [%1+128];" : "=f"(t1) : "r"(__byte_perm(w, c0, 0x7614)));
        v[i] = t0 + t1;
      }
    }
    // 16 rows over 32 lanes: fold the two half-warps first, then transpose-reduce over 16 lanes
#pragma unroll
    for (int i = 0; i < RB; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], 16);
#pragma unroll
    for (int dd = RB / 2, n = RB; dd >= 1; dd >>= 1, n >>= 1) {
      const bool up = (lane & dd) != 0;
#pragma unroll
      for (int i = 0; i < n / 2; ++i) {
        const float send = up ? v[i] : v[i + n / 2];
        const float keep = up ? v[i + n / 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, dd);
      }
    }
    // lane (l & (RB-1)) holds the slab total of row r0 + (l & (RB-1)): push it to the CTA that finishes that row
    const int rr = r0 - row_begin + (lane & (RB - 1));
    if (lane < RB && r0 + (lane & (RB - 1)) < row_end) {
      const int owner = rr / per;
      const uint32_t local = recv_s + 4u * (uint32_t)(slab * per + (rr - owner * per));
      uint32_t remote;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"((uint32_t)owner));
      asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(v[0]) : "memory");
    }
  }
  // ---- cross-slab sum: everything I need has been pushed into MY shared memory once the cluster barrier completes ----
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  {
    const int nrows = row_end - row_begin;
    const int lo = slab * per, hi = min(nrows, lo + per);
    for (int r = lo + tid; r < hi; r += (int)blockDim.x) {
      float acc = 0.f;
      for (int s2 = 0; s2 < p.n_slabs; ++s2) acc += *reinterpret_cast<volatile float*>(recv + s2 * per + (r - lo));
      const int row = row_begin + r;
      if (p.partial_f32) {
        reinterpret_cast<float*>(p.y)[row] = acc;
      } else {
        const float sc = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        const float bi = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
        reinterpret_cast<T*>(p.y)[row] = DT<T>::from_float(fmaf(acc, sc, bi));
      }
    }
  }
}

}  // namespace aqlm_b200
