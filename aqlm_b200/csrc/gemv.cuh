// Fused code-gather + additive dequant + GEMV (batch <= 8 rows per pass) with scale/bias epilogue.
//
// Replaces Code1x16MatVec / Code2x8MatVec / CodeKx8MatVec (reference cuda_kernel.cu:7-95, 144-233,
// 296-390) plus the host loop and the 3-4 epilogue launches around them (cuda_kernel.cpp:148-182,
// 95-111), and the Triton path used for 8x8 (kernel_selector.py:91-94).  Not a port: the kernel is
// persistent (grid sized from the SM count), stages x once per CTA in XOR-swizzled shared memory, reads
// each lane's 16-byte code chunk with ONE 128-bit streaming load (the reference compiles to 8 two-byte
// loads, SURVEY §2b), accumulates in fp32, handles up to 8 batch rows per pass against one gather of the
// weights, and applies scale+bias in the same launch.
#pragma once

#include "common.cuh"

namespace aqlm_b200 {

struct GemvParams {
  const void* codes;
  const void* codebooks;
  const void* scales;
  const void* bias;
  const void* x;  // [batch, in_features]
  void* y;        // [batch, out_features] T, or float when partial
  int out_features;
  int in_groups;
  int in_features;
  int nbits;
  int num_codebooks;  // runtime K for the generic kernel
  int batch;          // rows in this pass (<= BT)
  int partial_f32;
  // grouped launch (several linears sharing x, rows concatenated): segment i covers rows [seg_end[i-1], seg_end[i]) and
  // uses the codebook at codebooks + i * (K << nbits) * g elements.  n_seg == 1 for a plain linear.
  int n_seg;
  int seg_end[4];
  // rows per CTA when every CTA owns ONE CONTIGUOUS block of rows (0: rows dealt round-robin).  The fused exchange needs
  // contiguous blocks so that a CTA's partials travel as 16-byte vectors.
  int row_block;
};

// Peer-memory exchange fused into the GEMV (in_features-sharded path): see gemv_1x16_kernel<..., PEER = true>.
struct GemvPeer {
  uint8_t* peer_base[16];  // every rank's shared buffer as mapped in this process (flags, then [set][src rank][max_elems] floats)
  unsigned int* step;      // local: steps completed (advanced by the last CTA)
  unsigned int* tickets;   // local: [2], zero on entry, left zero
  long long max_elems;
  int rank, world;
  long long ll_offset;     // byte offset of the tagged-word slots ([set][src rank][max_elems] u64) in each shared buffer
};

constexpr int kGemvThreads = 256;  // generic (fallback) kernel
constexpr int kSliceChunks = 32;   // one K-slice = 32 16-byte code chunks = one coalesced 512-byte warp load

// ---------------------------------------------------------------------------------------------------
// Vector path: a row of codes is a whole number of 16-byte chunks and K*CODE_BYTES divides 16.
//   T          __half | __nv_bfloat16
//   K          codebooks per group;  CODE_BYTES 1|2;  G in_group_size (8|16);  BT batch rows per pass
//   CBS        codebooks staged in shared memory (256-entry codebooks) vs gathered from global/L2 (1x16)
//   THREADS    CTA size; the grid is persistent: (SM count) x (CTAs per SM that fit)
//
// Work decomposition (load balance is what matters: the kernel is bound by the per-SM gather rate, so every
// SM must get the same number of gathers): output rows are dealt round-robin to CTAs (row r -> CTA r % grid),
// each row is cut into K-slices of 32 chunks, and the (row, slice) tasks of a CTA are dealt round-robin to its
// warps.  A warp reduces its task with shuffles and parks the partial in shared memory; after one barrier the
// CTA adds the slices of each of its rows IN A FIXED ORDER (deterministic, batch-invariant) and applies
// scale + bias.  No atomics, no second launch.
// ---------------------------------------------------------------------------------------------------
template <typename T, int K, int CODE_BYTES, int G, int BT, bool CBS, int THREADS>
__global__ void __launch_bounds__(THREADS, 1) gemv_vec_kernel(const GemvParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  constexpr int GPC = 16 / (K * CODE_BYTES);  // groups per 16-byte chunk
  constexpr int UPG = G / 8;                  // 16-byte units per group
  constexpr int kWarps = THREADS / 32;
  const int upr = p.in_features >> 3;         // 16-byte units per x row
  // PDL: let the next kernel in the stream start launching; everything below that touches only WEIGHTS
  // (codes, codebooks) may overlap the previous kernel's tail.  x and y are touched after griddep_wait().
  griddep_launch_dependents();
  if ((int)blockIdx.x >= p.out_features) return;

  uint4* sx = reinterpret_cast<uint4*>(smem_raw);
  uint4* scb = sx + BT * upr;  // [K][2^nbits][UPG] when CBS
  float* spart = reinterpret_cast<float*>(scb + (CBS ? (K << p.nbits) * UPG : 0));  // [rows_cta][slices][BT]

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int chunks = p.in_groups / GPC;
  const int slices = (chunks + kSliceChunks - 1) / kSliceChunks;
  const int rows_cta = (p.out_features - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int tasks = rows_cta * slices;
  const size_t row_bytes = (size_t)p.in_groups * K * CODE_BYTES;
  const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);

  // code chunk of task t for this lane (zero chunk when the lane is past the end of the row)
  auto load_codes = [&](int t, bool& live) -> uint4 {
    const int ri = t / slices;
    const int sl = t - ri * slices;
    const int c = sl * kSliceChunks + lane;
    live = (t < tasks) && (c < chunks);
    if (!live) return make_uint4(0, 0, 0, 0);
    const int row = (int)blockIdx.x + ri * (int)gridDim.x;
    return ld_stream_v4(reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.codes) + row * row_bytes) + c);
  };

  // ---- prologue: first code chunk in flight, codebooks (weights) staged, THEN wait for x -----------
  bool live_next = false;
  uint4 cw_next = load_codes(warp, live_next);
  if constexpr (CBS) {
    const int n = (K << p.nbits) * UPG;
    for (int u = tid; u < n; u += THREADS) scb[u] = gcb[u];
  }
  griddep_wait();
  {
    const uint4* gx = reinterpret_cast<const uint4*>(p.x);
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      if (b < p.batch) {
        for (int u = tid; u < upr; u += THREADS) sx[b * upr + swz16(u)] = gx[(size_t)b * upr + u];
      } else {
        for (int u = tid; u < upr; u += THREADS) sx[b * upr + u] = make_uint4(0, 0, 0, 0);
      }
    }
  }
  __syncthreads();

  for (int t = warp; t < tasks; t += kWarps) {
    const uint4 cw = cw_next;
    const bool live = live_next;
    cw_next = load_codes(t + kWarps, live_next);  // prefetch: hides the HBM latency of the code stream
    const int sl = t % slices;
    const int c = sl * kSliceChunks + lane;
    float acc[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = 0.f;
    if (live) {
      if constexpr (K == 1) {
        // single codebook: keep the gathered vectors packed, issue all GPC gathers before any math
        uint4 wv[GPC][UPG];
#pragma unroll
        for (int e = 0; e < GPC; ++e) {
          const uint32_t code = chunk_code<CODE_BYTES>(cw, e);
          if constexpr (!CBS && UPG == 2) {  // g = 16: the 32-byte entry is one 256-bit request
            ld_gather_v8(gcb + (size_t)code * 2, wv[e][0], wv[e][1]);
          } else {
#pragma unroll
            for (int h = 0; h < UPG; ++h) {
              if constexpr (CBS) wv[e][h] = scb[code * UPG + h];
              else wv[e][h] = ld_gather_v4<0>(gcb + (size_t)code * UPG + h);
            }
          }
        }
#pragma unroll
        for (int e = 0; e < GPC; ++e) {
          const int u0 = (c * GPC + e) * UPG;
#pragma unroll
          for (int h = 0; h < UPG; ++h) {
#pragma unroll
            for (int b = 0; b < BT; ++b) acc[b] = dot8<T>(wv[e][h], sx[b * upr + swz16(u0 + h)], acc[b]);
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < GPC; ++e) {
          float wf[UPG][8];
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const uint32_t code = chunk_code<CODE_BYTES>(cw, e * K + k);
            const size_t off = (((size_t)k << p.nbits) + code) * UPG;
#pragma unroll
            for (int h = 0; h < UPG; ++h) {
              uint4 v;
              if constexpr (CBS) v = scb[off + h];
              else v = ld_gather_v4<0>(gcb + off + h);
              if (k == 0) unpack8<T>(v, wf[h]);
              else accum8<T>(v, wf[h]);
            }
          }
          const int u0 = (c * GPC + e) * UPG;
#pragma unroll
          for (int h = 0; h < UPG; ++h) {
#pragma unroll
            for (int b = 0; b < BT; ++b) acc[b] = dot8f<T>(wf[h], sx[b * upr + swz16(u0 + h)], acc[b]);
          }
        }
      }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = warp_sum(acc[b]);
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < BT; ++b) spart[(size_t)t * BT + b] = acc[b];
    }
  }
  __syncthreads();

  // ---- fixed-order reduction over slices + epilogue ------------------------------------------------
  for (int i = tid; i < rows_cta * BT; i += THREADS) {
    const int ri = i / BT;
    const int b = i - ri * BT;
    if (b >= p.batch) continue;
    const int row = (int)blockIdx.x + ri * (int)gridDim.x;
    float v = 0.f;
    for (int sl = 0; sl < slices; ++sl) v += spart[((size_t)ri * slices + sl) * BT + b];
    if (p.partial_f32) {
      reinterpret_cast<float*>(p.y)[(size_t)b * p.out_features + row] = v;
    } else {
      const float s = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
      const float bv = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
      reinterpret_cast<T*>(p.y)[(size_t)b * p.out_features + row] = DT<T>::from_float(fmaf(v, s, bv));
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// 1x16 (g = 8) specialisation of the vector path: same decomposition and reduction as gemv_vec_kernel, but
//   * 512-thread CTAs (<= 128 registers): a PDL-launched successor kernel can be co-resident on the SM, so its
//     weight-only prologue (code loads AND the first codebook gathers) overlaps this kernel's tail;
//   * two tasks per warp in flight (double-buffered gather registers): 16 gathers per lane outstanding.
// ---------------------------------------------------------------------------------------------------
constexpr int kGemv1x16Threads = 512;

// PEER = true (in_features-sharded multi-GPU path): the kernel's own reduction epilogue performs the ONE exchange of the
// linear over NVLink peer memory, so a sharded linear is ONE launch and the partials never round-trip through HBM:
//   every CTA owns a contiguous block of output rows (the same block on every rank); after the fixed-order slice sum each
//   thread pushes its element as a tagged 64-bit word {fp32, step} to EVERY rank over NVLink and then spins on the W tagged
//   words of that element in its own buffer, adds them in rank order (deterministic) and applies scale + bias -- no
//   fence, flag or barrier in between (see the epilogue).  A thread only ever waits for the same element of the other ranks.
// Two buffer sets alternate by step parity; `step` is read after griddepcontrol.wait (the previous launch, which
// advances it, has completed).  The grid is one CTA per SM, all co-resident, so the cross-rank wait cannot deadlock.
// LORA (not with PEER): the epilogue adds a LoRA adapter's up-projection (LoraArgs, forward form) to every output
// element before its rounding; the adapter's U row and B row are read from global memory (L1) after griddep_wait().
template <typename T, int BT, bool PEER, bool LORA>
__device__ __forceinline__ void gemv_1x16(const GemvParams& p, const GemvPeer& pc, const LoraArgs& lora) {
  static_assert(!(PEER && LORA), "the fused exchange has no adapter term");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  constexpr int THREADS = kGemv1x16Threads;
  constexpr int kWarps = THREADS / 32;
  const int upr = p.in_features >> 3;
  griddep_launch_dependents();
  if (!PEER && (int)blockIdx.x >= p.out_features) return;  // (a PEER CTA without rows still takes part in the step count)

  uint4* sx = reinterpret_cast<uint4*>(smem_raw);
  float* spart = reinterpret_cast<float*>(sx + BT * upr);  // [rows_cta][slices][BT]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int chunks = p.in_groups >> 3;
  const int slices = (chunks + kSliceChunks - 1) / kSliceChunks;
  // row ownership: round-robin (row = cta + i*grid) or one contiguous block per CTA (row = cta*row_block + i)
  const int row_first = p.row_block ? (int)blockIdx.x * p.row_block : (int)blockIdx.x;
  const int row_step = p.row_block ? 1 : (int)gridDim.x;
  const int rows_cta = p.row_block ? max(0, min(p.row_block, p.out_features - row_first))
                                   : (p.out_features - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int tasks = rows_cta * slices;
  const size_t row_bytes = (size_t)p.in_groups * 2;
  const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);

  auto load_codes = [&](int t, bool& live) -> uint4 {
    const int ri = t / slices;
    const int c = (t - ri * slices) * kSliceChunks + lane;
    live = (t < tasks) && (c < chunks);
    if (!live) return make_uint4(0, 0, 0, 0);
    const int row = row_first + ri * row_step;
    return ld_stream_v4(reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.codes) + row * row_bytes) + c);
  };
  // codebook of the segment that owns task t's row (grouped launches stack one 1 MiB codebook per segment)
  auto task_codebook = [&](int t) -> const uint4* {
    if (p.n_seg <= 1) return gcb;
    const int row = row_first + (t / slices) * row_step;
    int seg = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) seg += (i < p.n_seg - 1 && row >= p.seg_end[i]) ? 1 : 0;
    return gcb + (size_t)seg * 65536;
  };
  auto gather = [&](int t, const uint4& cw, uint4 (&w)[8]) {
    const uint4* cb = task_codebook(t);
#pragma unroll
    for (int e = 0; e < 8; ++e) w[e] = ld_gather_v4<0>(cb + chunk_code<2>(cw, e));
  };
  auto consume = [&](int t, bool live, const uint4 (&w)[8]) {
    float acc[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = 0.f;
    if (live) {
      const int c = (t % slices) * kSliceChunks + lane;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
#pragma unroll
        for (int b = 0; b < BT; ++b) acc[b] = dot8<T>(w[e], sx[b * upr + swz16(c * 8 + e)], acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = warp_sum(acc[b]);
    if (lane == 0) {
#pragma unroll
      for (int b = 0; b < BT; ++b) spart[(size_t)t * BT + b] = acc[b];
    }
  };

  // ---- weight-only prologue (may overlap the previous kernel under PDL) ----
  bool liveA = false, liveB = false;
  uint4 wA[8], wB[8];
  uint4 cwA = load_codes(warp, liveA);
  uint4 cwB = load_codes(warp + kWarps, liveB);
  if (liveA) gather(warp, cwA, wA);
  griddep_wait();
  {
    const uint4* gx = reinterpret_cast<const uint4*>(p.x);
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      if (b < p.batch) {
        for (int u = tid; u < upr; u += THREADS) sx[b * upr + swz16(u)] = gx[(size_t)b * upr + u];
      } else {
        for (int u = tid; u < upr; u += THREADS) sx[b * upr + u] = make_uint4(0, 0, 0, 0);
      }
    }
  }
  __syncthreads();

  for (int t = warp; t < tasks; t += 2 * kWarps) {
    // A = task t (gathers already in flight), B = task t + kWarps (codes loaded)
    if (liveB) gather(t + kWarps, cwB, wB);
    bool liveA2;
    cwA = load_codes(t + 2 * kWarps, liveA2);
    consume(t, liveA, wA);
    liveA = liveA2;
    if (liveA) gather(t + 2 * kWarps, cwA, wA);
    const int tb = t + kWarps;
    bool liveB2;
    const bool haveB = tb < tasks;
    const bool liveBcur = liveB;
    cwB = load_codes(t + 3 * kWarps, liveB2);
    if (haveB) consume(tb, liveBcur, wB);
    liveB = liveB2;
  }
  __syncthreads();

  if constexpr (!PEER) {
    for (int i = tid; i < rows_cta * BT; i += THREADS) {
      const int ri = i / BT;
      const int b = i - ri * BT;
      if (b >= p.batch) continue;
      const int row = row_first + ri * row_step;
      float v = 0.f;
      for (int sl = 0; sl < slices; ++sl) v += spart[((size_t)ri * slices + sl) * BT + b];
      if constexpr (LORA) {
        float l = 0.f;
        for (int j = 0; j < lora.rank; j += 4)
          l = dot4(lora_load4<T>(lora.lin, (size_t)b * lora.rank + j, lora.f32),
                   lora_load4<T>(lora.w, (size_t)row * lora.rank + j, lora.f32), l);
        const float s = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        const float bv = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
        reinterpret_cast<T*>(p.y)[(size_t)b * p.out_features + row] =
            DT<T>::from_float(__fadd_rn(fmaf(v, s, bv), __fmul_rn(lora.scaling, l)));
      } else if (p.partial_f32) {
        reinterpret_cast<float*>(p.y)[(size_t)b * p.out_features + row] = v;
      } else {
        const float s = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        const float bv = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
        reinterpret_cast<T*>(p.y)[(size_t)b * p.out_features + row] = DT<T>::from_float(fmaf(v, s, bv));
      }
    }
  } else {
    // ---- fused exchange, low-latency form: every value travels as ONE 64-bit word {fp32 bits, step tag} (like NCCL's LL
    //      protocol), so there is no fence, no flag and no CTA barrier between the push and the reduction: a thread sums
    //      the slices of its (row, batch) element, stores the tagged word into slot [set][my rank] of EVERY rank (8-byte
    //      NVLink stores, coalesced across the warp), then spins on the W tagged words of the same element in its OWN buffer
    //      and adds them in rank order (deterministic).  Two sets alternate by step parity; a tag from two steps ago never
    //      equals the current step. ----
    const unsigned int s = *pc.step + 1u;  // read after griddep_wait(): the launch that advances it has completed
    const int set = (int)(s & 1u);
    auto slot = [&](int dst, int src) -> unsigned long long* {
      return reinterpret_cast<unsigned long long*>(pc.peer_base[dst] + pc.ll_offset) + ((long long)set * pc.world + src) * pc.max_elems;
    };
    const int nelem = rows_cta * BT;
    for (int i = tid; i < nelem; i += THREADS) {
      const int b = i / rows_cta, ri = i - b * rows_cta;
      if (b >= p.batch) continue;
      float v = 0.f;
      for (int sl = 0; sl < slices; ++sl) v += spart[((size_t)ri * slices + sl) * BT + b];
      const unsigned long long word = ((unsigned long long)s << 32) | (unsigned long long)__float_as_uint(v);
      const size_t e = (size_t)b * p.out_features + (row_first + ri);
      for (int r = 0; r < pc.world; ++r)
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(slot(r, pc.rank) + e), "l"(word) : "memory");
    }
    for (int i = tid; i < nelem; i += THREADS) {
      const int b = i / rows_cta, ri = i - b * rows_cta;
      if (b >= p.batch) continue;
      const int row = row_first + ri;
      const size_t e = (size_t)b * p.out_features + row;
      float acc = 0.f;
      for (int r = 0; r < pc.world; ++r) {
        const unsigned long long* src = slot(pc.rank, r) + e;
        unsigned long long w;
        do {
          asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(src) : "memory");
        } while ((unsigned int)(w >> 32) != s);
        acc += __uint_as_float((unsigned int)w);
      }
      const float sc = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
      const float bv = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
      reinterpret_cast<T*>(p.y)[(size_t)b * p.out_features + row] = DT<T>::from_float(fmaf(acc, sc, bv));
    }
    // step bookkeeping: the last CTA to finish advances the local step counter
    __syncthreads();
    if (tid == 0) {
      const unsigned int old = atomicAdd(pc.tickets, 1u);
      if (old == gridDim.x - 1) {
        pc.tickets[0] = 0u;
        __threadfence();
        *pc.step = s;
      }
    }
  }
}

template <typename T, int BT, bool PEER = false>
__global__ void __launch_bounds__(kGemv1x16Threads, 1) gemv_1x16_kernel(const GemvParams p, const GemvPeer pc) {
  gemv_1x16<T, BT, PEER, false>(p, pc, LoraArgs{});
}

// A plain 1x16 linear with a LoRA adapter (rows dealt round-robin, no partials).
template <typename T, int BT>
__global__ void __launch_bounds__(kGemv1x16Threads, 1) gemv_1x16_lora_kernel(const GemvParams p, const LoraArgs lora) {
  gemv_1x16<T, BT, false, true>(p, GemvPeer{}, lora);
}

// ---------------------------------------------------------------------------------------------------
// Generic path: any K <= 16, any nbits <= 16, ragged rows (row bytes not a multiple of 16).  One group
// per lane per step, scalar code loads, x read through L1.  Slow but complete (the reference falls
// back to Triton / embedding_bag here, kernel_selector.py:91-102).
// ---------------------------------------------------------------------------------------------------
template <typename T, int CODE_BYTES, int G, int BT>
__global__ void __launch_bounds__(kGemvThreads) gemv_generic_kernel(const GemvParams p) {
  constexpr int UPG = G / 8;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  constexpr int kWarps = kGemvThreads / 32;
  const int K = p.num_codebooks;
  const int upr = p.in_features >> 3;
  const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);
  // x may be only element-aligned here (this kernel is also the fallback for a misaligned input): 2-byte loads
  const uint16_t* gx16 = reinterpret_cast<const uint16_t*>(p.x);
  auto load_x8 = [&](size_t unit) -> uint4 {
    const uint16_t* s = gx16 + unit * 8;
    uint4 v;
    v.x = (uint32_t)s[0] | ((uint32_t)s[1] << 16);
    v.y = (uint32_t)s[2] | ((uint32_t)s[3] << 16);
    v.z = (uint32_t)s[4] | ((uint32_t)s[5] << 16);
    v.w = (uint32_t)s[6] | ((uint32_t)s[7] << 16);
    return v;
  };
  const uint32_t mask = (1u << p.nbits) - 1u;

  for (int row = blockIdx.x * kWarps + warp; row < p.out_features; row += gridDim.x * kWarps) {
    float acc[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = 0.f;
    for (int j = lane; j < p.in_groups; j += 32) {
      float wf[UPG][8];
      const size_t cbase = ((size_t)row * p.in_groups + j) * K;
      for (int k = 0; k < K; ++k) {
        uint32_t code;
        if constexpr (CODE_BYTES == 2) code = reinterpret_cast<const uint16_t*>(p.codes)[cbase + k];
        else code = reinterpret_cast<const uint8_t*>(p.codes)[cbase + k];
        code &= mask;
        const size_t off = (((size_t)k << p.nbits) + code) * UPG;
#pragma unroll
        for (int h = 0; h < UPG; ++h) {
          const uint4 v = ld_gather_v4<0>(gcb + off + h);
          if (k == 0) unpack8<T>(v, wf[h]);
          else accum8<T>(v, wf[h]);
        }
      }
#pragma unroll
      for (int h = 0; h < UPG; ++h) {
#pragma unroll
        for (int b = 0; b < BT; ++b)
          if (b < p.batch) acc[b] = dot8f<T>(wf[h], load_x8((size_t)b * upr + j * UPG + h), acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = warp_sum(acc[b]);
    if (lane == 0) {
      if (p.partial_f32) {
        float* y = reinterpret_cast<float*>(p.y);
#pragma unroll
        for (int b = 0; b < BT; ++b)
          if (b < p.batch) y[(size_t)b * p.out_features + row] = acc[b];
      } else {
        const float s = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
        const float bv = p.bias ? DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]) : 0.f;
        T* y = reinterpret_cast<T*>(p.y);
#pragma unroll
        for (int b = 0; b < BT; ++b)
          if (b < p.batch) y[(size_t)b * p.out_features + row] = DT<T>::from_float(fmaf(acc[b], s, bv));
      }
    }
  }
}

// Epilogue of the sharded path (after the all-reduce of fp32 partials).
template <typename T>
__global__ void scale_bias_kernel(const float* __restrict__ partial, const T* __restrict__ scales,
                                  const T* __restrict__ bias, T* __restrict__ out, int64_t batch, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * n) return;
  const int64_t o = i % n;
  const float s = DT<T>::to_float(scales[o]);
  const float b = bias ? DT<T>::to_float(bias[o]) : 0.f;
  out[i] = DT<T>::from_float(fmaf(partial[i], s, b));
}

}  // namespace aqlm_b200
