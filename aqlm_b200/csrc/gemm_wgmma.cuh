// Fused additive-dequant + tensor-core GEMM for batch > 6:  Y[bs, out] = X[bs, in] . W^T, W never touches HBM.
//
// Replaces code{1x16,2x8,1x8}_matmat_dequant (reference cuda_kernel.cpp:249-301, 450-484, 615-649), which
// materialise W [out,in] in HBM with a Dequant kernel (cuda_kernel.cu:98-142) and then call cuBLAS.
//
// H100 design (wgmma / TMA / mbarrier, hand-written PTX in gemm_wgmma_ptx.cuh):
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
//
// This file holds the pipeline itself (gemm_pipeline: shared-memory layout, barrier protocol, the three warp roles,
// epilogue, split-K fix-up), written once for this kernel and for the transposed one of gemm_wgmma_t.cuh, and the
// forward direction: GemmForward and gemm_dequant_kernel.  What a direction is, is listed at GemmForward.
//
// Grouped calls (q/k/v, gate/up: linears that read the same input): the weights are concatenated along the out rows
// and GemmParams::n_seg / seg_end name the segments, each with its own stacked codebooks; one launch covers the group.
//
// Routed calls (mixture-of-experts: E experts of one shape, each applied to its own run of the input rows, which are
// sorted by expert): one launch covers every expert.  The grid's third index is a slot, not a batch tile; a CTA
// resolves it to (expert, first row, end row) from the device-side expert offsets (routing.cuh) and offsets its code
// tiles, codebooks, scales and bias by the expert.  PDL: the offsets are written by the previous kernel, so a routed
// CTA waits for it (griddep_wait) before it knows its expert, and its weight-side prologue (code tiles, gathers) no
// longer overlaps the previous kernel's tail as the plain and grouped kernels' does.
#pragma once

#include <type_traits>

#include "gemm_wgmma_ptx.cuh"
#include "routing.cuh"

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
constexpr int kCodeTileBytes = 128;      // forward: bytes of codes per row per code tile (TMA box inner extent)
constexpr int kCodeTileStages = 2;

// Parameters of both directions.  The GEMM is D[m_size x batch] = A[m_size x K] . B[batch x K]^T stored as y[batch][m_size]:
// forward m_size = out_features and K = in_features, transposed m_size = in_features and K = out_features.
struct GemmParams {
  const void* codebooks;
  const void* scales;   // [out_features]; forward: null with partial_f32
  const void* bias;     // forward only, may be null
  void* y;              // [batch, m_size]
  float* ws_partials;   // [m_tiles][n_tiles][ksplit][N][128] fp32 (ksplit > 1)
  unsigned int* ws_counters;  // [m_tiles * n_tiles], zero on entry
  int m_size;
  int batch;
  int nbits;
  int total_kblocks;    // ceil(K / 64)
  int ksplit;
  int stages;
  int tile_m;           // forward only: output rows per CTA tile (<= 128): ragged tile heights balance the grid
  int gather_mode;      // 0: ld.global.nc (L1 allocate), 1: ld.global.cg
  int partial_f32;      // forward only.  1: y is fp32 and gets the UNSCALED sums (no scale, no bias)
  int k_size;           // transposed only (scales of rows past it count as 0)
  // grouped call (several linears sharing the input, out rows concatenated), as GemvParams: segment i covers out rows
  // [seg_end[i-1], seg_end[i]) and its codebooks start at codebooks + i * (K << nbits) * 8 elements.  n_seg == 1: a
  // plain linear.  scales / bias are concatenated like the rows, so the epilogue needs nothing per segment.
  int n_seg;
  int seg_end[4];
  // routed call: expert e covers input / output rows [expert_off[e], expert_off[e+1]) (clamped, see routing.cuh) and
  // owns out rows [e * out, (e + 1) * out) of the stacked codes, scales and bias and codebook sets [e * n_seg, (e + 1) *
  // n_seg).  batch is the total row count.  Unused by plain and grouped calls.
  const int* expert_off;
  int n_experts;
};

// Where the codebooks of the segment that owns out row `row` start, in 16-byte vectors from p.codebooks (rows past the
// last segment end take the last segment's; seg_end[i] for i >= n_seg - 1 is the row count).  Branch-free on purpose:
// the loop form `i < n_seg - 1 && row >= seg_end[i]` made ptxas keep GemmParams in local memory and spill.
template <int K>
__device__ __forceinline__ uint32_t gemm_segment_cb_offset(const GemmParams& p, int row) {
  const uint32_t seg = (uint32_t)(row >= p.seg_end[0]) + (uint32_t)(row >= p.seg_end[1]) + (uint32_t)(row >= p.seg_end[2]);
  return (min(seg, (uint32_t)p.n_seg - 1u) * K) << p.nbits;
}

// shared-memory carve-up (all offsets from a 1024-byte aligned base); ctile_bytes: one code-tile stage, a multiple of 16
struct GemmSmem {
  uint32_t a, b, codes, full, empty, cfull, cempty, flag;
  size_t total;
};
__host__ __device__ inline GemmSmem gemm_smem_layout(int stages, int n_tile, int ctile_bytes) {
  GemmSmem L;
  size_t off = 0;
  L.a = (uint32_t)off; off += (size_t)stages * kGemmBlockM * 128;
  L.b = (uint32_t)off; off += (size_t)stages * n_tile * 128;
  off = (off + 1023) & ~(size_t)1023;
  L.codes = (uint32_t)off; off += (size_t)kCodeTileStages * ctile_bytes;
  L.full = (uint32_t)off; off += 8 * 8;
  L.empty = (uint32_t)off; off += 8 * 8;
  L.cfull = (uint32_t)off; off += 8 * kCodeTileStages;
  L.cempty = (uint32_t)off; off += 8 * kCodeTileStages;
  L.flag = (uint32_t)off; off += 4;
  L.total = off + 1024;  // slack for manual 1024-byte alignment of the dynamic smem base
  return L;
}

// The LoRA term of one tile (LoraArgs), staged in fp32 in the pipeline's shared memory once the main loop has drained
// it (stage buffers and code tiles: everything below the barriers, which the plan always has room for,
// gemm_lora_smem_bytes): ws = the weight side w(m, j) of the tile's 128 rows, us = lin of its N batch rows, each row
// ld = rank + 4 floats apart (an odd number of 16-byte chunks: float4 reads of 8 consecutive rows are conflict-free).
// Rows past the tile's end are staged as zeros.
__host__ __device__ inline size_t gemm_lora_smem_bytes(int rank, int n_tile) {
  return (size_t)(kGemmBlockM + n_tile) * (rank + 4) * 4;
}

struct GemmLoraTile {
  LoraArgs a;
  float* ws;
  float* us;
  int ld;

  // Every thread tid < nthreads of the caller's group takes part; the caller synchronises the group afterwards.
  // Forward: w(m, j) = B[m0 + m][j], rows of B.  Transposed: w(m, j) = A[j][m0 + m], columns of A (m_size = in, a
  // multiple of 8, so 4 consecutive columns are one aligned load).  us: lin rows n0 .. n0 + n_tile - 1.
  template <typename T, bool TRANSPOSED>
  __device__ __forceinline__ void stage(int m0, int rows, int m_size, int n0, int ncols, int n_tile, int tid,
                                        int nthreads) const {
    const int q4 = a.rank >> 2;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (TRANSPOSED) {
      for (int i = tid; i < a.rank * (kGemmBlockM / 4); i += nthreads) {
        const int j = i / (kGemmBlockM / 4), m = 4 * (i % (kGemmBlockM / 4));
        const float4 v = m < rows ? lora_load4<T>(a.w, (size_t)j * m_size + m0 + m, a.f32) : zero;
        ws[(m + 0) * ld + j] = v.x;
        ws[(m + 1) * ld + j] = v.y;
        ws[(m + 2) * ld + j] = v.z;
        ws[(m + 3) * ld + j] = v.w;
      }
    } else {
      for (int i = tid; i < kGemmBlockM * q4; i += nthreads) {
        const int m = i / q4, q = i % q4;
        *reinterpret_cast<float4*>(ws + m * ld + 4 * q) =
            m < rows ? lora_load4<T>(a.w, (size_t)(m0 + m) * a.rank + 4 * q, a.f32) : zero;
      }
    }
    for (int i = tid; i < n_tile * q4; i += nthreads) {
      const int c = i / q4, q = i % q4;
      *reinterpret_cast<float4*>(us + c * ld + 4 * q) =
          c < ncols ? lora_load4<T>(a.lin, (size_t)(n0 + c) * a.rank + 4 * q, a.f32) : zero;
    }
  }

  // scaling * L for tile row m and the 4 columns c0 + u * step (columns past the staged ones read the last staged one;
  // the caller discards them)
  __device__ __forceinline__ void cols4(int m, int c0, int step, int ncols, float (&out)[4]) const {
    float l[4] = {0.f, 0.f, 0.f, 0.f};
    const float* w = ws + m * ld;
    const float* u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = us + min(c0 + k * step, ncols - 1) * ld;
    for (int q = 0; q < a.rank; q += 4) {
      const float4 wv = *reinterpret_cast<const float4*>(w + q);
#pragma unroll
      for (int k = 0; k < 4; ++k) l[k] = dot4(wv, *reinterpret_cast<const float4*>(u[k] + q), l[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) out[k] = __fmul_rn(a.scaling, l[k]);
  }
};

// Split-K fix-up shared by both GEMM kernels: the LAST-arriving split of a tile adds all partials in split order
// (deterministic) with the whole CTA; partials are [split][column][128 rows].  Writes y[n * ld + row0 + r] =
// v * scale[row] + bias[row] (scales == nullptr: no scale / bias); an fp32 output (OutT = float) gets the sum v itself.
// LORA: the last CTA stages the tile's LoRA term (lt, direction TRANSPOSED) and adds it before the rounding.
template <typename T, typename OutT = T, bool LORA = false, bool TRANSPOSED = false>
__device__ __forceinline__ void gemm_splitk_fixup(uint32_t* flag, unsigned int* counter, const float* parts, int ksplit, int N,
                                                  int ncols, OutT* y, long long ld, int n0, int row0, int rows,
                                                  const T* scales, const T* bias, const GemmLoraTile* lt = nullptr) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int old = atomicAdd(counter, 1u);
    const bool last = (old == (unsigned int)ksplit - 1);
    *flag = last ? 1u : 0u;
    if (last) *counter = 0u;  // leave the counter clean for the next call
  }
  __syncthreads();
  if constexpr (LORA) {
    if (*flag) lt->stage<T, TRANSPOSED>(row0, rows, (int)ld, n0, ncols, N, threadIdx.x, kGemmThreads);
    __syncthreads();
  }
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
float l[4];
        if constexpr (LORA) lt->cols4(rrow, c, kPhases, ncols, l);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int cc = c + u * kPhases;
          if (cc >= ncols) continue;
          if constexpr (std::is_same<OutT, float>::value) y[(size_t)(n0 + cc) * ld + row] = v[u];
          else if constexpr (LORA) y[(size_t)(n0 + cc) * ld + row] = DT<T>::from_float(__fadd_rn(fmaf(v[u], sc, bi), l[u]));
          else y[(size_t)(n0 + cc) * ld + row] = DT<T>::from_float(fmaf(v[u], sc, bi));
        }
      }
    }
  }
}

// The forward direction.  A direction is a compile-time description of everything the two GEMMs differ in: the A
// operand's layout (descriptor on the consumer side, chunk addresses on the producer side), the code tile (TMA box,
// where a producer thread finds its codes), the producer's thread mapping (and the out row, hence the segment of a
// grouped call, whose codes it dequantizes), and where the row scale is applied.
// K = codebooks per group, CODE_BYTES = 1|2; in_group_size == 8.
template <int K_, int CODE_BYTES_>
struct GemmForward {
  static constexpr int K = K_, CODE_BYTES = CODE_BYTES_;
  static constexpr int CB4 = 4 * K * CODE_BYTES;  // code bytes of one producer thread's 4 groups
  static constexpr int GB = 2 * CB4;              // code bytes per row per k-block
  static_assert(GB <= kCodeTileBytes, "scheme too wide for the code tile");

  // A stage: K-major, row r of the tile = 128 bytes of 64 in-features, 16-byte chunks XOR-swizzled with r & 7;
  // warpgroup wg reads rows [64 wg, 64 wg + 64)
  static constexpr int TA = 0;
  static constexpr uint32_t kALbo = 16, kASbo = 1024;
  static constexpr uint32_t kAStepK = 2;  // 16 K-elements = 32 bytes = +2 in the descriptor's address field
  static constexpr uint32_t kAWarpgroup = 64 * 128;

  // Scale (and bias) are applied to the sums in the epilogue / the split-K fix-up; tiles may be ragged (tile_m < 128).
  static constexpr bool kScaleInProducer = false;
  static constexpr bool kTransposed = false;
  static __device__ __forceinline__ int tile_m(const GemmParams& p) { return p.tile_m; }
  // out rows of one expert of a routed call (the forward's output rows)
  static __device__ __forceinline__ int out_rows(const GemmParams& p) { return p.m_size; }

  // code tile: tile_m rows x 128 bytes of codes, SWIZZLE_128B; covers kKbPerCtile k-blocks
  static constexpr int kCtileBytes = kGemmBlockM * kCodeTileBytes;
  static constexpr int kKbPerCtile = kCodeTileBytes / GB;
  static __device__ __forceinline__ uint32_t ctile_tx_bytes(int tile_m) { return (uint32_t)tile_m * kCodeTileBytes; }
  static __device__ __forceinline__ int2 ctile_coord(int m_tile, int tile_m, int ct) {
    return make_int2(ct * kCodeTileBytes, m_tile * tile_m);
  }

  // producer thread pt -> (row pt / 2 of the tile, half pt % 2 of the 8 groups of a k-block)
  // rows past the (ragged) tile height: no gathers, nothing to write
  static __device__ __forceinline__ bool active(int pt, int tile_m) { return (pt >> 1) < tile_m; }
  // the out row whose codes the thread dequantizes: the same tile row for every k-block, so a grouped call resolves
  // its segment's codebooks once, before the k loop (a ragged tile may straddle a segment end: per row, not per tile)
  static constexpr bool kRowPerKblock = false;
  static __device__ __forceinline__ int out_row(int pt, int m0, int) { return m0 + (pt >> 1); }
  // byte 16 q of the thread's CB4 code bytes for k-block st_in of the staged tile: logical offset inside the 128-byte
  // code row -> physical (SWIZZLE_128B: 16-byte chunk ^= row & 7)
  static __device__ __forceinline__ int code_offset(int pt, int st_in, int q) {
    const int row = pt >> 1, lbyte = st_in * GB + (pt & 1) * CB4 + 16 * q;
    return row * 128 + (((lbyte >> 4) ^ (row & 7)) << 4) + (lbyte & 15);
  }
  // group e of the thread's 4 = 16-byte chunk half * 4 + e inside the 128-byte K row
  static __device__ __forceinline__ int a_chunk_offset(int pt, int e) {
    const int row = pt >> 1, j = (pt & 1) * 4 + e;
    return row * 128 + ((j ^ (row & 7)) << 4);
  }
};

// The pipeline of both GEMM kernels; Dir is GemmForward or GemmTransposed, N the MMA width (columns of the batch tile).
// tmap_b loads the K-major B operand (activations / grad_output), tmap_codes the code tiles.  GROUPED: the kernel of
// grouped calls (GemmParams::n_seg / seg_end); plain linears run kernels without any segment arithmetic.  ROUTED (with
// GROUPED): the kernel of routed calls (GemmParams::expert_off / n_experts); see the file comment.  LORA (plain linears
// only): the epilogue and the split-K fix-up add the LoRA term of `lora` (see LoraArgs) to every output element before
// its rounding, staged over the drained pipeline (GemmLoraTile).
template <typename T, int N, typename Dir, bool GROUPED = false, bool ROUTED = false, bool LORA = false>
__device__ __forceinline__ void gemm_pipeline(const CUtensorMap& tmap_b, const CUtensorMap& tmap_codes, const GemmParams& p,
                                              const LoraArgs& lora = LoraArgs{}) {
  static_assert(!ROUTED || GROUPED, "a routed kernel resolves segments too");
  static_assert(!LORA || !GROUPED, "an adapter belongs to one plain linear");
  constexpr int K = Dir::K, CODE_BYTES = Dir::CODE_BYTES, CB4 = Dir::CB4;
  constexpr int KB_PER_CTILE = Dir::kKbPerCtile;  // k-blocks covered by one code tile
  static_assert(KB_PER_CTILE >= 1, "scheme too wide for the code tile");
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* gbase = smem_dyn + (base - smem_u32(smem_dyn));
  const GemmSmem L = gemm_smem_layout(p.stages, N, Dir::kCtileBytes);
  const int S = p.stages;
  const int TM = Dir::tile_m(p);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, split = blockIdx.y, n_blk = blockIdx.z;
  const int m0 = m_tile * TM;
  // PDL: the next kernel of the stream may be dispatched as soon as SM resources free up (no launch gap).  Everything this
  // kernel does before griddep_wait() touches WEIGHTS only (code tiles, codebook gathers, scales); the B tiles are read
  // and y / the workspace written after it.
  griddep_launch_dependents();
  // Columns of the tile: batch rows [n0, n0 + N), valid below n_end().  A routed CTA takes them, and its expert, from
  // its slot; the expert's weights start e_rows out rows (and e_cb codebook vectors) into the stacks.  Plain and grouped
  // kernels read p.batch where they always did (a local copy of it changed their register allocation).
  RoutedSlot rs{0, 0, 0};
  size_t e_rows = 0;
  uint32_t e_cb = 0;
  if constexpr (ROUTED) {
    griddep_wait();  // the offsets are the previous kernel's output
    rs = routed_slot(p.expert_off, p.n_experts, p.batch, N, n_blk);
    if (rs.expert < 0) return;  // past the last tile: no barrier, no workspace touched
    e_rows = (size_t)rs.expert * Dir::out_rows(p);
    e_cb = ((uint32_t)rs.expert * (uint32_t)p.n_seg * K) << p.nbits;
  }
  const int n0 = ROUTED ? rs.row0 : n_blk * N;
  auto n_end = [&]() { return ROUTED ? rs.row1 : p.batch; };
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
      const uint64_t ad = wgmma_desc(base + L.a + s * kGemmBlockM * 128 + wg * Dir::kAWarpgroup, Dir::kALbo, Dir::kASbo);
      const uint64_t bd = wgmma_desc(base + L.b + s * N * 128, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kGemmBlockK / 16; ++k)  // B: 16 K-elements = 32 bytes = +2 in the descriptor's address field
        wgmma_tile<T, N, Dir::TA>(acc, ad + (uint64_t)(Dir::kAStepK * k), bd + (uint64_t)(2 * k));
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
    if constexpr (LORA) {
      if (p.ksplit == 1) {
        // both warpgroups' MMAs have completed, so every stage is drained: stage the tile's LoRA term over them
        constexpr int kConsumerThreads = kGemmConsumerWarps * 32;
        const int ld = lora.rank + 4;
        const GemmLoraTile lt{lora, reinterpret_cast<float*>(gbase + L.a), reinterpret_cast<float*>(gbase + L.a) + kGemmBlockM * ld, ld};
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        lt.stage<T, Dir::kTransposed>(m0, min(TM, p.m_size - m0), p.m_size, n0, min(N, n_end() - n0), N, threadIdx.x,
                                      kConsumerThreads);
        asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // the thread's tile rows: r0 and r0 + 8
        float sc[2] = {1.f, 1.f}, bi[2] = {0.f, 0.f};
        bool ok[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int row = m0 + r0 + 8 * j;
          ok[j] = r0 + 8 * j < TM && row < p.m_size;
          if (!Dir::kScaleInProducer && ok[j]) {
            sc[j] = DT<T>::to_float(reinterpret_cast<const T*>(p.scales)[row]);
            if (p.bias) bi[j] = DT<T>::to_float(reinterpret_cast<const T*>(p.bias)[row]);
          }
        }
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
          const int col0 = 8 * i + 2 * (lane & 3);
          const float* w0 = lt.ws + r0 * ld;
          const float* u0 = lt.us + col0 * ld;
          float l[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
          for (int q = 0; q < lora.rank; q += 4) {
            const float4 a0 = *reinterpret_cast<const float4*>(w0 + q), a1 = *reinterpret_cast<const float4*>(w0 + 8 * ld + q);
            const float4 b0 = *reinterpret_cast<const float4*>(u0 + q), b1 = *reinterpret_cast<const float4*>(u0 + ld + q);
            l[0][0] = dot4(a0, b0, l[0][0]);
            l[0][1] = dot4(a0, b1, l[0][1]);
            l[1][0] = dot4(a1, b0, l[1][0]);
            l[1][1] = dot4(a1, b1, l[1][1]);
          }
#pragma unroll
          for (int j = 0; j < 2; ++j) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              if (!ok[j] || n0 + col0 + c >= n_end()) continue;
              const float v = acc[4 * i + 2 * j + c], t = __fmul_rn(lora.scaling, l[j][c]);
              y[(size_t)(n0 + col0 + c) * p.m_size + m0 + r0 + 8 * j] =
                  DT<T>::from_float(Dir::kScaleInProducer ? __fadd_rn(v, t) : __fadd_rn(fmaf(v, sc[j], bi[j]), t));
            }
          }
        }
        return;  // without a split nothing follows the roles
      }
    }
    // accumulator fragment: register 4i + 2j + c holds (row 16 (warp % 4) + lane / 4 + 8 j, column 8 i + 2 (lane % 4) + c)
    float* my_part = p.ws_partials ? p.ws_partials + ((tile_id * p.ksplit + split) * (size_t)N) * kGemmBlockM : nullptr;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * j;
      const int row = m0 + row_in_tile;
      const bool row_ok = row_in_tile < TM && row < p.m_size;
      float sc = 1.f, bi = 0.f;
      if constexpr (!Dir::kScaleInProducer) {
        if (row_ok && p.ksplit == 1 && !p.partial_f32) {
          sc = DT<T>::to_float((reinterpret_cast<const T*>(p.scales) + e_rows)[row]);
          if (p.bias) bi = DT<T>::to_float((reinterpret_cast<const T*>(p.bias) + e_rows)[row]);
        }
      }
#pragma unroll
      for (int i = 0; i < N / 8; ++i) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int col = 8 * i + 2 * (lane & 3) + c;
          const float v = acc[4 * i + 2 * j + c];
          if (p.ksplit == 1) {
            if (row_ok && n0 + col < n_end()) {
              const size_t o = (size_t)(n0 + col) * p.m_size + row;
              if constexpr (Dir::kScaleInProducer) {
                y[o] = DT<T>::from_float(v);
              } else {
                if (p.partial_f32) reinterpret_cast<float*>(p.y)[o] = v;
                else y[o] = DT<T>::from_float(fmaf(v, sc, bi));
              }
            }
          } else {
            my_part[(size_t)col * kGemmBlockM + row_in_tile] = v;
          }
        }
      }
    }
  } else if (warp == kGemmTmaWarp) {
    if (nkb > 0) {
      // ===== TMA producer (whole warp, one elected lane issues): code tiles (one per KB_PER_CTILE k-blocks) and one B
      //       tile per k-block =====
      int ct_loaded = ct0;
      auto load_ctile = [&](int ct) {
        const int cs = (ct - ct0) % kCodeTileStages;
        const int it = (ct - ct0) / kCodeTileStages;
        if (it > 0) mbar_wait(cempty_bar(cs), (it - 1) & 1);  // every producer warp released the previous tenant
        if (elect_one()) {
          const int2 at = Dir::ctile_coord(m_tile, TM, ct);
          mbar_expect_tx(cfull_bar(cs), Dir::ctile_tx_bytes(TM));
          tma_load_2d(base + L.codes + cs * Dir::kCtileBytes, &tmap_codes, at.x, at.y + (int)e_rows, cfull_bar(cs));
        }
        __syncwarp();
      };
      load_ctile(ct_loaded++);
      griddep_wait();  // B is produced by the previous kernel
      int s = 0, it = 0;  // B stage and its use count (no runtime division in this loop)
      for (int i = 0; i < nkb; ++i) {
        if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
        if (elect_one()) {
          mbar_expect_tx(full_bar(s), (uint32_t)N * 128);
          tma_load_2d(base + L.b + s * N * 128, &tmap_b, (kb0 + i) * kGemmBlockK, n0, full_bar(s));
        }
        __syncwarp();
        // prefetch the NEXT code tile while the producers work on the current one
        const int ct_cur = (kb0 + i) / KB_PER_CTILE;
        if (ct_loaded < ct1 && ct_loaded <= ct_cur + 1) load_ctile(ct_loaded++);
        if (++s == S) { s = 0; ++it; }
      }
    }
  } else if (nkb > 0) {
    // ===== dequant producers: 256 threads, each dequantizes 4 groups (4 x 8 weights) per k-block =====
    // Software-pipelined for K <= 2: the gathers of the next D k-blocks are in flight while k-block i is written to smem
    // (the kernel is bound by gather latency unless several gathers per thread are outstanding).  K >= 4 gathers and
    // sums group by group (the 256-entry codebooks of those schemes are L1-resident).
    const int pt = threadIdx.x - kGemmProducer0;
    const bool active = Dir::active(pt, TM);
    const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);
    // codebooks of the segment that owns the thread's out row (grouped calls only)
    uint32_t cb_row = 0;
    if constexpr (GROUPED && !Dir::kRowPerKblock) cb_row = e_cb + gemm_segment_cb_offset<K>(p, Dir::out_row(pt, m0, 0));
    constexpr int CW = (CB4 + 3) / 4;        // 32-bit words holding the thread's CB4 code bytes
    constexpr bool INREG = K <= 2;           // hold the raw gathered vectors in registers until the write
    constexpr int KR = INREG ? K : 1;
    constexpr int D = (K == 1) ? 2 : 1;      // k-blocks of gathers held in registers ahead of the writes
    auto gather = [&](const uint4* gp) -> uint4 {
      return p.gather_mode == 1 ? ld_gather_v4<1>(gp) : ld_gather_v4<0>(gp);
    };

    // codes of k-block index i (relative) -> the 4 groups' gathers (K <= 2) or their dequantized sums (K >= 4), and the
    // row scale where the producer applies it
    auto issue = [&](int i, uint4 (&wv)[4][KR], float& sc) {
      const int kb = kb0 + i;
      const int ct = kb / KB_PER_CTILE, st_in = kb % KB_PER_CTILE;
      const int cs = (ct - ct0) % kCodeTileStages, cit = (ct - ct0) / kCodeTileStages;
      if constexpr (Dir::kScaleInProducer) sc = Dir::template row_scale<T>(p, pt, kb, e_rows);
      uint32_t cbo = cb_row;
      if constexpr (GROUPED && Dir::kRowPerKblock) cbo = e_cb + gemm_segment_cb_offset<K>(p, Dir::out_row(pt, m0, kb));
      // codebook k's vector `code` (a plain linear: the first and only codebook set)
      auto cb_vec = [&](int k, uint32_t code) -> const uint4* {
        if constexpr (GROUPED) return gcb + (cbo + ((uint32_t)k << p.nbits) + code);
        else return gcb + (((size_t)k << p.nbits) + code);
      };
      mbar_wait(cfull_bar(cs), cit & 1);
      uint32_t cw[CW];
      const uint8_t* ctile = gbase + L.codes + cs * Dir::kCtileBytes;
      if (!active) {
#pragma unroll
        for (int q = 0; q < CW; ++q) cw[q] = 0u;
      } else if constexpr (CB4 >= 16) {
#pragma unroll
        for (int q = 0; q < CB4 / 16; ++q) {
          const uint4 v = *reinterpret_cast<const uint4*>(ctile + Dir::code_offset(pt, st_in, q));
          cw[4 * q + 0] = v.x; cw[4 * q + 1] = v.y; cw[4 * q + 2] = v.z; cw[4 * q + 3] = v.w;
        }
      } else {
        const uint8_t* src = ctile + Dir::code_offset(pt, st_in, 0);
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
            wv[e][k] = active ? gather(cb_vec(k, code_at(e * K + k))) : make_uint4(0u, 0u, 0u, 0u);
        } else {
          float f[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) f[q] = 0.f;
          if (active) {
            unpack8<T>(gather(cb_vec(0, code_at(e * K))), f);
#pragma unroll
            for (int k = 1; k < K; ++k) accum8<T>(gather(cb_vec(k, code_at(e * K + k))), f);
          }
          // the transposed direction scales the fp32 sum here, so that it is rounded to T once
          if constexpr (Dir::kScaleInProducer) {
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] *= sc;
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
    int st_next = 0, it_next = 0;  // commit() runs for k-blocks 0, 1, 2, ... in order: stage / use count without division
    // additive dequant (+ row scale) + write the 4 groups of k-block i into the swizzled A stage, then signal the consumers
    auto commit = [&](uint4 (&wv)[4][KR], float sc) {
      const int s = st_next, it = it_next;
      if (++st_next == S) { st_next = 0; ++it_next; }
      if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
      uint8_t* astage = gbase + L.a + s * kGemmBlockM * 128;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        uint4 v = wv[e][0];
        if constexpr (!INREG) {
          // K >= 4: issue() wrote the finished vector (the fp32 sum, scaled in the transposed direction, rounded once)
        } else if constexpr (Dir::kScaleInProducer && K == 1) {
          // one codebook: scale the packed vector with 4 packed multiplies (the product of two fp16 or two bf16 values is
          // exact in fp32, so the packed multiply's one rounding gives what fp32-multiply-then-round-to-T gives)
          if constexpr (DT<T>::is_bf16) {
            const __nv_bfloat162 s2 = __float2bfloat162_rn(sc);
            __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
            for (int q = 0; q < 4; ++q) h[q] = __hmul2(h[q], s2);
          } else {
            const __half2 s2 = __float2half2_rn(sc);
            __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
            for (int q = 0; q < 4; ++q) h[q] = __hmul2(h[q], s2);
          }
        } else if constexpr (Dir::kScaleInProducer || K == 2) {
          float f[8];
          unpack8<T>(wv[e][0], f);
#pragma unroll
          for (int k = 1; k < KR; ++k) accum8<T>(wv[e][k], f);
          if constexpr (Dir::kScaleInProducer) {
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] *= sc;
          }
          v.x = DT<T>::pack2(f[0], f[1]); v.y = DT<T>::pack2(f[2], f[3]);
          v.z = DT<T>::pack2(f[4], f[5]); v.w = DT<T>::pack2(f[6], f[7]);
        }
        if (active) *reinterpret_cast<uint4*>(astage + Dir::a_chunk_offset(pt, e)) = v;
      }
      fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(full_bar(s));
    };
    uint4 w[D][4][KR];
    float scv[D];
#pragma unroll
    for (int d = 0; d < D; ++d)
      if (d < nkb) issue(d, w[d], scv[d]);
    for (int i = 0; i < nkb; i += D) {
#pragma unroll
      for (int d = 0; d < D; ++d) {
        if (i + d < nkb) {
          commit(w[d], scv[d]);
          if (i + d + D < nkb) issue(i + d + D, w[d], scv[d]);
        }
      }
    }
  }

  if (p.ksplit > 1) {
    griddep_wait();
    uint32_t* flag = reinterpret_cast<uint32_t*>(gbase + L.flag);
    const float* parts = p.ws_partials + (tile_id * p.ksplit) * (size_t)N * kGemmBlockM;
    const int ncols = min(N, n_end() - n0), rows = min(TM, p.m_size - m0);
    if constexpr (LORA) {
      const int ld = lora.rank + 4;
      const GemmLoraTile lt{lora, reinterpret_cast<float*>(gbase + L.a), reinterpret_cast<float*>(gbase + L.a) + kGemmBlockM * ld, ld};
      gemm_splitk_fixup<T, T, true, Dir::kTransposed>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, y, p.m_size,
                                                      n0, m0, rows, Dir::kScaleInProducer ? nullptr : reinterpret_cast<const T*>(p.scales),
                                                      Dir::kScaleInProducer ? nullptr : reinterpret_cast<const T*>(p.bias), &lt);
    } else if constexpr (Dir::kScaleInProducer) {
      gemm_splitk_fixup<T>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, y, p.m_size, n0, m0, rows, nullptr, nullptr);
    } else {
      if (p.partial_f32)
        gemm_splitk_fixup<T, float>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, reinterpret_cast<float*>(p.y),
                                    p.m_size, n0, m0, rows, nullptr, nullptr);
      else {
        const T* scales = reinterpret_cast<const T*>(p.scales);
        const T* bias = reinterpret_cast<const T*>(p.bias);
        if constexpr (ROUTED) {
          scales += e_rows;
          if (bias) bias += e_rows;
        }
        gemm_splitk_fixup<T>(flag, p.ws_counters + tile_id, parts, p.ksplit, N, ncols, y, p.m_size, n0, m0, rows, scales, bias);
      }
    }
  }
}

template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_codes, const GemmParams p) {
  gemm_pipeline<T, N, GemmForward<K, CODE_BYTES>>(tmap_x, tmap_codes, p);
}

// The same over the row-concatenated weights of a grouped call (q/k/v, gate/up: one launch for the group).
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_grouped_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_codes,
                            const GemmParams p) {
  gemm_pipeline<T, N, GemmForward<K, CODE_BYTES>, true>(tmap_x, tmap_codes, p);
}

// A plain linear with a LoRA adapter (LoraArgs, forward form): y = x W^T s + b + scaling (x A^T) B^T, one rounding.
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_lora_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_codes,
                         const GemmParams p, const LoraArgs lora) {
  gemm_pipeline<T, N, GemmForward<K, CODE_BYTES>, false, false, true>(tmap_x, tmap_codes, p, lora);
}

// A routed call: every expert of a mixture-of-experts projection in one launch, over expert-sorted input rows.
template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_routed_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_codes,
                           const GemmParams p) {
  gemm_pipeline<T, N, GemmForward<K, CODE_BYTES>, true, true>(tmap_x, tmap_codes, p);
}

}  // namespace aqlm_b200
