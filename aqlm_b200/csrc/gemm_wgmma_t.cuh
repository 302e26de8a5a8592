// Fused additive-dequant + TRANSPOSED tensor-core GEMM (the backward w.r.t. the input):
//     grad_in[bs, in] = (grad_out[bs, out] * scales[out]) . W[out, in]          W never touches HBM.
//
// Replaces code{1x16,2x8,1x8}_matmat_dequant_transposed (reference cuda_kernel.cpp:303-354, 486-519, 651-684), which
// materialise W [out,in] in HBM with a Dequant kernel and call cuBLAS on (grad_out * scales); the reference's 2x8/1x8
// variants forget the scaled input (cuda_kernel.cpp:497,518,662,683) -- not reproduced.
//
// Same wgmma / TMA skeleton and warp roles as gemm_wgmma.cuh with the contraction running over OUT rows:
//   D[128 in-features x N batch] (fp32, registers)  +=  A[128 x 64] . B[N x 64]^T        per k-block of 64 out rows
//   A = W^T tile, produced on chip.  A gathered codebook vector is 8 CONSECUTIVE in-features of ONE out row, i.e. 16
//       contiguous bytes along M: the A stage is therefore kept MN-MAJOR (canonical SWIZZLE_128B MN-major layout,
//       64 x 8 element atoms, wgmma transpose-A), so a gather still lands with ONE 16-byte store;
//       the per-row scale is applied to the vector before it is written (fp32 multiply, one rounding);
//   B = grad_out tile [N x 64 out columns], K-major, TMA-loaded with 128B swizzle (OOB rows/columns zero-filled);
//   code tiles: TMA boxes of 256 out rows x (16 groups * K codes) bytes, un-swizzled.
// Grid = (in/128 tiles, K splits over the out rows, N tiles); split partials and the deterministic last-CTA fix-up are
// the forward kernel's.
#pragma once

#include "gemm_wgmma.cuh"

namespace aqlm_b200 {

constexpr int kGemmTCtileRows = 256;  // out rows per code tile (= 4 k-blocks)

struct GemmTParams {
  const void* codebooks;
  const void* scales;         // [out]
  void* y;                    // grad_in [batch, in_features]
  float* ws_partials;
  unsigned int* ws_counters;
  int in_features;
  int out_features;
  int batch;
  int nbits;
  int total_kblocks;          // ceil(out / 64)
  int ksplit;
  int stages;
  int gather_mode;
};

struct GemmTSmem {
  uint32_t a, b, codes, full, empty, cfull, cempty, flag;
  size_t total;
};
__host__ __device__ inline GemmTSmem gemm_t_smem_layout(int stages, int n_tile, int ctile_row_bytes) {
  GemmTSmem L;
  size_t off = 0;
  L.a = (uint32_t)off; off += (size_t)stages * kGemmBlockM * 128;
  L.b = (uint32_t)off; off += (size_t)stages * n_tile * 128;
  off = (off + 1023) & ~(size_t)1023;
  L.codes = (uint32_t)off; off += (size_t)kCodeTileStages * kGemmTCtileRows * ctile_row_bytes;
  off = (off + 15) & ~(size_t)15;
  L.full = (uint32_t)off; off += 8 * 8;
  L.empty = (uint32_t)off; off += 8 * 8;
  L.cfull = (uint32_t)off; off += 8 * kCodeTileStages;
  L.cempty = (uint32_t)off; off += 8 * kCodeTileStages;
  L.flag = (uint32_t)off; off += 4;
  L.total = off + 1024;
  return L;
}

template <typename T, int K, int CODE_BYTES, int N>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_dequant_t_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_codes, const GemmTParams p) {
  constexpr int GBT = 16 * K * CODE_BYTES;  // code bytes per out row per tile (16 groups = 128 in-features)
  constexpr int CB4 = 4 * K * CODE_BYTES;   // code bytes of one thread's 4 adjacent groups
  constexpr int CW = (CB4 + 3) / 4;
  constexpr bool INREG = K <= 2;
  constexpr int KR = INREG ? K : 1;
  constexpr int D = (K == 1) ? 2 : 1;       // k-blocks of gathers held in registers ahead of the writes
  constexpr int KB_PER_CTILE = kGemmTCtileRows / kGemmBlockK;
  extern __shared__ uint8_t smem_dyn[];
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* gbase = smem_dyn + (base - smem_u32(smem_dyn));
  const GemmTSmem L = gemm_t_smem_layout(p.stages, N, GBT);
  const int S = p.stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, split = blockIdx.y, n_blk = blockIdx.z;
  const int m0 = m_tile * kGemmBlockM, n0 = n_blk * N;
  const int kb0 = (int)(((long long)p.total_kblocks * split) / p.ksplit);
  const int kb1 = (int)(((long long)p.total_kblocks * (split + 1)) / p.ksplit);
  const int nkb = kb1 - kb0;
  const int ct0 = kb0 / KB_PER_CTILE, ct1 = (kb1 + KB_PER_CTILE - 1) / KB_PER_CTILE;
  griddep_launch_dependents();  // PDL, as in the forward kernel: weights before griddep_wait(), grad_out / outputs after

  auto full_bar = [&](int s) { return base + L.full + 8 * s; };
  auto empty_bar = [&](int s) { return base + L.empty + 8 * s; };
  auto cfull_bar = [&](int s) { return base + L.cfull + 8 * s; };
  auto cempty_bar = [&](int s) { return base + L.cempty + 8 * s; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), kGemmProducerWarps + 1);
      mbar_init(empty_bar(s), kGemmConsumerWarps);
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
    // ===== consumers: warpgroup wg owns in-features [64 wg, 64 wg + 64) of the tile = MN atom wg of every K atom =====
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
      // atoms are laid out [k_atom (8)][m_atom (2)][1024 B]: LBO (next MN atom) 1024 B, SBO (next K atom) 2048 B
      const uint64_t ad = wgmma_desc(base + L.a + s * kGemmBlockM * 128 + wg * 1024, 1024, 2048);
      const uint64_t bd = wgmma_desc(base + L.b + s * N * 128, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kGemmBlockK / 16; ++k)  // 16 out rows = 2 K atoms: A advances 4096 bytes (+256), B 32 bytes (+2)
        wgmma_tile<T, N, 1>(acc, ad + (uint64_t)(256 * k), bd + (uint64_t)(2 * k));
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
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(prev));
    }
    griddep_wait();  // before any global write
    float* my_part = p.ws_partials ? p.ws_partials + ((tile_id * p.ksplit + split) * (size_t)N) * kGemmBlockM : nullptr;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row_in_tile = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * j;
      const int col = m0 + row_in_tile;  // in-feature index
      const bool col_ok = col < p.in_features;
#pragma unroll
      for (int i = 0; i < N / 8; ++i) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int n = 8 * i + 2 * (lane & 3) + c;
          const float v = acc[4 * i + 2 * j + c];
          if (p.ksplit == 1) {
            if (col_ok && n0 + n < p.batch) y[(size_t)(n0 + n) * p.in_features + col] = DT<T>::from_float(v);
          } else {
            my_part[(size_t)n * kGemmBlockM + row_in_tile] = v;
          }
        }
      }
    }
  } else if (warp == kGemmTmaWarp) {
    if (nkb > 0) {
      // ===== TMA producer (whole warp, one elected lane issues): code tiles (256 out rows x GBT bytes) and one grad_out
      //       tile per k-block =====
      int ct_loaded = ct0;
      auto load_ctile = [&](int ct) {
        const int cs = (ct - ct0) % kCodeTileStages, it = (ct - ct0) / kCodeTileStages;
        if (it > 0) mbar_wait(cempty_bar(cs), (it - 1) & 1);
        if (elect_one()) {
          mbar_expect_tx(cfull_bar(cs), kGemmTCtileRows * GBT);
          tma_load_2d(base + L.codes + cs * kGemmTCtileRows * GBT, &tmap_codes, m_tile * GBT, ct * kGemmTCtileRows, cfull_bar(cs));
        }
        __syncwarp();
      };
      load_ctile(ct_loaded++);
      griddep_wait();  // grad_out is produced by the previous kernel
      int s = 0, it = 0;
      for (int i = 0; i < nkb; ++i) {
        if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
        if (elect_one()) {
          mbar_expect_tx(full_bar(s), (uint32_t)N * 128);
          tma_load_2d(base + L.b + s * N * 128, &tmap_g, (kb0 + i) * kGemmBlockK, n0, full_bar(s));
        }
        __syncwarp();
        const int ct_cur = (kb0 + i) / KB_PER_CTILE;
        if (ct_loaded < ct1 && ct_loaded <= ct_cur + 1) load_ctile(ct_loaded++);
        if (++s == S) { s = 0; ++it; }
      }
    }
  } else if (nkb > 0) {
    // ===== dequant producers: 256 threads, thread -> (out row kk of the k-block, 4 adjacent in-groups) =====
    const int pt = threadIdx.x - kGemmProducer0;
    const int kk = pt >> 2, gq = pt & 3;  // kk: 0..63, gq: groups 4gq .. 4gq+3 (of 16)
    const uint4* gcb = reinterpret_cast<const uint4*>(p.codebooks);
    const T* gsc = reinterpret_cast<const T*>(p.scales);
    auto gather = [&](const uint4* gp) -> uint4 {
      return p.gather_mode == 1 ? ld_gather_v4<1>(gp) : ld_gather_v4<0>(gp);
    };

    auto issue = [&](int i, uint4 (&wv)[4][KR], float& sc) {
      const int kb = kb0 + i;
      const int ct = kb / KB_PER_CTILE, st_in = kb % KB_PER_CTILE;
      const int cs = (ct - ct0) % kCodeTileStages, cit = (ct - ct0) / kCodeTileStages;
      const int o = kb * kGemmBlockK + kk;
      sc = o < p.out_features ? DT<T>::to_float(gsc[o]) : 0.f;  // rows past the end contribute nothing
      mbar_wait(cfull_bar(cs), cit & 1);
      const uint8_t* src = gbase + L.codes + cs * kGemmTCtileRows * GBT + (st_in * kGemmBlockK + kk) * GBT + gq * CB4;
      uint32_t cw[CW];
      if constexpr (CB4 >= 16) {
#pragma unroll
        for (int q = 0; q < CB4 / 16; ++q) {
          const uint4 v = reinterpret_cast<const uint4*>(src)[q];
          cw[4 * q + 0] = v.x; cw[4 * q + 1] = v.y; cw[4 * q + 2] = v.z; cw[4 * q + 3] = v.w;
        }
      } else if constexpr (CB4 == 8) {
        const uint2 v = *reinterpret_cast<const uint2*>(src);
        cw[0] = v.x; cw[1] = v.y;
      } else {
        cw[0] = *reinterpret_cast<const uint32_t*>(src);
      }
      auto code_at = [&](int idx) -> uint32_t {
        if constexpr (CODE_BYTES == 2) return (cw[idx >> 1] >> ((idx & 1) * 16)) & 0xffffu;
        else return (cw[idx >> 2] >> ((idx & 3) * 8)) & 0xffu;
      };
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if constexpr (INREG) {
#pragma unroll
          for (int k = 0; k < K; ++k) wv[e][k] = gather(gcb + (((size_t)k << p.nbits) + code_at(e * K + k)));
        } else {
          float f[8];
          unpack8<T>(gather(gcb + code_at(e * K)), f);
#pragma unroll
          for (int k = 1; k < K; ++k) accum8<T>(gather(gcb + (((size_t)k << p.nbits) + code_at(e * K + k))), f);
          wv[e][0].x = DT<T>::pack2(f[0], f[1]); wv[e][0].y = DT<T>::pack2(f[2], f[3]);
          wv[e][0].z = DT<T>::pack2(f[4], f[5]); wv[e][0].w = DT<T>::pack2(f[6], f[7]);
        }
      }
      if (st_in == KB_PER_CTILE - 1 || i == nkb - 1) {  // after the gathers were issued: the code reads have completed
        __syncwarp();
        if (lane == 0) mbar_arrive(cempty_bar(cs));
      }
    };
    int st_next = 0, it_next = 0;  // commit() runs for k-blocks 0, 1, 2, ... in order: stage / use count without division
    auto commit = [&](uint4 (&wv)[4][KR], float sc) {
      const int s = st_next, it = it_next;
      if (++st_next == S) { st_next = 0; ++it_next; }
      if (it > 0) mbar_wait(empty_bar(s), (it - 1) & 1);
      // MN-major SWIZZLE_128B: atom (kk>>3, m_atom) at [(kk>>3)*2 + m_atom]*1024; inside an atom row kk&7 is 128 bytes of
      // 64 consecutive in-features, its 16-byte chunks XOR-swizzled with (kk&7)
      uint8_t* abase = gbase + L.a + s * kGemmBlockM * 128 + (kk >> 3) * 2048 + (kk & 7) * 128;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        uint4 v;
        if constexpr (K == 1) {
          // one codebook: scale the packed vector with 4 packed multiplies (a 16-bit x 16-bit product is exact in fp32, so
          // the packed multiply rounds exactly like fp32-multiply-then-round)
          v = wv[e][0];
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
        } else {
          float f[8];
          unpack8<T>(wv[e][0], f);
#pragma unroll
          for (int k = 1; k < KR; ++k) accum8<T>(wv[e][k], f);
#pragma unroll
          for (int q = 0; q < 8; ++q) f[q] *= sc;
          v.x = DT<T>::pack2(f[0], f[1]); v.y = DT<T>::pack2(f[2], f[3]);
          v.z = DT<T>::pack2(f[4], f[5]); v.w = DT<T>::pack2(f[6], f[7]);
        }
        const int j = gq * 4 + e;  // group 0..15 of the tile = 16-byte chunk j along M
        *reinterpret_cast<uint4*>(abase + (j >> 3) * 1024 + (((j & 7) ^ (kk & 7)) << 4)) = v;
      }
      fence_proxy_async();
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
    gemm_splitk_fixup<T>(reinterpret_cast<uint32_t*>(gbase + L.flag), p.ws_counters + tile_id,
                         p.ws_partials + (tile_id * p.ksplit) * (size_t)N * kGemmBlockM, p.ksplit, N,
                         min(N, p.batch - n0), y, p.in_features, n0, m0, min(kGemmBlockM, p.in_features - m0),
                         nullptr, nullptr);
  }
}

}  // namespace aqlm_b200
