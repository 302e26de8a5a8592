// C-ABI of aqlm_b200 (see include/aqlm_b200.h): argument validation, kernel selection, launches.  The launch plans
// (GEMM tiles / splits / stages, LUT grids) are pure functions in plan.cuh.
// The host-side role of the reference's cuda_kernel.cpp (dtype check 9-25, group-size switch 113-146,
// launch heuristics cuda_kernel.cu:476-516) without torch types.
#include <cstring>
#include <mutex>
#include <type_traits>

#include "dequant.cuh"
#include "peer_allreduce.cuh"
#include "plan.cuh"

namespace aqlm_b200 {

std::atomic<uint64_t> g_launch_count{0};

const DeviceInfo* device_info() {
  static DeviceInfo infos[kMaxDevices];
  static std::mutex mu;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) {
    fail(AQLM_B200_ERR_CUDA, "cudaGetDevice failed (no CUDA device / driver?)");
    return nullptr;
  }
  DeviceInfo& d = infos[dev];
  if (!d.ok) {
    std::lock_guard<std::mutex> lock(mu);
    if (!d.ok) {
      cudaError_t e = cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
      if (e == cudaSuccess) e = cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
      if (e == cudaSuccess) e = cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
      if (e == cudaSuccess) e = cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
      if (e != cudaSuccess) {
        fail(AQLM_B200_ERR_CUDA, "cudaDeviceGetAttribute failed: %s", cudaGetErrorString(e));
        return nullptr;
      }
      d.index = dev;
      d.ok = true;
    }
  }
  if (d.cc_major != 9 || d.cc_minor != 0) {
    fail(AQLM_B200_ERR_ARCH, "aqlm_b200 is built for sm_90a only; device %d is sm_%d%d", dev, d.cc_major, d.cc_minor);
    return nullptr;
  }
  return &d;
}

// The current device's info in *di, or the status a C-ABI call returns without one: AQLM_B200_ERR_ARCH for a device
// that is not sm_90a, AQLM_B200_ERR_CUDA otherwise.
static int current_device(const DeviceInfo** di) {
  *di = device_info();
  if (*di) return AQLM_B200_OK;
  return strstr(tls_error_buf(), "sm_90a") ? AQLM_B200_ERR_ARCH : AQLM_B200_ERR_CUDA;
}

static Tunables& tun() {
  static Tunables t = [] { Tunables x; x.load(); return x; }();
  return t;
}

static int validate(const aqlm_b200_weight_t* w, bool need_scales) {
  if (!w) return fail(AQLM_B200_ERR_SHAPE, "weight descriptor is NULL");
  if (w->dtype != AQLM_B200_F16 && w->dtype != AQLM_B200_BF16)
    return fail(AQLM_B200_ERR_DTYPE,
                "AQLM CUDA kernels only support float16 and bfloat16. Please specify the correct `torch_dtype` "
                "when loading the model.");
  if (w->out_group_size != 1)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "aqlm_b200 kernels require out_group_size == 1, got %d", w->out_group_size);
  if (w->in_group_size != 8 && w->in_group_size != 16)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "AQLM CUDA kernels only support codebooks with 8 or 16 features. Got %d.",
                w->in_group_size);
  if (w->nbits_per_codebook < 1 || w->nbits_per_codebook > 16)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "nbits_per_codebook must be in [1,16], got %d", w->nbits_per_codebook);
  if (w->num_codebooks < 1 || w->num_codebooks > 16)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "num_codebooks must be in [1,16], got %d", w->num_codebooks);
  if (w->in_features <= 0 || w->out_features <= 0 || w->in_features % w->in_group_size != 0)
    return fail(AQLM_B200_ERR_SHAPE, "bad shape: in_features=%lld out_features=%lld in_group_size=%d",
                (long long)w->in_features, (long long)w->out_features, w->in_group_size);
  if (w->in_features > (1ll << 30) || w->out_features > (1ll << 30))
    return fail(AQLM_B200_ERR_SHAPE, "dimension too large");
  if (!w->codes || !w->codebooks) return fail(AQLM_B200_ERR_SHAPE, "codes/codebooks pointer is NULL");
  if (need_scales && !w->scales) return fail(AQLM_B200_ERR_SHAPE, "scales pointer is NULL");
  if ((reinterpret_cast<uintptr_t>(w->codebooks) & 15) != 0)
    return fail(AQLM_B200_ERR_SHAPE, "codebooks must be 16-byte aligned");
  return AQLM_B200_OK;
}

// ---- runtime values to template arguments: f is called with std::integral_constant / Type<T> tags -------------
template <int V>
using Int = std::integral_constant<int, V>;
template <typename T>
struct Type {
  using type = T;
};

template <typename F>
static int with_dtype(int dtype, F&& f) {
  return dtype == AQLM_B200_F16 ? f(Type<__half>{}) : f(Type<__nv_bfloat16>{});
}

// batch rows of one GEMV pass -> the batch tile compiled for them: 1, 2, 4 or 8
template <typename F>
static int with_batch_tile(int64_t rows, F&& f) {
  if (rows == 1) return f(Int<1>{});
  if (rows == 2) return f(Int<2>{});
  if (rows <= 4) return f(Int<4>{});
  return f(Int<8>{});
}

// (codebooks, code bytes) of the wgmma GEMMs: K in {1, 2, 4, 8}, 8- or 16-bit codes
template <typename F>
static int with_gemm_scheme(const aqlm_b200_weight_t* w, F&& f) {
  const auto k = [&](auto CB) {
    switch (w->num_codebooks) {
      case 1: return f(Int<1>{}, CB);
      case 2: return f(Int<2>{}, CB);
      case 4: return f(Int<4>{}, CB);
      default: return f(Int<8>{}, CB);
    }
  };
  return w->nbits_per_codebook <= 8 ? k(Int<1>{}) : k(Int<2>{});
}

// wgmma N of a GEMM plan: 16, 32, 64 or 128
template <typename F>
static int with_n_tile(int n_tile, F&& f) {
  switch (n_tile) {
    case 16: return f(Int<16>{});
    case 32: return f(Int<32>{});
    case 64: return f(Int<64>{});
    default: return f(Int<128>{});
  }
}

// ---- launches -------------------------------------------------------------------------------------------------
// Opt-in dynamic shared memory.  cudaFuncSetAttribute applies to the CURRENT device only, so the high-water mark is
// kept per (kernel instantiation, device): a process that drives several GPUs configures each of them.  The marks are
// keyed on the kernel itself, not on its type: several kernels share one function-pointer type.
template <auto Kernel>
static int ensure_smem(size_t smem, const DeviceInfo* di) {
  static std::atomic<size_t> marks[kMaxDevices];
  std::atomic<size_t>& m = marks[di->index];
  if (smem > 48 * 1024 && m.load(std::memory_order_relaxed) < smem) {
    AQLM_CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    m.store(smem, std::memory_order_relaxed);
  }
  return AQLM_B200_OK;
}

// One launch of Kernel(args...) with programmatic dependent launch as AQLM_B200_PDL says (the kernel's prologue may
// overlap the previous kernel's tail) and, for cluster_x > 0, clusters of cluster_x CTAs along x.
template <auto Kernel, typename... Args>
static int launch(const DeviceInfo* di, dim3 grid, int threads, size_t smem, cudaStream_t st, int cluster_x,
                  const Args&... args) {
  if (int rc = ensure_smem<Kernel>(smem, di)) return rc;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 0) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = tun().pdl ? 1 : 0;
  ++n;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = n;
  AQLM_CUDA_CHECK(cudaLaunchKernelEx(&cfg, Kernel, args...));
  count_launch();
  return AQLM_B200_OK;
}

// ---- gather GEMV: host side -------------------------------------------------------------------------------------
// GEMV parameters of one plain linear (one segment, rows dealt round-robin)
static GemvParams gemv_params(const aqlm_b200_weight_t* w, const void* x, void* y, int64_t batch, bool partial) {
  GemvParams p;
  p.codes = w->codes;
  p.codebooks = w->codebooks;
  p.scales = w->scales;
  p.bias = w->bias;
  p.x = x;
  p.y = y;
  p.out_features = (int)w->out_features;
  p.in_features = (int)w->in_features;
  p.in_groups = (int)(w->in_features / w->in_group_size);
  p.nbits = w->nbits_per_codebook;
  p.num_codebooks = w->num_codebooks;
  p.batch = (int)batch;
  p.partial_f32 = partial ? 1 : 0;
  p.n_seg = 1;
  p.row_block = 0;
  p.seg_end[0] = p.seg_end[1] = p.seg_end[2] = p.seg_end[3] = p.out_features;
  return p;
}

// smem bytes of the vector GEMV: x tile + staged codebooks + per-(row,slice) partials
static size_t vec_smem_bytes(const GemvParams& p, int K, int code_bytes, int G, int BT, bool cbs, int grid) {
  const int gpc = 16 / (K * code_bytes);
  const int chunks = p.in_groups / gpc;
  const int slices = (chunks + kSliceChunks - 1) / kSliceChunks;
  const int rows_cta = (p.out_features + grid - 1) / grid;
  return (size_t)BT * p.in_features * 2 + (cbs ? ((size_t)K << p.nbits) * G * 2 : 0) +
         (size_t)rows_cta * slices * BT * 4;
}

template <typename T, int K, int CB, int G, int BT, bool CBS>
static int launch_vec(const GemvParams& p, const DeviceInfo* di, cudaStream_t st) {
  constexpr int THREADS = (BT <= 2) ? 1024 : 512;
  const int grid = di->sm_count * tun().gemv_ctas_per_sm;
  return launch<gemv_vec_kernel<T, K, CB, G, BT, CBS, THREADS>>(di, grid, THREADS,
                                                                vec_smem_bytes(p, K, CB, G, BT, CBS, grid), st, 0, p);
}

template <typename T, int BT>
static int launch_1x16(const GemvParams& p, const DeviceInfo* di, cudaStream_t st) {
  const int grid = di->sm_count;
  return launch<gemv_1x16_kernel<T, BT>>(di, grid, kGemv1x16Threads, vec_smem_bytes(p, 1, 2, 8, BT, false, grid), st, 0,
                                         p, GemvPeer{});
}

// Fused GEMV + peer-memory exchange (gemv_1x16_kernel<..., PEER = true>): contiguous row blocks, one CTA per SM.
template <typename T, int BT>
static int launch_1x16_peer(GemvParams p, const GemvPeer& pc, const DeviceInfo* di, cudaStream_t st) {
  const int grid = di->sm_count;
  if (grid > kPeerFlagStride) return fail(AQLM_B200_ERR_UNSUPPORTED, "fused exchange: more SMs than flag slots");
  int rb = (p.out_features + grid - 1) / grid;
  rb = (rb + 3) & ~3;
  p.row_block = rb;
  const int chunks = p.in_groups / 8;
  const int slices = (chunks + kSliceChunks - 1) / kSliceChunks;
  const size_t smem = (size_t)BT * p.in_features * 2 + (size_t)rb * slices * BT * 4;
  if (smem > (size_t)di->max_smem_optin - 1024)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "fused exchange: activation tile + partials do not fit in shared memory");
  return launch<gemv_1x16_kernel<T, BT, true>>(di, grid, kGemv1x16Threads, smem, st, 0, p, pc);
}

template <typename T, int CB, int G, int BT>
static int launch_generic(const GemvParams& p, const DeviceInfo* di, cudaStream_t st) {
  int blocks = (p.out_features + 7) / 8;
  if (blocks > di->sm_count * 8) blocks = di->sm_count * 8;
  gemv_generic_kernel<T, CB, G, BT><<<blocks, kGemvThreads, 0, st>>>(p);
  count_launch();
  AQLM_CUDA_CHECK(cudaGetLastError());
  return AQLM_B200_OK;
}

template <typename T, int BT>
static int dispatch_bt(const aqlm_b200_weight_t* w, const GemvParams& p, const DeviceInfo* di, cudaStream_t st) {
  const int K = w->num_codebooks, nbits = w->nbits_per_codebook, G = w->in_group_size;
  const int code_bytes = nbits <= 8 ? 1 : 2;
  const size_t row_bytes = (size_t)p.in_groups * K * code_bytes;
  const bool vec_ok = (row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(w->codes) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.x) & 15) == 0) && !tun().force_generic;
  const size_t budget = (size_t)di->max_smem_optin - 1024;
  const int grid = di->sm_count * tun().gemv_ctas_per_sm;
  const bool pow2k = (K == 1 || K == 2 || K == 4 || K == 8);
  const size_t need = pow2k ? vec_smem_bytes(p, K, code_bytes, G, BT, nbits == 8, grid) : (size_t)-1;
  if (vec_ok && nbits == 16 && K == 1 && G == 8 && vec_smem_bytes(p, 1, 2, 8, BT, false, di->sm_count) <= budget)
    return launch_1x16<T, BT>(p, di, st);
  // g = 16: one codebook entry is fetched as ONE 256-bit request, which needs a 32-byte aligned table (any torch
  // allocation is); a 16-byte aligned table handed in through the C-ABI takes the generic kernel below
  if (vec_ok && nbits == 16 && K == 1 && G == 16 && need <= budget && (reinterpret_cast<uintptr_t>(w->codebooks) & 31) == 0)
    return launch_vec<T, 1, 2, 16, BT, false>(p, di, st);
  if (vec_ok && nbits == 8 && G == 8 && pow2k && need <= budget) {
    if (K == 1) return launch_vec<T, 1, 1, 8, BT, true>(p, di, st);
    if (K == 2) return launch_vec<T, 2, 1, 8, BT, true>(p, di, st);
    if (K == 4) return launch_vec<T, 4, 1, 8, BT, true>(p, di, st);
    if (K == 8) return launch_vec<T, 8, 1, 8, BT, true>(p, di, st);
  }
  if (code_bytes == 2) {
    if (G == 8) return launch_generic<T, 2, 8, BT>(p, di, st);
    return launch_generic<T, 2, 16, BT>(p, di, st);
  }
  if (G == 8) return launch_generic<T, 1, 8, BT>(p, di, st);
  return launch_generic<T, 1, 16, BT>(p, di, st);
}

template <typename T>
static int matmat_typed(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                        const DeviceInfo* di, cudaStream_t st) {
  const bool partial = (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0;
  const size_t out_elt = partial ? 4 : 2;
  // largest pass size whose x tile fits in shared memory
  int max_bt = 8;
  while (max_bt > 1 && (size_t)max_bt * w->in_features * 2 + 40 * 1024 > (size_t)di->max_smem_optin) max_bt >>= 1;
  for (int64_t b0 = 0; b0 < batch; b0 += max_bt) {
    const int nb = (int)((batch - b0) < max_bt ? (batch - b0) : max_bt);
    const GemvParams p = gemv_params(w, reinterpret_cast<const uint8_t*>(input) + (size_t)b0 * w->in_features * 2,
                                     reinterpret_cast<uint8_t*>(output) + (size_t)b0 * w->out_features * out_elt, nb,
                                     partial);
    if (int rc = with_batch_tile(nb, [&](auto BT) { return dispatch_bt<T, BT>(w, p, di, st); })) return rc;
  }
  return AQLM_B200_OK;
}

template <typename T>
static int dequant_typed(const aqlm_b200_weight_t* w, void* out, int apply_scales, cudaStream_t st) {
  const int in_groups = (int)(w->in_features / w->in_group_size);
  const int64_t n = w->out_features * in_groups;
  const int threads = 256;
  const int64_t blocks = (n + threads - 1) / threads;
  if (blocks > 0x7fffffffll) return fail(AQLM_B200_ERR_SHAPE, "weight too large for one dequant launch");
  const T* sc = apply_scales ? reinterpret_cast<const T*>(w->scales) : nullptr;
  const auto go = [&](auto CB, auto G) {
    dequant_kernel<T, CB, G><<<(unsigned)blocks, threads, 0, st>>>(w->codes, w->codebooks, sc, out, w->out_features,
                                                                   in_groups, w->num_codebooks, w->nbits_per_codebook);
  };
  const bool g8 = w->in_group_size == 8;
  if (w->nbits_per_codebook <= 8) g8 ? go(Int<1>{}, Int<8>{}) : go(Int<1>{}, Int<16>{});
  else g8 ? go(Int<2>{}, Int<8>{}) : go(Int<2>{}, Int<16>{});
  count_launch();
  AQLM_CUDA_CHECK(cudaGetLastError());
  return AQLM_B200_OK;
}

// ---- Kx8 LUT GEMV: host side ------------------------------------------------------------------------
template <typename T, int K, int J>
static int launch_lut(const aqlm_b200_weight_t* w, const void* input, void* output, uint32_t flags, const LutPlan& L,
                      void* workspace, const DeviceInfo* di, cudaStream_t st) {
  LutParams p;
  p.codes = w->codes;
  p.codebooks = w->codebooks;
  p.scales = w->scales;
  p.bias = w->bias;
  p.x = input;
  p.y = output;
  p.ws_counters = reinterpret_cast<unsigned int*>(workspace);
  p.ws_gen = p.ws_counters + kGemmMaxTiles;  // generation words live in the upper half of the counter region
  p.ws_partials = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + kWsCountersBytes);
  p.out_features = (int)w->out_features;
  p.in_groups = (int)(w->in_features / 8);
  p.n_slabs = L.n_slabs;
  p.rows_per_block = L.rows_per_block;
  p.partial_f32 = (flags & AQLM_B200_FLAG_PARTIAL_F32) ? 1 : 0;
  constexpr int THREADS = (K <= 2) ? 256 : 512;  // K >= 4: one CTA per SM (128 KiB LUT), so give it 16 warps
  return launch<gemv_lut_kernel<T, K, J, THREADS>>(di, dim3(L.n_slabs, L.row_blocks), THREADS, L.smem, st, 0, p);
}

template <typename T>
static int lut_typed(const aqlm_b200_weight_t* w, const void* input, void* output, uint32_t flags, const LutPlan& L,
                     void* workspace, const DeviceInfo* di, cudaStream_t st) {
  switch (w->num_codebooks) {
    case 1: return launch_lut<T, 1, 32>(w, input, output, flags, L, workspace, di, st);
    case 2: return launch_lut<T, 2, 32>(w, input, output, flags, L, workspace, di, st);
    case 4: return launch_lut<T, 4, 32>(w, input, output, flags, L, workspace, di, st);
    default: return launch_lut<T, 8, 16>(w, input, output, flags, L, workspace, di, st);
  }
}

static LutClusterParams lut_cluster_params(const aqlm_b200_weight_t* w, const void* input, void* output,
                                           uint32_t flags, int n_slabs, int rows_per_block) {
  LutClusterParams p;
  p.codes = w->codes;
  p.codebooks = w->codebooks;
  p.scales = w->scales;
  p.bias = w->bias;
  p.x = input;
  p.y = output;
  p.out_features = (int)w->out_features;
  p.in_groups = (int)(w->in_features / 8);
  p.n_slabs = n_slabs;
  p.rows_per_block = rows_per_block;
  p.partial_f32 = (flags & AQLM_B200_FLAG_PARTIAL_F32) ? 1 : 0;
  return p;
}

// ---- Kx8 LUT GEMV, cluster / DSMEM variant (K <= 2, at most 8 slabs of 64 groups): host side ---------------
template <typename T, int K>
static int launch_lut_cluster(const aqlm_b200_weight_t* w, const void* input, void* output, uint32_t flags,
                              const DeviceInfo* di, cudaStream_t st, bool* taken) {
  *taken = false;
  const int n_slabs = lut_cluster_slabs(*w);
  const size_t lut_bytes = (size_t)K * 256 * kLutCJ * 4;
  // How many clusters of n_slabs CTAs can be resident at once; the grid is sized from this.  The query describes
  // 512-thread CTAs with the LUT + 8 KiB of shared memory, not the launch below: at 512 threads the 768-thread build's
  // registers allow one CTA per SM, as the launch's shared memory does.
  static std::atomic<int> max_clusters[kMaxDevices][9];
  int mc = max_clusters[di->index][n_slabs].load(std::memory_order_relaxed);
  if (mc == 0) {
    constexpr auto kernel = gemv_lut_cluster_kernel<T, K, 768>;
    const size_t smem_max = lut_bytes + 8192;
    if (int rc = ensure_smem<kernel>(smem_max, di)) return rc;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = n_slabs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(n_slabs, di->sm_count);
    cfg.blockDim = dim3(512);
    cfg.dynamicSmemBytes = smem_max;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess || n < 1) {
      (void)cudaGetLastError();
      n = -1;  // not launchable as a cluster here: use the workspace kernel
    }
    mc = n;
    max_clusters[di->index][n_slabs].store(mc, std::memory_order_relaxed);
  }
  const LutClusterRows r = lut_cluster_rows(*w, mc);
  if (!r.rows_per_block) return AQLM_B200_OK;
  const LutClusterParams p = lut_cluster_params(w, input, output, flags, n_slabs, r.rows_per_block);
  // one warp per 16-row batch of the row block (8 to 32 warps); up to 768 threads the 80-register build
  int warps = (r.rows_per_block + 15) / 16;
  warps = warps < 8 ? 8 : (warps > 32 ? 32 : warps);
  const size_t smem = (size_t)kLutAbs + lut_bytes;  // LUT ends at 0x10000 * (1 + K) whatever the window base
  const auto go = [&](auto MAXT) {
    return launch<gemv_lut_cluster_kernel<T, K, MAXT>>(di, dim3(n_slabs, r.row_blocks), warps * 32, smem, st, n_slabs,
                                                       p);
  };
  const int rc = warps <= 24 ? go(Int<768>{}) : go(Int<1024>{});
  *taken = rc == AQLM_B200_OK;
  return rc;
}

// Batch-1 call on a 1x8 / 2x8 weight whose in_features fit 8 slabs: no workspace needed.
static int try_lut_cluster(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                           const DeviceInfo* di, cudaStream_t st, bool* taken) {
  *taken = false;
  if (!lut_cluster_eligible(*w, input, batch, tun())) return AQLM_B200_OK;
  return with_dtype(w->dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    return w->num_codebooks == 1 ? launch_lut_cluster<T, 1>(w, input, output, flags, di, st, taken)
                                 : launch_lut_cluster<T, 2>(w, input, output, flags, di, st, taken);
  });
}

// ---- fused dequant + wgmma GEMM: host side ------------------------------------------------------
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static tmap_encode_fn get_tmap_encode() {
  static tmap_encode_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<tmap_encode_fn>(p);
  });
  return fn;
}

// cuTensorMapEncodeTiled is a DRIVER entry point: it needs a current context on the calling thread.  Threads that have
// only made runtime calls that do not bind one (e.g. an autograd worker thread: error 201, CUDA_ERROR_INVALID_CONTEXT)
// get the primary context bound by a no-op runtime call, once per thread.
static void ensure_driver_context() {
  static thread_local bool bound = false;
  if (!bound) {
    (void)cudaFree(nullptr);
    bound = true;
  }
}

// TMA map of a row-major [rows][cols] matrix (row_bytes apart) in boxes of box_rows x box_cols; `what` names it in errors
static int encode_tmap(CUtensorMap* map, const char* what, CUtensorMapDataType type, const void* base, uint64_t cols,
                       uint64_t rows, uint64_t row_bytes, uint32_t box_cols, uint32_t box_rows,
                       CUtensorMapSwizzle swizzle) {
  tmap_encode_fn enc = get_tmap_encode();
  if (!enc) return fail(AQLM_B200_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  ensure_driver_context();
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {row_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t es[2] = {1, 1};
  CUresult r = enc(map, type, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(AQLM_B200_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r);
  return AQLM_B200_OK;
}

template <typename T>
constexpr CUtensorMapDataType kTmapType = DT<T>::is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;

// One launch of either GEMM.  Forward: b = x [batch][in_features], y [batch][out_features] (fp32 sums with `partial`).
// TRANSPOSED (backward w.r.t. the input): b = grad_output [batch][out_features], y = grad_input [batch][in_features].
// The directions differ in the code-tile map and in which side of W is the contraction; the rest is shared.
// Segments of the out rows (GemmParams::n_seg / seg_end): one for a plain linear, up to 4 for a grouped call.
struct GemmSegments {
  int n_seg = 1;
  int seg_end[4] = {0, 0, 0, 0};
};

static GemmSegments single_segment(const aqlm_b200_weight_t* w) {
  GemmSegments s;
  for (int& e : s.seg_end) e = (int)w->out_features;
  return s;
}

// A routed call (expert_off != NULL) covers n_experts stacked experts of w's shape: the code map spans all of them.
template <typename T, int K, int CB, bool TRANSPOSED>
static int launch_gemm(const aqlm_b200_weight_t* w, const void* b, void* y, int64_t batch, bool partial, const GemmPlan& g,
                       const GemmSegments& segs, void* workspace, const DeviceInfo* di, cudaStream_t st,
                       const int32_t* expert_off = nullptr, int n_experts = 1) {
  using Dir = std::conditional_t<TRANSPOSED, GemmTransposed<K, CB>, GemmForward<K, CB>>;
  const int64_t k_size = TRANSPOSED ? w->out_features : w->in_features;
  const size_t row_bytes = (size_t)(w->in_features / 8) * K * CB;
  CUtensorMap tb, tc;
  if (int rc = encode_tmap(&tb, TRANSPOSED ? "grad_output" : "x", kTmapType<T>, b, k_size, batch, k_size * 2, kGemmBlockK,
                           g.n_tile, CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  const uint64_t code_rows = (uint64_t)w->out_features * (uint64_t)n_experts;
  if (int rc = TRANSPOSED ? encode_tmap(&tc, "codes, transposed", CU_TENSOR_MAP_DATA_TYPE_UINT8, w->codes, row_bytes,
                                        code_rows, row_bytes, 16 * K * CB, kGemmTCtileRows, CU_TENSOR_MAP_SWIZZLE_NONE)
                          : encode_tmap(&tc, "codes", CU_TENSOR_MAP_DATA_TYPE_UINT8, w->codes, row_bytes, code_rows,
                                        row_bytes, kCodeTileBytes, g.tile_m, CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  GemmParams p;
  p.codebooks = w->codebooks;
  p.scales = partial ? nullptr : w->scales;
  p.bias = partial || TRANSPOSED ? nullptr : w->bias;
  p.partial_f32 = partial ? 1 : 0;
  p.y = y;
  p.ws_counters = g.ksplit > 1 ? reinterpret_cast<unsigned int*>(workspace) : nullptr;
  p.ws_partials = g.ksplit > 1 ? reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + g.counters_bytes) : nullptr;
  p.m_size = (int)(TRANSPOSED ? w->in_features : w->out_features);
  p.k_size = (int)k_size;
  p.batch = (int)batch;
  p.nbits = w->nbits_per_codebook;
  p.total_kblocks = g.total_kblocks;
  p.ksplit = g.ksplit;
  p.stages = g.stages;
  p.tile_m = g.tile_m;
  p.gather_mode = tun().gemm_gather_mode >= 0 ? tun().gemm_gather_mode : (w->nbits_per_codebook > 8 ? 1 : 0);
  p.n_seg = segs.n_seg;
  for (int i = 0; i < 4; ++i) p.seg_end[i] = segs.seg_end[i];
  p.expert_off = expert_off;
  p.n_experts = n_experts;
  return with_n_tile(g.n_tile, [&](auto N) {
    const dim3 grid(g.m_tiles, g.ksplit, g.n_tiles);  // routed: n_tiles is the slot count
    const size_t smem = gemm_smem_layout(g.stages, N, Dir::kCtileBytes).total;
    if (expert_off) {
      constexpr auto kernel = TRANSPOSED ? gemm_dequant_t_routed_kernel<T, K, CB, N> : gemm_dequant_routed_kernel<T, K, CB, N>;
      return launch<kernel>(di, grid, kGemmThreads, smem, st, 0, tb, tc, p);
    }
    if (segs.n_seg > 1) {
      constexpr auto kernel = TRANSPOSED ? gemm_dequant_t_grouped_kernel<T, K, CB, N> : gemm_dequant_grouped_kernel<T, K, CB, N>;
      return launch<kernel>(di, grid, kGemmThreads, smem, st, 0, tb, tc, p);
    }
    constexpr auto kernel = TRANSPOSED ? gemm_dequant_t_kernel<T, K, CB, N> : gemm_dequant_kernel<T, K, CB, N>;
    return launch<kernel>(di, grid, kGemmThreads, smem, st, 0, tb, tc, p);
  });
}

static aqlm_b200_weight_t make_weight(const void* codes, const void* codebooks, const void* scales, const void* bias,
                                      int64_t in_features, int64_t out_features, int K, int nbits, int g, int dtype) {
  aqlm_b200_weight_t w;
  memset(&w, 0, sizeof(w));
  w.codes = codes;
  w.codebooks = codebooks;
  w.scales = scales;
  w.bias = bias;
  w.in_features = in_features;
  w.out_features = out_features;
  w.num_codebooks = K;
  w.nbits_per_codebook = nbits;
  w.in_group_size = g;
  w.out_group_size = 1;
  w.dtype = dtype;
  return w;
}

// ---- grouped wgmma GEMM (forward and transposed): host side -----------------------------------------------------
// Everything a grouped GEMM call checks without a device, in this order: arguments and segment table (ERR_SHAPE), then
// the layouts the wgmma kernels take (ERR_UNSUPPORTED).  There is no GEMV form of a grouped call above 8 rows, so a
// layout the kernels do not take is an error the caller handles (by running the members one by one).
// The segment table of a grouped or routed call (ERR_SHAPE).
static int gemm_segment_table(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const char* what,
                              GemmSegments* segs) {
  if (!seg_rows || n_seg < 1 || n_seg > 4) return fail(AQLM_B200_ERR_SHAPE, "%s GEMM takes 1..4 segments, got %d", what, n_seg);
  int64_t acc = 0;
  for (int i = 0; i < n_seg; ++i) {
    if (seg_rows[i] <= 0) return fail(AQLM_B200_ERR_SHAPE, "segment %d has %lld rows", i, (long long)seg_rows[i]);
    acc += seg_rows[i];
    if (acc > w->out_features) break;
    segs->seg_end[i] = (int)acc;
  }
  if (acc != w->out_features)
    return fail(AQLM_B200_ERR_SHAPE, "segment rows do not add up to out_features (%lld)", (long long)w->out_features);
  for (int i = n_seg; i < 4; ++i) segs->seg_end[i] = (int)acc;
  segs->n_seg = n_seg;
  return AQLM_B200_OK;
}

// The layouts the wgmma kernels of a grouped or routed call take (ERR_UNSUPPORTED otherwise).
static int gemm_layout_checks(const aqlm_b200_weight_t* w, const void* b, bool transposed, const char* what) {
  const int K = w->num_codebooks, nbits = w->nbits_per_codebook, cb = nbits <= 8 ? 1 : 2;
  if (w->in_group_size != 8 || (nbits != 8 && nbits != 16) || !(K == 1 || K == 2 || K == 4 || K == 8))
    return fail(AQLM_B200_ERR_UNSUPPORTED,
                "%s GEMM covers in_group_size 8, 8/16-bit codes and 1/2/4/8 codebooks; got %dx%d, in_group_size %d",
                what, K, nbits, w->in_group_size);
  if (!transposed && w->in_features % kGemmBlockK != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "%s GEMM needs in_features %% 64 == 0, got %lld", what,
                (long long)w->in_features);
  if (transposed && w->out_features % 8 != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "%s transposed GEMM needs out_features %% 8 == 0, got %lld", what,
                (long long)w->out_features);
  if (((size_t)(w->in_features / 8) * K * cb) % 16 != 0 || (reinterpret_cast<uintptr_t>(w->codes) & 15) != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "%s GEMM needs 16-byte aligned code rows", what);
  if ((reinterpret_cast<uintptr_t>(b) & 15) != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "%s GEMM needs a 16-byte aligned %s", what, transposed ? "grad_output" : "input");
  return AQLM_B200_OK;
}

static int grouped_gemm_checks(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* b,
                               const void* y, int64_t batch, bool partial, bool transposed, GemmSegments* segs) {
  int rc = validate(w, !partial);
  if (rc) return rc;
  if (batch < 0) return fail(AQLM_B200_ERR_SHAPE, "negative batch");
  if (!b || !y) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  if ((rc = gemm_segment_table(w, seg_rows, n_seg, "grouped", segs))) return rc;
  return gemm_layout_checks(w, b, transposed, "grouped");
}

// One launch of the forward (y [batch][out], fp32 sums with `partial`) or the transposed (y = grad_input [batch][in])
// GEMM over the row-concatenated weight, with the plan of the concatenated descriptor.
template <bool TRANSPOSED>
static int grouped_gemm(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* b, void* y,
                        int64_t batch, bool partial, void* workspace, size_t workspace_bytes, void* stream) {
  GemmSegments segs;
  int rc = grouped_gemm_checks(w, seg_rows, n_seg, b, y, batch, partial, TRANSPOSED, &segs);
  if (rc || batch == 0) return rc;
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  const auto plan = [&](bool split) {
    return TRANSPOSED ? gemm_t_plan(*w, batch, *di, tun(), split) : gemm_plan(*w, batch, *di, tun(), split);
  };
  GemmPlan g = plan(workspace != nullptr);
  if (g.ok && g.ksplit > 1 && workspace_bytes < g.counters_bytes + g.partials_bytes) g = plan(false);
  if (!g.ok) return fail(AQLM_B200_ERR_UNSUPPORTED, "grouped GEMM: no wgmma plan for this descriptor and batch");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_dtype(w->dtype, [&](auto tag) {
    return with_gemm_scheme(w, [&](auto K, auto CB) {
      return launch_gemm<typename decltype(tag)::type, K, CB, TRANSPOSED>(w, b, y, batch, partial, g, segs, workspace, di,
                                                                          st);
    });
  });
}

// ---- routed wgmma GEMM (mixture-of-experts, forward and transposed): host side -----------------------------------
constexpr int kRoutedMaxExperts = 64;

// Everything a routed call checks without a device, in this order: descriptor, segment table, expert count, pointers
// (ERR_SHAPE); then the layouts the wgmma kernels take (ERR_UNSUPPORTED), exactly as for a grouped call.
static int routed_gemm_checks(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, int n_experts,
                              const int32_t* expert_off, const void* b, const void* y, int64_t rows, bool transposed,
                              GemmSegments* segs) {
  int rc = validate(w, true);
  if (rc) return rc;
  if (rows < 0) return fail(AQLM_B200_ERR_SHAPE, "negative row count");
  if (rows > 0x7fffffffll) return fail(AQLM_B200_ERR_SHAPE, "routed GEMM takes at most 2^31 - 1 rows");
  const int64_t one[1] = {w->out_features};
  if ((rc = gemm_segment_table(w, (seg_rows || n_seg != 1) ? seg_rows : one, n_seg, "routed", segs))) return rc;
  if (n_experts < 1 || n_experts > kRoutedMaxExperts)
    return fail(AQLM_B200_ERR_SHAPE, "routed GEMM takes 1..%d experts, got %d", kRoutedMaxExperts, n_experts);
  if (w->out_features * n_experts > 0x7fffffffll)  // the stacked out rows are a TMA coordinate
    return fail(AQLM_B200_ERR_SHAPE, "routed GEMM: %d experts x %lld out rows exceed 2^31 - 1", n_experts,
                (long long)w->out_features);
  if (!expert_off) return fail(AQLM_B200_ERR_SHAPE, "expert offsets pointer is NULL");
  if (!b || !y) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  return gemm_layout_checks(w, b, transposed, "routed");
}

template <bool TRANSPOSED>
static int routed_gemm(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, int n_experts,
                       const int32_t* expert_off, const void* b, void* y, int64_t rows, void* workspace,
                       size_t workspace_bytes, void* stream) {
  GemmSegments segs;
  int rc = routed_gemm_checks(w, seg_rows, n_seg, n_experts, expert_off, b, y, rows, TRANSPOSED, &segs);
  if (rc || rows == 0) return rc;
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  const auto plan = [&](bool split) { return gemm_routed_plan(*w, rows, n_experts, *di, tun(), split, TRANSPOSED); };
  GemmPlan g = plan(workspace != nullptr);
  if (g.ok && g.ksplit > 1 && workspace_bytes < g.counters_bytes + g.partials_bytes) g = plan(false);
  if (!g.ok) return fail(AQLM_B200_ERR_UNSUPPORTED, "routed GEMM: no wgmma plan for this descriptor and row count");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_dtype(w->dtype, [&](auto tag) {
    return with_gemm_scheme(w, [&](auto K, auto CB) {
      return launch_gemm<typename decltype(tag)::type, K, CB, TRANSPOSED>(w, b, y, rows, false, g, segs, workspace, di,
                                                                          st, expert_off, n_experts);
    });
  });
}

// ---- fused weight-gradient GEMM: host side ------------------------------------------------------------------------
// Everything a weight-gradient call checks without a device: descriptor, pointers (ERR_SHAPE), then the layouts the
// kernel takes (ERR_UNSUPPORTED).
static int weight_grad_checks(const aqlm_b200_weight_t* w, const void* input, const void* grad_output, int64_t batch,
                              const float* grad_codebooks, const float* grad_scales) {
  int rc = validate(w, grad_codebooks != nullptr);
  if (rc) return rc;
  if (batch < 0 || batch > 0x7fffffffll) return fail(AQLM_B200_ERR_SHAPE, "weight gradient: batch %lld out of range", (long long)batch);
  if (!input || !grad_output) return fail(AQLM_B200_ERR_SHAPE, "weight gradient: input/grad_output pointer is NULL");
  if (!grad_codebooks && !grad_scales)
    return fail(AQLM_B200_ERR_SHAPE, "weight gradient: neither grad_codebooks nor grad_scales requested");
  const int K = w->num_codebooks, nbits = w->nbits_per_codebook, cb = nbits <= 8 ? 1 : 2;
  if (w->in_group_size != 8 || (nbits != 8 && nbits != 16) || !(K == 1 || K == 2 || K == 4 || K == 8))
    return fail(AQLM_B200_ERR_UNSUPPORTED,
                "weight gradient covers in_group_size 8, 8/16-bit codes and 1/2/4/8 codebooks; got %dx%d, in_group_size %d",
                K, nbits, w->in_group_size);
  if (w->out_features % 8 != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "weight gradient needs out_features %% 8 == 0, got %lld", (long long)w->out_features);
  if (((size_t)(w->in_features / 8) * K * cb) % 16 != 0 || (reinterpret_cast<uintptr_t>(w->codes) & 15) != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "weight gradient needs 16-byte aligned code rows");
  if ((reinterpret_cast<uintptr_t>(input) & 15) != 0 || (reinterpret_cast<uintptr_t>(grad_output) & 15) != 0)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "weight gradient needs a 16-byte aligned input and grad_output");
  return AQLM_B200_OK;
}

template <typename T, int K, int CB>
static int launch_weight_grad(const aqlm_b200_weight_t* w, const void* input, const void* grad_output, int64_t batch,
                              float* grad_codebooks, float* grad_scales, void* workspace, const WgradPlan& g,
                              const DeviceInfo* di, cudaStream_t st) {
  CUtensorMap tg, tx;
  if (int rc = encode_tmap(&tg, "grad_output", kTmapType<T>, grad_output, w->out_features, batch, w->out_features * 2, 64,
                           kWgradBlockK, CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  if (int rc = encode_tmap(&tx, "input", kTmapType<T>, input, w->in_features, batch, w->in_features * 2, 64, kWgradBlockK,
                           CU_TENSOR_MAP_SWIZZLE_128B))
    return rc;
  WgradParams p;
  p.codes = w->codes;
  p.codebooks = w->codebooks;
  p.scales = w->scales;
  p.grad_codebooks = grad_codebooks;
  p.grad_scales = grad_scales;
  p.ws_counters = grad_scales ? reinterpret_cast<unsigned int*>(workspace) : nullptr;
  p.ws_dots = grad_scales ? reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + g.counters_bytes) : nullptr;
  p.out_features = (int)w->out_features;
  p.in_features = (int)w->in_features;
  p.nbits = w->nbits_per_codebook;
  p.total_kblocks = g.total_kblocks;
  p.stages = g.stages;
  return launch<gemm_wgrad_kernel<T, K, CB>>(di, dim3(g.out_tiles, g.in_tiles), kWgradThreads, g.smem, st, 0, tg, tx, p);
}

}  // namespace aqlm_b200

using namespace aqlm_b200;

extern "C" {

int aqlm_b200_version(void) { return AQLM_B200_VERSION; }
void aqlm_b200_reload_tunables(void) { tun().load(); }
const char* aqlm_b200_last_error(void) { return tls_error_buf(); }
uint64_t aqlm_b200_launch_count(void) { return g_launch_count.load(); }

int aqlm_b200_matmat_ex(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                        void* stream) {
  const bool partial = (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0;
  int rc = validate(w, !partial);
  if (rc) return rc;
  if (batch < 0) return fail(AQLM_B200_ERR_SHAPE, "negative batch");
  if (batch == 0) return AQLM_B200_OK;
  if (!input || !output) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  {
    // batch 1 -- and batch 2-3 as one launch per row, like the reference's per-row host loop (cuda_kernel.cpp:387-421):
    // up to 3 rows this replaces one pass of the gather kernel (AQLM_B200_LUT_BATCH_LOOP=0 selects that pass instead)
    const int64_t lut_rows = (batch == 1 || (tun().lut_batch_loop && batch <= 3)) ? batch : 0;
    const size_t out_elt = partial ? 4 : 2;
    int64_t done = 0;
    for (; done < lut_rows; ++done) {
      bool taken = false;
      rc = try_lut_cluster(w, reinterpret_cast<const uint8_t*>(input) + (size_t)done * w->in_features * 2,
                           reinterpret_cast<uint8_t*>(output) + (size_t)done * w->out_features * out_elt, 1, flags, di, st, &taken);
      if (rc) return rc;
      if (!taken) break;  // not applicable (decided before any launch: `taken` is the same for every row)
    }
    if (lut_rows > 0 && done == lut_rows) return AQLM_B200_OK;
  }
  return with_dtype(w->dtype, [&](auto tag) {
    return matmat_typed<typename decltype(tag)::type>(w, input, output, batch, flags, di, st);
  });
}

size_t aqlm_b200_matmat_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch) {
  if (validate(w, false) != AQLM_B200_OK || batch <= 0) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return 0;
  if (batch > 2) return 0;
  const LutPlan L = lut_plan(*w, 1, *di, tun());
  return L.ok ? kWsCountersBytes + L.partials_bytes : 0;
}

int aqlm_b200_matmat_ws(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                        void* workspace, size_t workspace_bytes, void* stream) {
  const bool partial = (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0;
  int rc = validate(w, !partial);
  if (rc) return rc;
  const int64_t ws_rows = (batch == 1 || (tun().lut_batch_loop && batch == 2 && w->num_codebooks >= 4)) ? batch : 0;
  if (ws_rows > 0 && workspace && input && output && (reinterpret_cast<uintptr_t>(input) & 3) == 0) {
    const DeviceInfo* di;
    if ((rc = current_device(&di))) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (batch == 1) {  // K <= 2, in <= 4096: the cluster kernel needs no workspace (matmat_ex also loops it for batch 2-3)
      bool taken = false;
      rc = try_lut_cluster(w, input, output, 1, flags, di, st, &taken);
      if (rc || taken) return rc;
    }
    const LutPlan L = lut_plan(*w, 1, *di, tun());
    const bool cluster_case = w->num_codebooks <= 2 && (w->in_features / 8) <= 8 * kLutCJ;
    if (L.ok && workspace_bytes >= kWsCountersBytes + L.partials_bytes && !(batch > 1 && cluster_case)) {
      const size_t out_elt = partial ? 4 : 2;
      for (int64_t b = 0; b < ws_rows; ++b) {  // launches are stream-ordered: the workspace is reused row after row
        const void* xin = reinterpret_cast<const uint8_t*>(input) + (size_t)b * w->in_features * 2;
        void* yout = reinterpret_cast<uint8_t*>(output) + (size_t)b * w->out_features * out_elt;
        rc = with_dtype(w->dtype, [&](auto tag) {
          return lut_typed<typename decltype(tag)::type>(w, xin, yout, flags, L, workspace, di, st);
        });
        if (rc) return rc;
      }
      return AQLM_B200_OK;
    }
  }
  return aqlm_b200_matmat_ex(w, input, output, batch, flags, stream);
}

int aqlm_b200_matmat_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* input,
                             void* output, int64_t batch, uint32_t flags, void* stream) {
  const bool partial = (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0;
  int rc = validate(w, !partial);
  if (rc) return rc;
  if (!seg_rows || n_seg < 1 || n_seg > 4) return fail(AQLM_B200_ERR_SHAPE, "grouped launch takes 1..4 segments");
  if (w->num_codebooks != 1 || w->nbits_per_codebook != 16 || w->in_group_size != 8)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "grouped launch is implemented for the 1x16 (in_group 8) scheme only");
  if (batch < 1 || batch > 8) return fail(AQLM_B200_ERR_UNSUPPORTED, "grouped launch takes 1..8 batch rows");
  if (!input || !output) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  int64_t total = 0;
  for (int i = 0; i < n_seg; ++i) total += seg_rows[i];
  if (total != w->out_features) return fail(AQLM_B200_ERR_SHAPE, "segment rows do not add up to out_features");
  const size_t row_bytes = (size_t)(w->in_features / 8) * 2;
  if (row_bytes % 16 != 0 || (reinterpret_cast<uintptr_t>(w->codes) & 15) || (reinterpret_cast<uintptr_t>(input) & 15))
    return fail(AQLM_B200_ERR_UNSUPPORTED, "grouped launch needs 16-byte aligned code rows and input");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  GemvParams p = gemv_params(w, input, output, batch, partial);
  p.n_seg = n_seg;
  int64_t acc = 0;
  for (int i = 0; i < 4; ++i) {
    if (i < n_seg) acc += seg_rows[i];
    p.seg_end[i] = (int)acc;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_batch_tile(batch, [&](auto BT) {
    if (vec_smem_bytes(p, 1, 2, 8, BT, false, di->sm_count) > (size_t)di->max_smem_optin - 1024)
      return fail(AQLM_B200_ERR_UNSUPPORTED, "grouped launch: activation tile does not fit in shared memory");
    return with_dtype(w->dtype, [&](auto tag) { return launch_1x16<typename decltype(tag)::type, BT>(p, di, st); });
  });
}

int aqlm_b200_matmat(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, void* stream) {
  return aqlm_b200_matmat_ex(w, input, output, batch, 0, stream);
}

size_t aqlm_b200_matmat_dequant_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch) {
  if (validate(w, false) != AQLM_B200_OK || batch <= 0) return 0;  // the plan never reads scales
  const DeviceInfo* di = device_info();
  if (!di) return 0;
  const GemmPlan g = gemm_plan(*w, batch, *di, tun(), true);
  if (!g.ok || g.ksplit <= 1) return 0;
  return g.counters_bytes + g.partials_bytes;
}

int aqlm_b200_matmat_dequant_ex(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch,
                                uint32_t flags, void* workspace, size_t workspace_bytes, void* stream) {
  const bool partial = (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0;
  int rc = validate(w, !partial);
  if (rc) return rc;
  if (batch < 0) return fail(AQLM_B200_ERR_SHAPE, "negative batch");
  if (batch == 0) return AQLM_B200_OK;
  if (!input || !output) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GemmPlan g = gemm_plan(*w, batch, *di, tun(), workspace != nullptr);
  if (g.ok && g.ksplit > 1 && workspace_bytes < g.counters_bytes + g.partials_bytes) g = gemm_plan(*w, batch, *di, tun(), false);
  if (!g.ok || (reinterpret_cast<uintptr_t>(input) & 15) != 0) {
    // shapes the tensor-core kernel does not cover (in_group 16, in_features % 64 != 0, odd KxN):
    // batch passes of 8 rows through the fused gather+dequant+dot kernel
    return aqlm_b200_matmat_ex(w, input, output, batch, flags, stream);
  }
  return with_dtype(w->dtype, [&](auto tag) {
    return with_gemm_scheme(w, [&](auto K, auto CB) {
      return launch_gemm<typename decltype(tag)::type, K, CB, false>(w, input, output, batch, partial, g, single_segment(w),
                                                             workspace, di, st);
    });
  });
}

int aqlm_b200_matmat_dequant_ws(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch,
                                void* workspace, size_t workspace_bytes, void* stream) {
  return aqlm_b200_matmat_dequant_ex(w, input, output, batch, 0, workspace, workspace_bytes, stream);
}

int aqlm_b200_matmat_dequant(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch,
                             void* stream) {
  return aqlm_b200_matmat_dequant_ws(w, input, output, batch, nullptr, 0, stream);  // no workspace: no split-K
}

int aqlm_b200_dequant(const aqlm_b200_weight_t* w, void* weight_out, int apply_scales, void* stream) {
  int rc = validate(w, apply_scales != 0);
  if (rc) return rc;
  if (!weight_out || (reinterpret_cast<uintptr_t>(weight_out) & 15))
    return fail(AQLM_B200_ERR_SHAPE, "weight_out must be a 16-byte aligned device pointer");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_dtype(w->dtype, [&](auto tag) {
    return dequant_typed<typename decltype(tag)::type>(w, weight_out, apply_scales, st);
  });
}

size_t aqlm_b200_matmat_dequant_transposed_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch) {
  if (validate(w, true) != AQLM_B200_OK || batch <= 0) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return 0;
  const GemmPlan g = gemm_t_plan(*w, batch, *di, tun(), true);
  if (!g.ok || g.ksplit <= 1) return 0;
  return g.counters_bytes + g.partials_bytes;
}

int aqlm_b200_matmat_dequant_transposed(const aqlm_b200_weight_t* w, const void* grad_output, void* grad_input,
                                        int64_t batch, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = validate(w, true);
  if (rc) return rc;
  if (batch < 0) return fail(AQLM_B200_ERR_SHAPE, "negative batch");
  if (batch == 0) return AQLM_B200_OK;
  if (!grad_output || !grad_input) return fail(AQLM_B200_ERR_SHAPE, "grad_output/grad_input pointer is NULL");
  if ((reinterpret_cast<uintptr_t>(grad_output) & 15) != 0)
    return fail(AQLM_B200_ERR_SHAPE, "grad_output must be 16-byte aligned");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  GemmPlan g = gemm_t_plan(*w, batch, *di, tun(), workspace != nullptr);
  if (g.ok && g.ksplit > 1 && workspace_bytes < g.counters_bytes + g.partials_bytes) g = gemm_t_plan(*w, batch, *di, tun(), false);
  if (!g.ok)
    return fail(AQLM_B200_ERR_UNSUPPORTED,
                "matmat_dequant_transposed: the fused kernel covers in_group_size 8, 8/16-bit codes, 1/2/4/8 codebooks, "
                "16-byte aligned code rows and out_features %% 8 == 0");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_dtype(w->dtype, [&](auto tag) {
    return with_gemm_scheme(w, [&](auto K, auto CB) {
      return launch_gemm<typename decltype(tag)::type, K, CB, true>(w, grad_output, grad_input, batch, false, g, single_segment(w),
                                                            workspace, di, st);
    });
  });
}

int aqlm_b200_matmat_dequant_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* input,
                                     void* output, int64_t batch, uint32_t flags, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  return grouped_gemm<false>(w, seg_rows, n_seg, input, output, batch, (flags & AQLM_B200_FLAG_PARTIAL_F32) != 0,
                             workspace, workspace_bytes, stream);
}

int aqlm_b200_matmat_dequant_transposed_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                                                const void* grad_output, void* grad_input, int64_t batch, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  return grouped_gemm<true>(w, seg_rows, n_seg, grad_output, grad_input, batch, false, workspace, workspace_bytes, stream);
}

size_t aqlm_b200_matmat_dequant_routed_workspace_bytes(const aqlm_b200_weight_t* w, int n_experts, int64_t rows,
                                                       int transposed) {
  if (validate(w, false) != AQLM_B200_OK || rows <= 0 || n_experts < 1 || n_experts > kRoutedMaxExperts) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return 0;
  const GemmPlan g = gemm_routed_plan(*w, rows, n_experts, *di, tun(), true, transposed != 0);
  if (!g.ok || g.ksplit <= 1) return 0;
  return g.counters_bytes + g.partials_bytes;
}

int aqlm_b200_matmat_dequant_routed(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, int n_experts,
                                    const int32_t* expert_offsets, const void* input, void* output, int64_t rows,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  return routed_gemm<false>(w, seg_rows, n_seg, n_experts, expert_offsets, input, output, rows, workspace,
                            workspace_bytes, stream);
}

int aqlm_b200_matmat_dequant_transposed_routed(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                                               int n_experts, const int32_t* expert_offsets, const void* grad_output,
                                               void* grad_input, int64_t rows, void* workspace, size_t workspace_bytes,
                                               void* stream) {
  return routed_gemm<true>(w, seg_rows, n_seg, n_experts, expert_offsets, grad_output, grad_input, rows, workspace,
                           workspace_bytes, stream);
}

size_t aqlm_b200_matmat_weight_grad_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch) {
  if (validate(w, false) != AQLM_B200_OK || batch <= 0) return 0;
  const DeviceInfo* di = device_info();
  if (!di) return 0;
  const WgradPlan g = gemm_wgrad_plan(*w, batch, *di, tun());
  return g.ok ? g.counters_bytes + g.dots_bytes : 0;
}

int aqlm_b200_matmat_weight_grad(const aqlm_b200_weight_t* w, const void* input, const void* grad_output,
                                 int64_t batch, float* grad_codebooks, float* grad_scales, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  int rc = weight_grad_checks(w, input, grad_output, batch, grad_codebooks, grad_scales);
  if (rc || batch == 0) return rc;
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  const WgradPlan g = gemm_wgrad_plan(*w, batch, *di, tun());
  if (!g.ok) return fail(AQLM_B200_ERR_UNSUPPORTED, "weight gradient: no wgmma plan for this descriptor and batch");
  if (grad_scales && (!workspace || workspace_bytes < g.counters_bytes + g.dots_bytes))
    return fail(AQLM_B200_ERR_SHAPE, "weight gradient: grad_scales needs a workspace of %zu bytes, got %zu",
                g.counters_bytes + g.dots_bytes, workspace ? workspace_bytes : (size_t)0);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_dtype(w->dtype, [&](auto tag) {
    return with_gemm_scheme(w, [&](auto K, auto CB) {
      return launch_weight_grad<typename decltype(tag)::type, K, CB>(w, input, grad_output, batch, grad_codebooks,
                                                                     grad_scales, workspace, g, di, st);
    });
  });
}

int aqlm_b200_scale_bias(const float* partial, const void* scales, const void* bias, void* output, int64_t batch,
                         int64_t out_features, int32_t dtype, void* stream) {
  if (!partial || !scales || !output) return fail(AQLM_B200_ERR_SHAPE, "NULL pointer");
  if (dtype != AQLM_B200_F16 && dtype != AQLM_B200_BF16) return fail(AQLM_B200_ERR_DTYPE, "dtype must be f16/bf16");
  if (batch <= 0 || out_features <= 0) return AQLM_B200_OK;
  const DeviceInfo* di;
  if (int rc = current_device(&di)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = batch * out_features;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  with_dtype(dtype, [&](auto tag) {
    using T = typename decltype(tag)::type;
    scale_bias_kernel<T><<<blocks, 256, 0, st>>>(partial, (const T*)scales, (const T*)bias, (T*)output, batch,
                                                 out_features);
    return AQLM_B200_OK;
  });
  count_launch();
  AQLM_CUDA_CHECK(cudaGetLastError());
  return AQLM_B200_OK;
}

// ---- peer-memory all-reduce (multi-GPU sharded path) -----------------------------------------------
struct aqlm_b200_comm {
  int rank, world;
  long long max_elems;
  uint8_t* peer_base[kPeerMaxWorld];
  unsigned int* local_state;  // [0] step, [1..2] tickets
  float* local_partials;      // [max_elems]
};

size_t aqlm_b200_comm_shared_bytes(int world, int64_t max_elems) {
  if (world < 1 || world > kPeerMaxWorld || max_elems <= 0) return 0;
  // flags + [set][src][max_elems] fp32 slots (stand-alone exchange kernel) + [set][src][max_elems] tagged 64-bit words
  // (exchange fused into the GEMV)
  return (size_t)kPeerFlagBytes + (size_t)2 * world * (size_t)max_elems * (sizeof(float) + sizeof(unsigned long long));
}

int aqlm_b200_shared_alloc(size_t bytes, void** ptr, void* handle64) {
  if (!ptr || !handle64 || bytes == 0) return fail(AQLM_B200_ERR_SHAPE, "bad shared_alloc arguments");
  AQLM_CUDA_CHECK(cudaMalloc(ptr, bytes));
  AQLM_CUDA_CHECK(cudaMemset(*ptr, 0, bytes));
  AQLM_CUDA_CHECK(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  AQLM_CUDA_CHECK(cudaIpcGetMemHandle(&h, *ptr));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  return AQLM_B200_OK;
}

int aqlm_b200_shared_open(const void* handle64, void** ptr) {
  if (!ptr || !handle64) return fail(AQLM_B200_ERR_SHAPE, "bad shared_open arguments");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  AQLM_CUDA_CHECK(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return AQLM_B200_OK;
}

int aqlm_b200_comm_create(int rank, int world, void* const* peer_ptrs, int64_t max_elems, aqlm_b200_comm** out) {
  if (!out || !peer_ptrs || world < 1 || world > kPeerMaxWorld || rank < 0 || rank >= world || max_elems <= 0 || (max_elems & 3))
    return fail(AQLM_B200_ERR_SHAPE, "bad comm_create arguments");
  aqlm_b200_comm* c = new aqlm_b200_comm();
  c->rank = rank;
  c->world = world;
  c->max_elems = max_elems;
  for (int r = 0; r < world; ++r) c->peer_base[r] = reinterpret_cast<uint8_t*>(peer_ptrs[r]);
  AQLM_CUDA_CHECK(cudaMalloc(&c->local_state, 64));
  AQLM_CUDA_CHECK(cudaMemset(c->local_state, 0, 64));
  AQLM_CUDA_CHECK(cudaMalloc(&c->local_partials, (size_t)max_elems * sizeof(float)));
  AQLM_CUDA_CHECK(cudaDeviceSynchronize());
  *out = c;
  return AQLM_B200_OK;
}

void* aqlm_b200_comm_partials(aqlm_b200_comm* c) { return c ? c->local_partials : nullptr; }

int aqlm_b200_comm_destroy(aqlm_b200_comm* c) {
  if (!c) return AQLM_B200_OK;
  cudaFree(c->local_state);
  cudaFree(c->local_partials);
  delete c;
  return AQLM_B200_OK;
}

int aqlm_b200_allreduce_scale_bias(aqlm_b200_comm* c, const float* partial, const void* scales, const void* bias,
                                   void* output, int64_t batch, int64_t out_features, int32_t dtype, void* stream) {
  if (!c || !partial || !scales || !output) return fail(AQLM_B200_ERR_SHAPE, "NULL pointer");
  if (dtype != AQLM_B200_F16 && dtype != AQLM_B200_BF16) return fail(AQLM_B200_ERR_DTYPE, "dtype must be f16/bf16");
  if (batch <= 0 || out_features <= 0) return AQLM_B200_OK;
  if (out_features > c->max_elems || (out_features & 3))
    return fail(AQLM_B200_ERR_SHAPE, "allreduce: out_features %lld exceeds the communicator's %lld elements (or %% 4 != 0)",
                (long long)out_features, c->max_elems);
  const DeviceInfo* di;
  if (int rc = current_device(&di)) return rc;
  PeerParams p;
  for (int r = 0; r < kPeerMaxWorld; ++r) p.peer_base[r] = r < c->world ? c->peer_base[r] : nullptr;
  p.scales = scales;
  p.bias = bias;
  p.step = c->local_state;
  p.tickets = c->local_state + 1;
  p.max_elems = c->max_elems;
  p.out_features = (int)out_features;
  p.rank = c->rank;
  p.world = c->world;
  // A call larger than the communicator's slots runs as consecutive exchanges of whole rows, each one launch on a row
  // slice of `partial` and `output`.  Every rank derives the same chunking from max_elems (checked equal at
  // construction), so all ranks run the same number of steps.
  const int64_t chunk_rows = c->max_elems / out_features;
  for (int64_t b0 = 0; b0 < batch; b0 += chunk_rows) {
    const int64_t n = (batch - b0 < chunk_rows ? batch - b0 : chunk_rows) * out_features;
    p.local = partial + b0 * out_features;
    p.y = reinterpret_cast<uint8_t*>(output) + (size_t)(b0 * out_features) * 2;
    p.n = (int)n;
    int grid = (int)((n / 4 + kPeerThreads - 1) / kPeerThreads);
    if (grid > kPeerMaxCtas) grid = kPeerMaxCtas;  // one flag per (source rank, CTA slice); every rank derives the same grid from n
    if (grid < 1) grid = 1;
    const int rc = with_dtype(dtype, [&](auto tag) {
      return launch<peer_allreduce_epilogue_kernel<typename decltype(tag)::type>>(
          di, grid, kPeerThreads, 0, reinterpret_cast<cudaStream_t>(stream), 0, p);
    });
    if (rc) return rc;
  }
  return AQLM_B200_OK;
}

int aqlm_b200_matmat_allreduce(aqlm_b200_comm* c, const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                               const void* input, void* output, int64_t batch, void* stream) {
  if (!c) return fail(AQLM_B200_ERR_SHAPE, "communicator is NULL");
  int rc = validate(w, true);
  if (rc) return rc;
  if (w->num_codebooks != 1 || w->nbits_per_codebook != 16 || w->in_group_size != 8)
    return fail(AQLM_B200_ERR_UNSUPPORTED, "fused GEMV + exchange is implemented for the 1x16 (in_group 8) scheme");
  if (batch < 1 || batch > 8) return fail(AQLM_B200_ERR_UNSUPPORTED, "fused GEMV + exchange takes 1..8 batch rows");
  if (n_seg < 1 || n_seg > 4 || (n_seg > 1 && !seg_rows)) return fail(AQLM_B200_ERR_SHAPE, "1..4 segments");
  if (!input || !output) return fail(AQLM_B200_ERR_SHAPE, "input/output pointer is NULL");
  if ((w->out_features & 3) || batch * w->out_features > c->max_elems)
    return fail(AQLM_B200_ERR_SHAPE, "fused exchange: out_features %% 4 != 0 or batch*out_features exceeds the communicator's %lld",
                c->max_elems);
  const size_t row_bytes = (size_t)(w->in_features / 8) * 2;
  if (row_bytes % 16 != 0 || (reinterpret_cast<uintptr_t>(w->codes) & 15) || (reinterpret_cast<uintptr_t>(input) & 15))
    return fail(AQLM_B200_ERR_UNSUPPORTED, "fused exchange needs 16-byte aligned code rows and input");
  const DeviceInfo* di;
  if ((rc = current_device(&di))) return rc;
  GemvParams p = gemv_params(w, input, output, batch, false);
  p.n_seg = n_seg;
  int64_t acc = 0;
  for (int i = 0; i < 4; ++i) {
    if (i < n_seg) acc += (n_seg > 1 ? seg_rows[i] : w->out_features);
    p.seg_end[i] = (int)acc;
  }
  if (acc != w->out_features) return fail(AQLM_B200_ERR_SHAPE, "segment rows do not add up to out_features");
  GemvPeer pc;
  for (int r = 0; r < 16; ++r) pc.peer_base[r] = r < c->world ? c->peer_base[r] : nullptr;
  pc.step = c->local_state;
  pc.tickets = c->local_state + 1;
  pc.max_elems = c->max_elems;
  pc.rank = c->rank;
  pc.world = c->world;
  pc.ll_offset = (long long)kPeerFlagBytes + (long long)2 * c->world * c->max_elems * (long long)sizeof(float);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return with_batch_tile(batch, [&](auto BT) {
    return with_dtype(w->dtype, [&](auto tag) { return launch_1x16_peer<typename decltype(tag)::type, BT>(p, pc, di, st); });
  });
}

int aqlm_b200_matmat_host(const aqlm_b200_weight_t* w, const void* input_host, void* output_host, void* input_dev,
                          void* output_dev, int64_t batch, void* stream) {
  int rc = validate(w, true);
  if (rc) return rc;
  if (!input_host || !output_host || !input_dev || !output_dev) return fail(AQLM_B200_ERR_SHAPE, "NULL buffer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AQLM_CUDA_CHECK(cudaMemcpyAsync(input_dev, input_host, (size_t)batch * w->in_features * 2, cudaMemcpyHostToDevice, st));
  rc = aqlm_b200_matmat_ex(w, input_dev, output_dev, batch, 0, stream);
  if (rc) return rc;
  AQLM_CUDA_CHECK(cudaMemcpyAsync(output_host, output_dev, (size_t)batch * w->out_features * 2, cudaMemcpyDeviceToHost, st));
  AQLM_CUDA_CHECK(cudaStreamSynchronize(st));
  return AQLM_B200_OK;
}

// ---- flat wrappers ------------------------------------------------------------------------------
#define AQLM_FLAT_MATMAT(NAME, K, NBITS, GEXPR, FN)                                                               \
  aqlm_b200_weight_t w = make_weight(codes, codebooks, scales, bias, in_features, out_features, K, NBITS, GEXPR, dtype); \
  return FN(&w, input, output, batch, stream)

int aqlm_b200_code1x16_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                              const void* bias, void* output, int64_t batch, int64_t in_features,
                              int64_t out_features, int32_t in_group_size, int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code1x16_matmat, 1, 16, in_group_size, aqlm_b200_matmat);
}
int aqlm_b200_code2x8_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                             const void* bias, void* output, int64_t batch, int64_t in_features,
                             int64_t out_features, int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code2x8_matmat, 2, 8, 8, aqlm_b200_matmat);
}
int aqlm_b200_code1x8_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                             const void* bias, void* output, int64_t batch, int64_t in_features,
                             int64_t out_features, int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code1x8_matmat, 1, 8, 8, aqlm_b200_matmat);
}
int aqlm_b200_code1x16_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                      const void* scales, const void* bias, void* output, int64_t batch,
                                      int64_t in_features, int64_t out_features, int32_t in_group_size,
                                      int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code1x16_matmat_dequant, 1, 16, in_group_size, aqlm_b200_matmat_dequant);
}
int aqlm_b200_code2x8_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                     const void* scales, const void* bias, void* output, int64_t batch,
                                     int64_t in_features, int64_t out_features, int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code2x8_matmat_dequant, 2, 8, 8, aqlm_b200_matmat_dequant);
}
int aqlm_b200_code1x8_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                     const void* scales, const void* bias, void* output, int64_t batch,
                                     int64_t in_features, int64_t out_features, int32_t dtype, void* stream) {
  AQLM_FLAT_MATMAT(code1x8_matmat_dequant, 1, 8, 8, aqlm_b200_matmat_dequant);
}
#undef AQLM_FLAT_MATMAT

int aqlm_b200_code1x16_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                               int64_t in_features, int64_t out_features, int32_t in_group_size, int32_t dtype,
                               void* stream) {
  aqlm_b200_weight_t w = make_weight(codes, codebooks, scales, nullptr, in_features, out_features, 1, 16, in_group_size, dtype);
  return aqlm_b200_dequant(&w, weight_out, 1, stream);
}
int aqlm_b200_code2x8_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                              int64_t in_features, int64_t out_features, int32_t dtype, void* stream) {
  aqlm_b200_weight_t w = make_weight(codes, codebooks, scales, nullptr, in_features, out_features, 2, 8, 8, dtype);
  return aqlm_b200_dequant(&w, weight_out, 1, stream);
}
int aqlm_b200_code1x8_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                              int64_t in_features, int64_t out_features, int32_t dtype, void* stream) {
  aqlm_b200_weight_t w = make_weight(codes, codebooks, scales, nullptr, in_features, out_features, 1, 8, 8, dtype);
  return aqlm_b200_dequant(&w, weight_out, 1, stream);
}

}  // extern "C"
