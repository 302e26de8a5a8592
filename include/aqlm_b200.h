/*
 * aqlm_b200 -- C-ABI of the H100-native (sm_90a) AQLM quantized-linear hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  Every entry point takes plain device (or,
 * for *_host, pinned host) pointers, sizes and a CUstream/cudaStream_t passed as `void*`; no torch types.
 * Each function returns an aqlm_b200_status; on failure aqlm_b200_last_error() returns a message for
 * the calling thread.  Kernels never allocate or free: the caller owns every buffer, and nothing is
 * kept between calls (reference ownership model, cuda_kernel.cpp:159-163).  All launches go to the
 * stream given and are CUDA-graph capturable.
 *
 * Reference citations are relative to /root/reference/inference_lib/src/aqlm/inference_kernels/.
 *
 * Tensor layouts (identical to the reference module, inference.py:39-61):
 *   codes      [out_features, in_groups, num_codebooks]   int8 (nbits<=8) | int16 (nbits<=16), two's-complement
 *              storage of UNSIGNED codes (utils.py:23-31) -- kernels reinterpret, never sign-extend
 *   codebooks  [num_codebooks, 2^nbits, 1, in_group_size]  f16 | bf16
 *   scales     [out_features] (the module's [out,1,1,1])  f16 | bf16
 *   bias       [out_features] or NULL                      f16 | bf16
 *   input      [batch, in_features] row-major              f16 | bf16
 *   output     [batch, out_features] row-major             f16 | bf16 (or f32 partials, see flags)
 */
#ifndef AQLM_B200_H_
#define AQLM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AQLM_B200_VERSION 100 /* 0.1.0 */

typedef enum {
  AQLM_B200_OK = 0,
  AQLM_B200_ERR_DTYPE = 1,       /* not f16/bf16 -> NotImplementedError (cuda_kernel.cpp:9-25) */
  AQLM_B200_ERR_UNSUPPORTED = 2, /* scheme/group size not implemented -> NotImplementedError (cuda_kernel.cpp:137-144) */
  AQLM_B200_ERR_SHAPE = 3,       /* inconsistent sizes / misaligned pointers -> ValueError */
  AQLM_B200_ERR_CUDA = 4,        /* CUDA runtime error (the reference never checks; we do) -> RuntimeError */
  AQLM_B200_ERR_ARCH = 5         /* device is not sm_90 -> RuntimeError */
} aqlm_b200_status;

typedef enum { AQLM_B200_F16 = 0, AQLM_B200_BF16 = 1 } aqlm_b200_dtype;

/* flags for aqlm_b200_matmat_ex, aqlm_b200_matmat_ws and aqlm_b200_matmat_dequant_ex */
#define AQLM_B200_FLAG_PARTIAL_F32 1u /* write UNSCALED fp32 partial sums (no scale, no bias): the per-rank
                                          result of an in_features-sharded matvec, to be all-reduced */

/* One quantized weight matrix (all pointers are device pointers). */
typedef struct {
  const void* codes;
  const void* codebooks;
  const void* scales; /* may be NULL only with AQLM_B200_FLAG_PARTIAL_F32 */
  const void* bias;   /* NULL = no bias (Llama) */
  int64_t in_features;
  int64_t out_features;
  int32_t num_codebooks;
  int32_t nbits_per_codebook;
  int32_t in_group_size;  /* 8 or 16 */
  int32_t out_group_size; /* must be 1 (every reference CUDA kernel assumes it) */
  int32_t dtype;          /* aqlm_b200_dtype of codebooks/scales/bias/input/output */
  int32_t reserved;
} aqlm_b200_weight_t;

int aqlm_b200_version(void);
const char* aqlm_b200_last_error(void);
/* Number of kernels this library has launched in this process (bench.py's `gpu_launches`). */
uint64_t aqlm_b200_launch_count(void);
/* The AQLM_B200_* experiment switches (environment variables) are read once per process; tools that change the
 * environment at run time call this to re-read them.  Not needed in normal use. */
void aqlm_b200_reload_tunables(void);

/* ---- generic entry points -------------------------------------------------------------------- */

/* Fused code-gather + additive dequant + GEMV with the scale/bias epilogue in the same launch.
 * Replaces code1x16_matmat / code2x8_matmat / code1x8_matmat (cuda_kernel.cpp:148-182, 387-421,
 * 552-586: a host loop of one MatVec launch per batch row + 3-4 epilogue launches) and the Triton
 * path the reference uses for 8x8 (kernel_selector.py:91-94).  Any batch; intended for batch <= 6. */
int aqlm_b200_matmat(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, void* stream);
int aqlm_b200_matmat_ex(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                        void* stream);

/* Same with a caller-owned workspace (layout and zero-init contract as for aqlm_b200_matmat_dequant_ws below).  With a
 * workspace, batch-1 calls on 256-entry-codebook schemes (1x8, 2x8, 4x8, 8x8) use the dot-product-LUT kernel
 * (tensor-core-built LUT in shared memory, conflict-free 4-byte lookups) instead of per-code vector gathers. */
size_t aqlm_b200_matmat_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch);
int aqlm_b200_matmat_ws(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, uint32_t flags,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Grouped launch for several 1x16 linears that share the same input (q/k/v, gate/up): `w` describes the ROW-CONCATENATED
 * weights (codes [sum(seg_rows), in/8, 1], scales/bias [sum(seg_rows)]) and w->codebooks points to n_seg codebooks stacked
 * back to back (1 MiB each); output is [batch, sum(seg_rows)].  One launch instead of n_seg; batch <= 8.  New work (the
 * reference launches every linear separately); SURVEY §8f.2. */
int aqlm_b200_matmat_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* input,
                             void* output, int64_t batch, uint32_t flags, void* stream);

/* Fused dequant + tensor-core GEMM for large batch: W never goes to HBM.  Replaces
 * code{1x16,2x8,1x8}_matmat_dequant (cuda_kernel.cpp:249-301, 450-484, 615-649: Dequant kernel ->
 * full W in HBM -> cuBLAS F::linear -> epilogue). */
int aqlm_b200_matmat_dequant(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch, void* stream);
/* Same with a caller-owned workspace, which lets the kernel split the K dimension across otherwise idle SMs
 * (the reduction is deterministic).  The first aqlm_b200_matmat_dequant_workspace_bytes() bytes... the whole
 * workspace must be ZERO before the first use and is left zero-initialised where it matters (tile counters),
 * so one persistent buffer per stream can be reused without memsets.  The size depends on the shape, the scheme and the
 * batch only: w->scales may be NULL here (as for a call with AQLM_B200_FLAG_PARTIAL_F32). */
size_t aqlm_b200_matmat_dequant_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch);
int aqlm_b200_matmat_dequant_ws(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch,
                                void* workspace, size_t workspace_bytes, void* stream);
/* Same with flags.  AQLM_B200_FLAG_PARTIAL_F32: `output` is fp32 [batch, out_features] and receives the UNSCALED sums
 * (scales and bias may be NULL and are ignored), as from aqlm_b200_matmat_ex -- the large-batch (prefill) form of an
 * in_features-sharded linear's partial product.  Layouts the tensor-core kernel does not cover (in_group_size 16,
 * in_features % 64 != 0, other KxN, an input that is not 16-byte aligned) run as aqlm_b200_matmat_ex with the same
 * flags.  aqlm_b200_matmat_dequant_ws is this call with flags = 0. */
int aqlm_b200_matmat_dequant_ex(const aqlm_b200_weight_t* w, const void* input, void* output, int64_t batch,
                                uint32_t flags, void* workspace, size_t workspace_bytes, void* stream);

/* Materialise W [out_features, in_features] (x scales when apply_scales != 0).  Replaces
 * code{1x16,2x8,1x8}_dequant (cuda_kernel.cpp:184-227, 423-448, 588-613). */
int aqlm_b200_dequant(const aqlm_b200_weight_t* w, void* weight_out, int apply_scales, void* stream);

/* Backward w.r.t. the input, fused: grad_input[batch, in] = (grad_output[batch, out] * scales) @ W_unscaled, with W
 * dequantized on chip (MN-major A tile, wgmma, scale folded into the tile) -- W never goes to HBM and no library
 * GEMM is involved.  Replaces code*_matmat_dequant_transposed (cuda_kernel.cpp:303-354, 486-519, 651-684: Dequant
 * kernel -> full W in HBM -> cuBLAS), with the 2x8/1x8 unscaled-input defect (cuda_kernel.cpp:497,518,662,683) NOT
 * reproduced.  The optional workspace (same zero-init contract as aqlm_b200_matmat_dequant_ws) enables split-K over the
 * out rows.  Returns AQLM_B200_ERR_UNSUPPORTED for layouts the fused kernel does not cover (in_group_size 16, ...). */
size_t aqlm_b200_matmat_dequant_transposed_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch);
int aqlm_b200_matmat_dequant_transposed(const aqlm_b200_weight_t* w, const void* grad_output, void* grad_input,
                                        int64_t batch, void* workspace, size_t workspace_bytes, void* stream);

/* Grouped form of the two tensor-core GEMMs above, for linears that share their input (q/k/v, gate/up) at any batch:
 * ONE launch over the row-concatenated weight.  `w`, `seg_rows` and `n_seg` describe the group as for
 * aqlm_b200_matmat_grouped: codes [sum(seg_rows), in/in_group, K], scales/bias [sum(seg_rows)], and w->codebooks
 * points to n_seg codebook sets stacked back to back (K * 2^nbits * 8 elements each).  The plan is the one of the
 * concatenated descriptor, so aqlm_b200_matmat_dequant[_transposed]_workspace_bytes(w, batch) gives the workspace.
 *   forward:     output [batch, sum(seg_rows)]; flags as for aqlm_b200_matmat_dequant_ex (AQLM_B200_FLAG_PARTIAL_F32:
 *                fp32 unscaled sums, scales/bias may be NULL).
 *   transposed:  grad_input [batch, in] = (grad_output [batch, sum(seg_rows)] * scales) @ W_concatenated.
 * Any scheme the tensor-core kernels cover: in_group_size 8, 8/16-bit codes, 1/2/4/8 codebooks, 16-byte aligned code
 * rows and input, and in_features % 64 == 0 (forward) or out_features % 8 == 0 (transposed).  Anything else returns
 * AQLM_B200_ERR_UNSUPPORTED: unlike aqlm_b200_matmat_dequant_ex there is no GEMV form to fall back to, so the caller
 * runs the members one by one.  n_seg outside 1..4, an empty segment, or rows that do not add up to out_features:
 * AQLM_B200_ERR_SHAPE.  Both checks come before any device query. */
int aqlm_b200_matmat_dequant_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, const void* input,
                                     void* output, int64_t batch, uint32_t flags, void* workspace, size_t workspace_bytes,
                                     void* stream);
int aqlm_b200_matmat_dequant_transposed_grouped(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                                                const void* grad_output, void* grad_input, int64_t batch, void* workspace,
                                                size_t workspace_bytes, void* stream);

/* Routed form of the two tensor-core GEMMs, for a mixture-of-experts projection: n_experts experts of one shape in ONE
 * launch, each applied to its own run of rows.  `w` describes ONE expert (out_features = sum(seg_rows)), and its
 * pointers point at the stacks of all experts: codes [E][out][in/8][K], codebooks [E][n_seg][K][2^nbits][8], scales and
 * bias [E][out].  `seg_rows` / `n_seg` split each expert's rows as for the grouped GEMM (Mixtral's w1|w3 pair: n_seg 2);
 * seg_rows == NULL with n_seg == 1 is a plain expert linear.
 *   forward:     output[r] = input[r] . W_e^T * scales_e + bias_e  for the expert e that owns row r;
 *                input [rows, in], output [rows, out]
 *   transposed:  grad_input[r] = (grad_output[r] * scales_e) . W_e;  grad_output [rows, out], grad_input [rows, in]
 * `expert_offsets` is a DEVICE int32 array [n_experts + 1]: expert e owns rows [off[e], off[e+1]), so the rows must be
 * sorted by expert.  The host never reads it: the call is capturable in a CUDA graph, and the routing may change between
 * replays.  The offsets are not trusted: each is clamped into [0, rows] and raised to its predecessor (a decreasing pair
 * is an empty expert), and rows outside [off[0], off[E]) are neither read for output nor written (their output rows keep
 * whatever they held).  The workspace (split-K) comes from aqlm_b200_matmat_dequant_routed_workspace_bytes; without it
 * the call runs unsplit.  Errors, before any device query: AQLM_B200_ERR_SHAPE for a bad descriptor, n_seg outside 1..4,
 * segments that do not add up to out_features, n_experts outside 1..64, or NULL offsets / buffers;
 * AQLM_B200_ERR_UNSUPPORTED for layouts the wgmma kernels do not take (as for the grouped GEMM).  rows == 0: OK, no
 * launch.  Exactly one launch otherwise. */
size_t aqlm_b200_matmat_dequant_routed_workspace_bytes(const aqlm_b200_weight_t* w, int n_experts, int64_t rows,
                                                       int transposed);
int aqlm_b200_matmat_dequant_routed(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg, int n_experts,
                                    const int32_t* expert_offsets, const void* input, void* output, int64_t rows,
                                    void* workspace, size_t workspace_bytes, void* stream);
int aqlm_b200_matmat_dequant_transposed_routed(const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                                               int n_experts, const int32_t* expert_offsets, const void* grad_output,
                                               void* grad_input, int64_t rows, void* workspace, size_t workspace_bytes,
                                               void* stream);

/* ---- weight gradient: the gradients of a linear's codebooks and scales in ONE fused wgmma GEMM ----------------
 * With D = grad_output^T . input [out, in] (fp32) and Wu the unscaled weight as the forward computes it:
 *   grad_codebooks[k][c][i] += sum over (r, g) with code(r, g, k) = c of scales[r] * D[r, 8 g + i]
 *   grad_scales[r]           = sum_j D[r, j] * Wu[r, j]
 * input [batch, in] and grad_output [batch, out] in w->dtype.  grad_codebooks is fp32 [K][2^nbits][8] and the call ADDS
 * into it (the caller zeroes it, or accumulates); grad_scales is fp32 [out] and is WRITTEN.  Either may be NULL (not
 * wanted), not both; w->scales is required with grad_codebooks.  grad_scales needs the workspace of
 * aqlm_b200_matmat_weight_grad_workspace_bytes (counters, left at zero, and per-tile row dots).  grad_scales is
 * deterministic; grad_codebooks is summed in atomic arrival order (fp32, denormals flushed), so its last bits can
 * differ from run to run.  Errors, before any device query: AQLM_B200_ERR_SHAPE for a bad descriptor, NULL input /
 * grad_output or both outputs NULL; AQLM_B200_ERR_UNSUPPORTED for layouts the kernel does not take (in_group 16,
 * codebook counts other than 1/2/4/8, codes other than 8/16-bit, code rows not 16-byte aligned, out_features % 8 != 0,
 * input or grad_output not 16-byte aligned).  batch == 0: OK, no launch.  Exactly one launch otherwise. */
size_t aqlm_b200_matmat_weight_grad_workspace_bytes(const aqlm_b200_weight_t* w, int64_t batch);
int aqlm_b200_matmat_weight_grad(const aqlm_b200_weight_t* w, const void* input, const void* grad_output,
                                 int64_t batch, float* grad_codebooks, float* grad_scales, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* Epilogue of the sharded path: output[b,o] = (T)(partial[b,o] * scales[o] + bias[o]) after the
 * all-reduce of the fp32 partials (new work; the reference has no multi-GPU hot path, SURVEY §8e). */
int aqlm_b200_scale_bias(const float* partial, const void* scales, const void* bias, void* output, int64_t batch,
                         int64_t out_features, int32_t dtype, void* stream);

/* ---- multi-GPU: one-shot all-reduce over NVLink peer memory, fused with the epilogue ------------------------
 * One process per GPU.  Each rank allocates a shared buffer of aqlm_b200_comm_shared_bytes() with
 * aqlm_b200_shared_alloc (cudaMalloc + cudaIpcGetMemHandle; the 64-byte handle is exchanged out of band, e.g. with
 * torch.distributed.all_gather_object), opens every peer's handle with aqlm_b200_shared_open, and builds a communicator
 * from the W mapped pointers (peer_ptrs[rank] = its own buffer).  aqlm_b200_allreduce_scale_bias then does, in ONE
 * kernel: push my fp32 partials into every peer's buffer (P2P stores), publish a release flag, wait for all W flags,
 * add the W partials in rank order, apply scale + bias, write `output`.  Every rank must call it the same number of
 * times in the same order, and every rank's communicator must have the same max_elems.  A call with
 * batch*out_features > max_elems runs as consecutive exchanges of max_elems / out_features whole rows each (one kernel
 * launch apiece); out_features itself must not exceed max_elems.  For aqlm_b200_matmat_allreduce below, max_elems
 * bounds batch*out_features of any call. */
typedef struct aqlm_b200_comm aqlm_b200_comm;
size_t aqlm_b200_comm_shared_bytes(int world, int64_t max_elems);
int aqlm_b200_shared_alloc(size_t bytes, void** ptr, void* handle64);
int aqlm_b200_shared_open(const void* handle64, void** ptr);
int aqlm_b200_comm_create(int rank, int world, void* const* peer_ptrs, int64_t max_elems, aqlm_b200_comm** out);
void* aqlm_b200_comm_partials(aqlm_b200_comm* comm); /* a device buffer of max_elems floats owned by the communicator */
int aqlm_b200_comm_destroy(aqlm_b200_comm* comm);
int aqlm_b200_allreduce_scale_bias(aqlm_b200_comm* comm, const float* partial, const void* scales, const void* bias,
                                   void* output, int64_t batch, int64_t out_features, int32_t dtype, void* stream);

/* The sharded linear as ONE kernel (1x16, in_group 8, batch <= 8): fused code-gather + dequant + GEMV on this rank's
 * in_features shard whose reduction epilogue performs the exchange over NVLink peer memory: every (row, batch) element
 * travels as one tagged 64-bit word {fp32 partial, step} stored into slot [step & 1][this rank] of EVERY rank's buffer
 * (8-byte P2P stores, coalesced per warp); the same thread then polls the W words of that element in its OWN buffer until
 * their tags equal the step, adds them in rank order (deterministic) and applies scale + bias -- no fence, flag or barrier
 * between push and reduction.  `w` describes the SHARD (in_features = local slice) with full-length scales/bias;
 * `seg_rows`/`n_seg` as in aqlm_b200_matmat_grouped (n_seg == 1: a plain linear, seg_rows may be NULL).  Every rank must
 * call it the same number of times in the same order (it shares the step counter with aqlm_b200_allreduce_scale_bias);
 * the grid is one CTA per SM so that all ranks' CTAs are resident while they wait for each other. */
int aqlm_b200_matmat_allreduce(aqlm_b200_comm* comm, const aqlm_b200_weight_t* w, const int64_t* seg_rows, int n_seg,
                               const void* input, void* output, int64_t batch, void* stream);

/* End-to-end variant with HOST buffers (pinned): H2D copy of `input_host` into `input_dev`, the fused
 * matmat, D2H copy of the result into `output_host`, and a stream synchronize.  `input_dev`/`output_dev`
 * are caller-owned device scratch of batch*in_features / batch*out_features elements. */
int aqlm_b200_matmat_host(const aqlm_b200_weight_t* w, const void* input_host, void* output_host, void* input_dev,
                          void* output_dev, int64_t batch, void* stream);

/* ---- flat wrappers named after the reference's pybind functions (cuda_kernel.cpp:686-699) ------
 * input [batch,in], codes, codebooks, scales, bias (nullable), output [batch,out]. */
int aqlm_b200_code1x16_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                              const void* bias, void* output, int64_t batch, int64_t in_features,
                              int64_t out_features, int32_t in_group_size, int32_t dtype, void* stream);
int aqlm_b200_code2x8_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                             const void* bias, void* output, int64_t batch, int64_t in_features,
                             int64_t out_features, int32_t dtype, void* stream);
int aqlm_b200_code1x8_matmat(const void* input, const void* codes, const void* codebooks, const void* scales,
                             const void* bias, void* output, int64_t batch, int64_t in_features,
                             int64_t out_features, int32_t dtype, void* stream);
int aqlm_b200_code1x16_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                      const void* scales, const void* bias, void* output, int64_t batch,
                                      int64_t in_features, int64_t out_features, int32_t in_group_size,
                                      int32_t dtype, void* stream);
int aqlm_b200_code2x8_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                     const void* scales, const void* bias, void* output, int64_t batch,
                                     int64_t in_features, int64_t out_features, int32_t dtype, void* stream);
int aqlm_b200_code1x8_matmat_dequant(const void* input, const void* codes, const void* codebooks,
                                     const void* scales, const void* bias, void* output, int64_t batch,
                                     int64_t in_features, int64_t out_features, int32_t dtype, void* stream);
int aqlm_b200_code1x16_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                               int64_t in_features, int64_t out_features, int32_t in_group_size, int32_t dtype,
                               void* stream);
int aqlm_b200_code2x8_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                              int64_t in_features, int64_t out_features, int32_t dtype, void* stream);
int aqlm_b200_code1x8_dequant(const void* codes, const void* codebooks, const void* scales, void* weight_out,
                              int64_t in_features, int64_t out_features, int32_t dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AQLM_B200_H_ */
