// Internal interface between the C-ABI layer (api.cu) and the kernel translation units.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/vptq_b200.h"
#include "../../include/vptq_b200_grad.h"
#include "../../include/vptq_b200_graph.h"
#include "../../include/vptq_b200_batch.h"
#include "../../include/vptq_b200_lists_dense.h"
#include "../../include/vptq_b200_lists16.h"

namespace vptq_b200 {

struct DeviceInfo {
  int device = -1;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
  int smem_optin = 0;  // max dynamic shared memory per block (opt-in), bytes
  int l2_bytes = 0;
};
// cached per device; returns nullptr (and sets the error) on failure
const DeviceInfo* device_info();

void set_error(const char* fmt, ...);

static inline int ilog2(int64_t v) {
  int r = 0;
  while ((int64_t(1) << (r + 1)) <= v) ++r;
  return r;
}
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Workspace convention shared by every op: bytes [0, kZeroRegionBytes) are the ONLY part that must be zero
// at rest (kernels leave them zeroed): first kCounterRegionBytes of uint32 arrival / split-K row counters, then
// 64 bytes per index row of 64-bit fixed-point output accumulators (list-based decode GEMV).  Everything behind
// is scratch that each op overwrites before reading.  The region's extent is fixed so that it never depends on
// which layer used the workspace last.
constexpr int kMaxIndexRows = 65536;
constexpr size_t kCounterRegionBytes = size_t(kMaxIndexRows) * 4;
constexpr size_t kZeroRegionBytes = kCounterRegionBytes + size_t(kMaxIndexRows) * 64;

// -------------------------------------------------------------------------------------------
// decode GEMV
// -------------------------------------------------------------------------------------------
// How one launch is cut up.  Units of work are (index row r, column chunk); a CTA owns one
// chunk (so its x' slice and codebooks are staged once) and a strided subset of the rows; each
// of its warps owns whole rows, streams their packed index words through a private TMA ring and
// keeps the v partial sums in registers.
struct GemvPlan {
  int threads;         // CTA size (multiple of 32)
  int grid;            // nch * cpc
  int nch;             // column chunks in total = G * cpg
  int cpg;             // chunks per codebook group
  int chunk_cols;      // columns per chunk (multiple of 128 except possibly the group's last)
  int cpc;             // CTAs per chunk (rows are dealt round-robin to them)
  int seg_fields;      // index fields per ring stage (multiple of 128)
  int stages;          // ring depth per warp
  int main_in_smem;    // main codebook staged in shared memory (else gathered through L1/L2)
  int main_rep;        // bank-group replication factor of the main codebook in smem (1 or 8)
  int res_rep;         // same for the residual codebook; 0: not in shared memory, gathered through L1/L2
  int nt;              // tokens per pass (1, 2 or 4)
  int sx_stride;       // floats per token row of x' in smem
  int cluster;         // 1: the nch CTAs of a row set form a thread-block cluster (DSMEM split-K)
  int ctas_per_sm;     // co-resident CTAs per SM the plan was sized for
  int wsplit;          // warps sharing one row of the chunk (1, 2 or 4); their sums meet in smem
  int sub_cols;        // columns per warp sub-range (multiple of 128)
  uint32_t off_bars, off_cbias, off_pcol, off_wb, off_sx, off_part, off_wsum, off_wcnt, off_res, off_main, off_raw,
      off_ring;
  uint32_t stage_bytes;
  uint32_t smem_bytes;
  // workspace carve-up
  size_t ws_counters_bytes;  // fixed 256 KiB region of uint32 row counters (zero at rest)
  size_t ws_partials_bytes;  // nch * nt * Ro*v floats (only when nch > 1)
};

// Fills `plan` for (desc, tokens-per-pass).  Returns 0 or a vptq_status.
int gemv_make_plan(const vptq_linear_desc& d, int tokens, const DeviceInfo& dev, GemvPlan* plan, int slots_override = 0,
                   int force_cpg = 0);
int gemv_multi_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride, void* const* ys,
                      const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream,
                      const vptq_tp_exchange* tp = nullptr, void* workspace = nullptr, size_t workspace_bytes = 0);
void gemv_set_profile_buffer(void* dev_ptr);
unsigned long long* gemv_profile_buffer();
// Launches ceil(tokens / plan.nt) passes.
int gemv_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, void* y, int64_t y_stride,
                int tokens, void* workspace, size_t workspace_bytes, uint32_t flags, cudaStream_t stream);

// shared launch plumbing (gemv.cu)
int ensure_smem_attr(const void* fn, int bytes);  // opt in to `bytes` of dynamic shared memory, once per kernel
// how many clusters of `csize` CTAs (threads, smem each) the device can hold at once; <= 0: unknown
int max_active_clusters(const void* fn, int csize, int threads, int smem, int optin);
int gemv_tune_lists();  // developer knob VPTQ_B200_GEMV_TUNE="lists=0|1" (-1: not set)

// -------------------------------------------------------------------------------------------
// decode GEMV, list-based variant (gemv_lists.cu): one token, layers carrying the slice x tile lists of
// vptq_linear_desc::lists_*.  Every CTA keeps one or two 64 KiB slices of the main codebook in shared
// memory and walks the lists of its units: every codebook gather is a shared-memory access instead of an
// L1/L2 one; the per-combo partial sums meet in the workspace (arrival counters, last arriver writes y).
// -------------------------------------------------------------------------------------------
constexpr int kMaxFusedLayers = 4;
bool gemv_lists_eligible(const vptq_linear_desc& d);
// n layers reading the same x in one launch.  VPTQ_ERR_UNSUPPORTED / VPTQ_ERR_WORKSPACE: use the generic kernel.
int gemv_lists_launch(int n, const vptq_linear_desc* const* descs, const void* x, void* const* ys, uint32_t flags,
                      cudaStream_t stream, void* workspace, size_t workspace_bytes, const vptq_tp_exchange* tp = nullptr);
size_t gemv_lists_workspace_bytes(const vptq_linear_desc& d);  // 0 when the layer is not eligible
// tagged-word activation buffer of a VPTQ_TP_TAGGED launch -> plain 16-bit values (waits for the tags)
int tp_untag_launch(const void* tagged, void* y, int n, const vptq_tp_exchange& tp, cudaStream_t stream);

// Batched variant (gemv_lists_batch.cu, C interface include/vptq_b200_batch.h): 1..8 tokens of layers carrying
// the same lists, one combo per CTA, every token's sums independent of the others in the launch.
int gemv_lists_batch_max_tokens(int n, const vptq_linear_desc* const* descs);  // 0: not eligible (error set)
int gemv_lists_batch_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride,
                            void* const* ys, const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream,
                            void* workspace, size_t workspace_bytes);

// Vector-length-16 variant (gemv_lists16.cu, C interface include/vptq_b200_lists16.h): 1..4 tokens of layers
// carrying lists with index rows of 16 outputs, the batched kernel's partition, the slice as two shared planes.
bool gemv_lists16_eligible(const vptq_linear_desc& d);
int gemv_lists16_max_tokens(int n, const vptq_linear_desc* const* descs);  // 0: not eligible (error set)
int gemv_lists16_launch(int n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride, void* const* ys,
                        const int64_t* y_strides, int tokens, uint32_t flags, cudaStream_t stream, void* workspace,
                        size_t workspace_bytes);

// -------------------------------------------------------------------------------------------
// dequant
// -------------------------------------------------------------------------------------------
size_t dequant_workspace_bytes(const vptq_linear_desc& d);
// ld: elements between output rows (0 = in_features)
int dequant_launch(const vptq_linear_desc& d, void* w_out, void* workspace, size_t workspace_bytes,
                   cudaStream_t stream, int64_t ld = 0);
bool dequant_orig_fast_ok(const vptq_linear_desc& d, const void* w_out, int64_t ld);  // 8-columns-per-thread path applies
// Wt[f][o] = W[o][f], rows in original feature order, pitch ld (multiple of 8, >= out_features), columns [O, ld) zero
int dequant_transposed_launch(const vptq_linear_desc& d, void* wt_out, int64_t ld, cudaStream_t stream);

// the same W (transposed: Wt) from the index lists (lists_dense.cu, C interface include/vptq_b200_lists_dense.h):
// layers with gemv_lists_eligible(d), out 16-byte aligned, ld % 8 == 0, ld >= in_features (Wt: >= out_features)
int lists_dense_launch(const vptq_linear_desc& d, void* out, int64_t ld, bool transposed, cudaStream_t stream);

// -------------------------------------------------------------------------------------------
// prefill GEMM (wgmma)
// -------------------------------------------------------------------------------------------
size_t gemm_workspace_bytes(const vptq_linear_desc& d, int tokens);
int gemm_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, void* y, int64_t y_stride,
                int tokens, void* workspace, size_t workspace_bytes, uint32_t flags, cudaStream_t stream);
// input gradient dx[T][I] = dy[T][O] . W (no bias): transposed dequant + the same wgmma GEMM
size_t dgrad_workspace_bytes(const vptq_linear_desc& d, int tokens);
int dgrad_launch(const vptq_linear_desc& d, const void* dy, int64_t dy_stride, void* dx, int64_t dx_stride, int tokens,
                 void* workspace, size_t workspace_bytes, cudaStream_t stream);
// prefill (transposed: input gradient) with W (Wt) written from the index lists instead of the packed words
size_t lists_gemm_workspace_bytes(const vptq_linear_desc& d, int tokens, bool transposed);
int lists_gemm_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, void* y, int64_t y_stride, int tokens,
                      void* workspace, size_t workspace_bytes, bool transposed, cudaStream_t stream);
// gamma[M][ld] (fp32, unrounded) = A[M][K] . B[N][K]^T with both operands K-major, K % 64 == 0, N and ld even
int wgrad_gamma_launch(int is_bf16, const void* a, const void* b, int M, int N, int K, float* gamma, int64_t ld,
                       cudaStream_t stream);

// Per-call state of the weight-gradient reduction (wgrad.cu), in the workspace.
struct WgHeader {
  int e_cb, e_bias, e_scale;       // fixed-point value q stands for q * 2^e
  int nonfinite;                   // 1: some input value (or an fp32 element of G) was inf / NaN
  uint32_t max_c, max_r, max_col;  // bit patterns of max |C|, |R|, |Col| (non-negative floats order like integers)
};

// Fused weight-gradient epilogue of the wgmma GEMM (G = dY^T x' with M = out_features, N = in_features in
// quantised column order): v = 8, one codebook group, no outlier columns, Kr <= 256.  Every accumulator element
// goes straight into the fixed-point sums; G is never stored.
struct WgradEpilogue {
  const uint32_t* indices;
  int64_t idx_stride_r;
  const void* centroids;
  const void* res_centroids;
  const void* scale_q;      // weight_scale in quantised column order, or nullptr (then scale[perm[c]])
  const void* scale;        // weight_scale [I] or nullptr
  const uint16_t* perm;     // or nullptr
  unsigned long long *acc_c, *acc_r, *acc_s, *acc_b;  // nullptr: not wanted
  WgHeader* hdr;
  int I, ib, rb;
  int res_table;            // entries of the per-CTA shared-memory dR table (Kr * 8), 0: dR not wanted
};
int wgrad_fused_launch(int is_bf16, const void* a, const void* b, int M, int N, int K, const WgradEpilogue& e,
                       cudaStream_t stream);

// -------------------------------------------------------------------------------------------
// weight gradients (wgrad.cu, C interface include/vptq_b200_grad.h)
// -------------------------------------------------------------------------------------------
size_t wgrad_workspace_bytes(const vptq_linear_desc& d, int tokens, int op);
int wgrad_launch(const vptq_linear_desc& d, const void* x, int64_t x_stride, const void* dy, int64_t dy_stride,
                 int tokens, const vptq_linear_grads& g, void* workspace, size_t workspace_bytes, uint32_t flags,
                 cudaStream_t stream);
int dequant_backward_launch(const vptq_linear_desc& d, const void* dw, int64_t dw_stride, const vptq_linear_grads& g,
                            void* workspace, size_t workspace_bytes, cudaStream_t stream);

// -------------------------------------------------------------------------------------------
// v2 GEMV (unpacked indices)
// -------------------------------------------------------------------------------------------
struct GemvV2Args {
  int dtype, tokens, in_features, out_features, vector_len, num_centroids, num_res_centroids;
  const void* x;
  void* y;
  const uint16_t* indices;
  const void* centroids;
  const void* residual_indices;
  int res_index_bytes;
  const void* residual_centroids;
  const void* scale_weights;
  const void* scale_bias;
  const void* bias;
};
size_t gemv_v2_workspace_bytes(int tokens, int in_features, int out_features, int vector_len);
int gemv_v2_launch(const GemvV2Args& a, void* workspace, size_t workspace_bytes, uint32_t flags,
                   cudaStream_t stream);

}  // namespace vptq_b200
