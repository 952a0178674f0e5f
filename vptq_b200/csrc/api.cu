// extern "C" surface of libvptq_b200.so: argument validation, error reporting, dispatch.
// Declarations and the mapping to the reference's pybind11 functions: include/vptq_b200.h.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "kernels.h"

namespace vptq_b200 {

namespace {
thread_local char g_error[1024] = "";
std::mutex g_dev_mutex;
DeviceInfo g_dev[64];
}  // namespace

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

const DeviceInfo* device_info() {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess || dev < 0 || dev >= 64) {
    set_error("cudaGetDevice: %s", cudaGetErrorString(e));
    return nullptr;
  }
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  DeviceInfo& d = g_dev[dev];
  if (d.device == dev) return &d;
  int v = 0;
  cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev);
  d.l2_bytes = v;
  d.device = dev;
  return &d;
}

namespace {

bool is_pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

int check_device() {
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  if (dev->cc_major != 9 || dev->cc_minor != 0) {
    set_error("device compute capability %d.%d: this library contains sm_90a code only", dev->cc_major,
              dev->cc_minor);
    return VPTQ_ERR_DEVICE;
  }
  return 0;
}

// Mirrors the reference's argument checks (csrc/quant_gemv.cu:252-282, csrc/dequant.cu:238-275,
// vptq/layers/vqlinear.py:77-81,128-146) as explicit return codes.
int validate(const vptq_linear_desc* d, bool need_device) {
  if (!d) {
    set_error("desc is NULL");
    return VPTQ_ERR_INVALID;
  }
  if (d->struct_size != sizeof(vptq_linear_desc)) {
    set_error("desc.struct_size %u != %zu (ABI mismatch)", d->struct_size, sizeof(vptq_linear_desc));
    return VPTQ_ERR_INVALID;
  }
  if (d->dtype != VPTQ_FP16 && d->dtype != VPTQ_BF16) {
    set_error("dtype %d: only fp16 (0) and bf16 (1) are supported", d->dtype);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (d->in_features <= 0 || d->out_features <= 0 || d->in_features > 65535) {
    set_error("in_features=%d out_features=%d out of range (perm is uint16: in_features <= 65535)",
              d->in_features, d->out_features);
    return VPTQ_ERR_INVALID;
  }
  if (d->vector_len < 2 || d->vector_len > 16 || (d->vector_len & 1)) {
    set_error("vector_len %d must be even and in [2,16]", d->vector_len);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!is_pow2(d->num_centroids) || d->num_centroids > 65536 || d->num_centroids < 2) {
    set_error("num_centroids %d must be a power of two in [2,65536]", d->num_centroids);
    return VPTQ_ERR_UNSUPPORTED;
  }
  // (a single residual entry would need 0 index bits: the packed format cannot tell it from "no residual", so it is
  // refused rather than added to some weights and not to others)
  if (d->num_res_centroids > 0 &&
      (!is_pow2(d->num_res_centroids) || d->num_res_centroids > 65536 || d->num_res_centroids < 2)) {
    set_error("num_res_centroids %d must be a power of two in [2,65536] (or <= 0: no residual)", d->num_res_centroids);
    return VPTQ_ERR_UNSUPPORTED;
  }
  const int ib = ilog2(d->num_centroids);
  const int rb = d->num_res_centroids > 0 ? ilog2(d->num_res_centroids) : 0;
  if (ib + rb > 32) {
    set_error("index_bits %d + res_index_bits %d > 32 (vptq/utils/pack.py:34-37)", ib, rb);
    return VPTQ_ERR_INVALID;
  }
  if (d->num_codebooks <= 0 || d->group_size <= 0) {
    set_error("num_codebooks=%d group_size=%d must be positive", d->num_codebooks, d->group_size);
    return VPTQ_ERR_INVALID;
  }
  const bool outl = d->outlier_size > 0 && d->outlier_indices != nullptr;
  const int S = outl ? d->outlier_size : 0;
  if (int64_t(S) + int64_t(d->num_codebooks) * d->group_size != d->in_features) {
    set_error("outlier_size %d + num_codebooks %d * group_size %d != in_features %d", S, d->num_codebooks,
              d->group_size, d->in_features);
    return VPTQ_ERR_INVALID;
  }
  if (outl) {
    if (!d->outlier_centroids || d->outlier_vector_len < 1 || d->num_outlier_centroids < 1 ||
        d->num_outlier_centroids > 65536) {
      set_error("outliers enabled but outlier_centroids/outlier_vector_len/num_outlier_centroids invalid");
      return VPTQ_ERR_INVALID;
    }
  }
  // `indices` may be NULL for a decode-only descriptor that carries the index lists instead (the packed words were
  // dropped after the lists were built): only single-token GEMV calls are possible then
  if ((!d->indices && !(d->lists_stream && d->lists_tab)) || !d->centroids) {
    set_error("indices (or the index lists) / centroids must not be NULL");
    return VPTQ_ERR_INVALID;
  }
  if (rb && !d->res_centroids) {
    set_error("num_res_centroids=%d but res_centroids is NULL", d->num_res_centroids);
    return VPTQ_ERR_INVALID;
  }
  if ((d->weight_scale == nullptr) != (d->weight_bias == nullptr)) {
    set_error("weight_scale and weight_bias must both be given or both be NULL");
    return VPTQ_ERR_INVALID;
  }
  const int64_t wd = (int64_t(d->group_size) * (ib + rb) + 31) / 32;
  if (d->indices && d->index_stride_row < wd) {
    set_error("index_stride_row %lld < %lld packed words per row", (long long)d->index_stride_row, (long long)wd);
    return VPTQ_ERR_INVALID;
  }
  if (d->centroid_stride < int64_t(d->num_centroids) * d->vector_len ||
      (rb && d->res_centroid_stride < int64_t(d->num_res_centroids) * d->vector_len)) {
    set_error("centroid stride smaller than one codebook");
    return VPTQ_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(d->indices) & 3u) || (reinterpret_cast<uintptr_t>(d->centroids) & 15u) ||
      (reinterpret_cast<uintptr_t>(d->res_centroids) & 15u) ||
      ((d->centroid_stride * 2) & 15) || (rb && ((d->res_centroid_stride * 2) & 15) && d->num_codebooks > 1)) {
    set_error("centroids must be 16-byte aligned (per codebook), indices 4-byte aligned");
    return VPTQ_ERR_INVALID;
  }
  return need_device ? check_device() : 0;
}

int need_packed(const vptq_linear_desc* d, const char* what) {
  if (d->indices) return 0;
  set_error("%s needs the packed index words, but this descriptor is decode-only (indices == NULL, index lists only)", what);
  return VPTQ_ERR_UNSUPPORTED;
}

// the gradient outputs must match tensors the layer has, 16-bit aligned
int validate_grads(const vptq_linear_desc* d, const vptq_linear_grads* g, uint32_t flags, uint32_t allowed_flags,
                   const char* what) {
  if (!g || g->struct_size != sizeof(vptq_linear_grads) || g->reserved != 0) {
    set_error("%s: grads is NULL or its struct_size / reserved field is wrong (ABI mismatch)", what);
    return VPTQ_ERR_INVALID;
  }
  if (flags & ~allowed_flags) {
    set_error("%s: unknown flags 0x%x", what, flags);
    return VPTQ_ERR_INVALID;
  }
  const bool outl = d->outlier_size > 0 && d->outlier_indices != nullptr;
  if ((g->res_centroids && d->num_res_centroids <= 0) || (g->outlier_centroids && !outl) ||
      ((g->weight_scale || g->weight_bias) && !d->weight_scale)) {
    set_error("%s: a gradient was requested for a tensor this layer does not have", what);
    return VPTQ_ERR_INVALID;
  }
  for (const void* p : {g->centroids, g->res_centroids, g->outlier_centroids, g->weight_scale, g->weight_bias})
    if (reinterpret_cast<uintptr_t>(p) & 1u) {
      set_error("%s: gradient outputs must be 2-byte aligned", what);
      return VPTQ_ERR_INVALID;
    }
  return 0;
}

}  // namespace
}  // namespace vptq_b200

using namespace vptq_b200;

extern "C" {

int vptq_b200_abi_version(void) { return VPTQ_B200_ABI_VERSION; }

void vptq_b200_debug_phase_stamps(void* device_buffer) { gemv_set_profile_buffer(device_buffer); }

const char* vptq_b200_last_error(void) { return g_error; }

size_t vptq_b200_workspace_bytes(const vptq_linear_desc* desc, int32_t tokens, int32_t op) {
  if (validate(desc, false)) return 0;
  if (tokens < 1) tokens = 1;
  switch (op) {
    case VPTQ_OP_GEMV: {
      if (!desc->indices) return gemv_lists_workspace_bytes(*desc);
      // exact for the current device; without one (CPU-only host) the H100 SXM geometry is assumed
      DeviceInfo h100;
      h100.sm_count = 132, h100.smem_optin = 232448, h100.cc_major = 9;
      const DeviceInfo* dev = device_info();
      GemvPlan pl;
      if (gemv_make_plan(*desc, tokens, dev ? *dev : h100, &pl)) return 0;
      return std::max(pl.ws_counters_bytes + pl.ws_partials_bytes, gemv_lists_workspace_bytes(*desc));
    }
    case VPTQ_OP_DEQUANT: return dequant_workspace_bytes(*desc);
    case VPTQ_OP_GEMM: return gemm_workspace_bytes(*desc, tokens);
    case VPTQ_OP_GEMM_DGRAD: return dgrad_workspace_bytes(*desc, tokens);
    default: set_error("workspace_bytes: unknown op %d", op); return 0;
  }
}

int vptq_b200_quant_gemv(const vptq_linear_desc* desc, const void* x, int64_t x_stride, void* y,
                         int64_t y_stride, int32_t tokens, void* workspace, size_t workspace_bytes,
                         uint32_t flags, void* stream) {
  if (int rc = validate(desc, true)) return rc;
  if (!x || !y || tokens < 1 || x_stride < desc->in_features || y_stride < desc->out_features) {
    set_error("quant_gemv: bad x/y/tokens/strides (tokens=%d x_stride=%lld y_stride=%lld)", tokens,
              (long long)x_stride, (long long)y_stride);
    return VPTQ_ERR_INVALID;
  }
  return gemv_launch(*desc, x, x_stride, y, y_stride, tokens, workspace, workspace_bytes, flags,
                     static_cast<cudaStream_t>(stream));
}

int vptq_b200_quant_gemv_multi(int32_t n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride,
                               void* const* ys, const int64_t* y_strides, int32_t tokens, uint32_t flags, void* stream) {
  if (!descs || !x || !ys || !y_strides || n < 1) {
    set_error("quant_gemv_multi: NULL argument");
    return VPTQ_ERR_INVALID;
  }
  for (int l = 0; l < n; ++l) {
    if (int rc = validate(descs[l], l == 0)) return rc;
    if (!ys[l] || y_strides[l] < descs[l]->out_features || x_stride < descs[l]->in_features) {
      set_error("quant_gemv_multi: bad y / stride for layer %d", l);
      return VPTQ_ERR_INVALID;
    }
  }
  return gemv_multi_launch(n, descs, x, x_stride, ys, y_strides, tokens, flags, static_cast<cudaStream_t>(stream));
}

int vptq_b200_quant_gemv_multi_ws(int32_t n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride,
                                  void* const* ys, const int64_t* y_strides, int32_t tokens, void* workspace,
                                  size_t workspace_bytes, uint32_t flags, void* stream) {
  if (!descs || !x || !ys || !y_strides || n < 1) {
    set_error("quant_gemv_multi_ws: NULL argument");
    return VPTQ_ERR_INVALID;
  }
  for (int l = 0; l < n; ++l) {
    if (int rc = validate(descs[l], l == 0)) return rc;
    if (!ys[l] || y_strides[l] < descs[l]->out_features || x_stride < descs[l]->in_features) {
      set_error("quant_gemv_multi_ws: bad y / stride for layer %d", l);
      return VPTQ_ERR_INVALID;
    }
  }
  return gemv_multi_launch(n, descs, x, x_stride, ys, y_strides, tokens, flags, static_cast<cudaStream_t>(stream), nullptr,
                           workspace, workspace_bytes);
}

int vptq_b200_quant_gemv_multi_tp(int32_t n, const vptq_linear_desc* const* descs, const void* x, int64_t x_stride,
                                  void* const* ys, const int64_t* y_strides, int32_t tokens,
                                  const vptq_tp_exchange* tp, void* workspace, size_t workspace_bytes, uint32_t flags,
                                  void* stream) {
  if (!descs || !x || !ys || !y_strides || n < 1 || !tp) {
    set_error("quant_gemv_multi_tp: NULL argument");
    return VPTQ_ERR_INVALID;
  }
  if (tp->struct_size != sizeof(vptq_tp_exchange) || tp->world < 1 || tp->world > VPTQ_MAX_RANKS || tp->rank < 0 ||
      tp->rank >= tp->world || tp->slot < 0 || !tp->epoch || !tp->done || !tp->error) {
    set_error("quant_gemv_multi_tp: bad vptq_tp_exchange (size %u, world %d, rank %d, slot %d)", tp->struct_size,
              tp->world, tp->rank, tp->slot);
    return VPTQ_ERR_INVALID;
  }
  // The exchange itself, before any descriptor: a slot outside the epoch / flag arrays or a store the kernel would
  // issue to a misaligned peer address must never reach a launch.
  if (tp->num_slots <= tp->slot || tp->wait_slot < -1 || tp->wait_slot >= tp->num_slots) {
    set_error("quant_gemv_multi_tp: need 0 <= slot < num_slots and -1 <= wait_slot < num_slots (slot %d, wait_slot "
              "%d, num_slots %d)", tp->slot, tp->wait_slot, tp->num_slots);
    return VPTQ_ERR_INVALID;
  }
  if (n > VPTQ_MAX_FUSED) {
    set_error("quant_gemv_multi_tp: %d layers exceed VPTQ_MAX_FUSED (%d)", n, VPTQ_MAX_FUSED);
    return VPTQ_ERR_INVALID;
  }
  const bool tagged = tp->format == VPTQ_TP_TAGGED;
  for (int l = 0; l < n; ++l) {
    const uintptr_t y = reinterpret_cast<uintptr_t>(ys[l]);
    if (!y) {
      set_error("quant_gemv_multi_tp: ys[%d] is NULL", l);
      return VPTQ_ERR_INVALID;
    }
    if (tagged && (y & 15u)) {
      set_error("quant_gemv_multi_tp: VPTQ_TP_TAGGED needs ys[%d] 16-byte aligned", l);
      return VPTQ_ERR_INVALID;
    }
    for (int r = 0; r < tp->world; ++r) {
      const uintptr_t peer = reinterpret_cast<uintptr_t>(tp->peer_y[l][r]);
      if (!peer) continue;  // (NULL: refused below for every rank but this one)
      if (tagged && (peer & 15u)) {
        set_error("quant_gemv_multi_tp: VPTQ_TP_TAGGED needs peer_y[%d][%d] 16-byte aligned", l, r);
        return VPTQ_ERR_INVALID;
      }
      if (!tagged && ((peer - y) & 15u)) {
        set_error("quant_gemv_multi_tp: peer_y[%d][%d] - ys[%d] must be a multiple of 16 bytes", l, r, l);
        return VPTQ_ERR_INVALID;
      }
    }
  }
  for (int l = 0; l < n; ++l) {
    if (int rc = validate(descs[l], l == 0)) return rc;
    if (!ys[l] || y_strides[l] < descs[l]->out_features || x_stride < descs[l]->in_features) {
      set_error("quant_gemv_multi_tp: bad y / stride for layer %d", l);
      return VPTQ_ERR_INVALID;
    }
    for (int r = 0; r < tp->world; ++r)
      if (r != tp->rank && (!tp->peer_y[l][r] || !tp->peer_flags[r])) {
        set_error("quant_gemv_multi_tp: NULL peer pointer (layer %d, rank %d)", l, r);
        return VPTQ_ERR_INVALID;
      }
  }
  return gemv_multi_launch(n, descs, x, x_stride, ys, y_strides, tokens, flags, static_cast<cudaStream_t>(stream), tp,
                           workspace, workspace_bytes);
}

int vptq_b200_tp_untag(const void* tagged, void* y, int32_t n, const vptq_tp_exchange* tp, void* stream) {
  if (!tagged || !y || !tp || n < 8 || (n % 8) || tp->struct_size != sizeof(vptq_tp_exchange) ||
      tp->format != VPTQ_TP_TAGGED || !tp->epoch || !tp->error || tp->slot < 0 || tp->slot >= tp->num_slots ||
      (reinterpret_cast<uintptr_t>(tagged) & 15u) || (reinterpret_cast<uintptr_t>(y) & 15u)) {
    set_error("tp_untag: NULL / misaligned argument, n %% 8 != 0 or not the exchange of a VPTQ_TP_TAGGED launch");
    return VPTQ_ERR_INVALID;
  }
  return tp_untag_launch(tagged, y, n, *tp, static_cast<cudaStream_t>(stream));
}

int vptq_b200_dequant(const vptq_linear_desc* desc, void* w_out, void* workspace, size_t workspace_bytes,
                      void* stream) {
  if (int rc = validate(desc, true)) return rc;
  if (!w_out) {
    set_error("dequant: w_out is NULL");
    return VPTQ_ERR_INVALID;
  }
  if (int rc = need_packed(desc, "dequant")) return rc;
  return dequant_launch(*desc, w_out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int vptq_b200_quant_gemm(const vptq_linear_desc* desc, const void* x, int64_t x_stride, void* y,
                         int64_t y_stride, int32_t tokens, void* workspace, size_t workspace_bytes,
                         uint32_t flags, void* stream) {
  if (flags & VPTQ_FLAG_TRANSPOSE) {  // input gradient: x = dY [tokens][O], y = dX [tokens][I]
    if (int rc = validate(desc, false)) return rc;
    if (!x || !y || tokens < 1 || x_stride < desc->out_features || y_stride < desc->in_features) {
      set_error("quant_gemm (transpose): bad x/y/tokens/strides (x_stride %lld must be >= out_features %d, y_stride "
                "%lld >= in_features %d)", (long long)x_stride, desc->out_features, (long long)y_stride,
                desc->in_features);
      return VPTQ_ERR_INVALID;
    }
    if (int rc = need_packed(desc, "quant_gemm (transpose)")) return rc;
    if (int rc = check_device()) return rc;
    return dgrad_launch(*desc, x, x_stride, y, y_stride, tokens, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream));
  }
  if (int rc = validate(desc, true)) return rc;
  if (!x || !y || tokens < 1 || x_stride < desc->in_features || y_stride < desc->out_features) {
    set_error("quant_gemm: bad x/y/tokens/strides");
    return VPTQ_ERR_INVALID;
  }
  if (int rc = need_packed(desc, "quant_gemm")) return rc;
  return gemm_launch(*desc, x, x_stride, y, y_stride, tokens, workspace, workspace_bytes, flags,
                     static_cast<cudaStream_t>(stream));
}

// ---- training entry points (include/vptq_b200_grad.h) ----
int vptq_b200_grad_version(void) { return VPTQ_B200_GRAD_VERSION; }

size_t vptq_b200_grad_workspace_bytes(const vptq_linear_desc* desc, int32_t tokens, int32_t op) {
  if (validate(desc, false)) return 0;
  if (op != VPTQ_GRAD_OP_WGRAD && op != VPTQ_GRAD_OP_DEQUANT_BACKWARD && op != VPTQ_GRAD_OP_WGRAD_GENERIC) {
    set_error("grad_workspace_bytes: unknown op %d", op);
    return 0;
  }
  return wgrad_workspace_bytes(*desc, tokens, op);
}

int vptq_b200_quant_gemm_wgrad(const vptq_linear_desc* desc, const void* x, int64_t x_stride, const void* dy,
                               int64_t dy_stride, int32_t tokens, const vptq_linear_grads* grads, void* workspace,
                               size_t workspace_bytes, uint32_t flags, void* stream) {
  if (int rc = validate(desc, false)) return rc;
  if (!x || !dy || tokens < 1 || x_stride < desc->in_features || dy_stride < desc->out_features ||
      (reinterpret_cast<uintptr_t>(x) & 1u) || (reinterpret_cast<uintptr_t>(dy) & 1u)) {
    set_error("quant_gemm_wgrad: bad x/dy/tokens/strides (tokens %d, x_stride %lld must be >= in_features %d, "
              "dy_stride %lld >= out_features %d)", tokens, (long long)x_stride, desc->in_features,
              (long long)dy_stride, desc->out_features);
    return VPTQ_ERR_INVALID;
  }
  if (int rc = validate_grads(desc, grads, flags, VPTQ_GRAD_FLAG_GENERIC, "quant_gemm_wgrad")) return rc;
  if (int rc = need_packed(desc, "quant_gemm_wgrad")) return rc;
  if (int rc = check_device()) return rc;
  return wgrad_launch(*desc, x, x_stride, dy, dy_stride, tokens, *grads, workspace, workspace_bytes, flags,
                      static_cast<cudaStream_t>(stream));
}

int vptq_b200_dequant_backward(const vptq_linear_desc* desc, const void* dw, int64_t dw_stride,
                               const vptq_linear_grads* grads, void* workspace, size_t workspace_bytes, uint32_t flags,
                               void* stream) {
  if (int rc = validate(desc, false)) return rc;
  if (!dw || dw_stride < desc->in_features || (reinterpret_cast<uintptr_t>(dw) & 1u)) {
    set_error("dequant_backward: bad dw / stride (dw_stride %lld must be >= in_features %d)", (long long)dw_stride,
              desc->in_features);
    return VPTQ_ERR_INVALID;
  }
  if (int rc = validate_grads(desc, grads, flags, 0u, "dequant_backward")) return rc;
  if (int rc = need_packed(desc, "dequant_backward")) return rc;
  if (int rc = check_device()) return rc;
  return dequant_backward_launch(*desc, dw, dw_stride, *grads, workspace, workspace_bytes,
                                 static_cast<cudaStream_t>(stream));
}

int vptq_b200_quant_gemv_v2(int32_t dtype, const void* x, void* y, int32_t tokens, int32_t in_features,
                            int32_t out_features, int32_t vector_len, int32_t num_centroids,
                            int32_t num_res_centroids, const uint16_t* indices, const void* centroids,
                            const void* residual_indices, int32_t res_index_bytes,
                            const void* residual_centroids, const void* scale_weights,
                            const void* scale_bias, const void* bias, void* workspace,
                            size_t workspace_bytes, uint32_t flags, void* stream) {
  if (dtype != VPTQ_FP16 && dtype != VPTQ_BF16) {
    set_error("quant_gemv_v2: dtype %d unsupported", dtype);
    return VPTQ_ERR_UNSUPPORTED;
  }
  if (!x || !y || !indices || !centroids || tokens < 1 || in_features < 1 || out_features < 1) {
    set_error("quant_gemv_v2: NULL pointer or non-positive size");
    return VPTQ_ERR_INVALID;
  }
  if ((scale_weights == nullptr) != (scale_bias == nullptr)) {
    set_error("quant_gemv_v2: scale_weights and scale_bias go together");
    return VPTQ_ERR_INVALID;
  }
  if (num_res_centroids > 0 && (!residual_indices || !residual_centroids ||
                                (res_index_bytes != 1 && res_index_bytes != 2))) {
    set_error("quant_gemv_v2: residual codebook given without u8/u16 residual indices");
    return VPTQ_ERR_INVALID;
  }
  const DeviceInfo* dev = device_info();
  if (!dev) return VPTQ_ERR_CUDA;
  if (dev->cc_major != 9 || dev->cc_minor != 0) {
    set_error("device compute capability %d.%d: sm_90a code only", dev->cc_major, dev->cc_minor);
    return VPTQ_ERR_DEVICE;
  }
  GemvV2Args a{dtype,     tokens,           in_features,     out_features,       vector_len,    num_centroids,
               num_res_centroids, x,        y,               indices,            centroids,     residual_indices,
               res_index_bytes,   residual_centroids, scale_weights, scale_bias, bias};
  return gemv_v2_launch(a, workspace, workspace_bytes, flags, static_cast<cudaStream_t>(stream));
}

int vptq_b200_linear_host(const vptq_linear_desc* desc, const void* x_host, void* y_host, int32_t tokens,
                          void* x_dev, void* y_dev, void* workspace, size_t workspace_bytes, uint32_t flags,
                          void* stream) {
  if (int rc = validate(desc, true)) return rc;
  if (!x_host || !y_host || !x_dev || !y_dev || tokens < 1) {
    set_error("linear_host: NULL buffer");
    return VPTQ_ERR_INVALID;
  }
  if (tokens >= 3)
    if (int rc = need_packed(desc, "linear_host (prefill)")) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t xb = size_t(tokens) * desc->in_features * 2, yb = size_t(tokens) * desc->out_features * 2;
  cudaError_t e = cudaMemcpyAsync(x_dev, x_host, xb, cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) {
    set_error("linear_host H2D: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  int rc;
  if (tokens < 3)  // the reference's routing rule, vptq/ops/quant_gemm.py:213
    rc = gemv_launch(*desc, x_dev, desc->in_features, y_dev, desc->out_features, tokens, workspace,
                     workspace_bytes, flags, s);
  else
    rc = gemm_launch(*desc, x_dev, desc->in_features, y_dev, desc->out_features, tokens, workspace,
                     workspace_bytes, flags, s);
  if (rc) return rc;
  e = cudaMemcpyAsync(y_host, y_dev, yb, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    set_error("linear_host D2H/sync: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  return 0;
}

int vptq_b200_stream_capture_id(void* stream, uint64_t* id) {
  if (!id) {
    set_error("stream_capture_id: NULL id");
    return VPTQ_ERR_INVALID;
  }
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  unsigned long long cid = 0;
  cudaError_t e = cudaStreamGetCaptureInfo(static_cast<cudaStream_t>(stream), &st, &cid);
  if (e != cudaSuccess) {
    set_error("cudaStreamGetCaptureInfo: %s", cudaGetErrorString(e));
    return VPTQ_ERR_CUDA;
  }
  *id = st == cudaStreamCaptureStatusActive ? uint64_t(cid) : 0;
  return st == cudaStreamCaptureStatusActive ? 1 : 0;
}

}  // extern "C"
