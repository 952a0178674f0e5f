/*
 * vptq_b200_lists_dense.h  --  prefill, dequant and input gradient of a layer from its slice x tile index lists
 * (vptq_linear_desc::lists_*), never from the packed index words.  This is what lets a decode-only descriptor
 * (indices == NULL: the packed words were freed once the lists were built, one copy of the indices resident) serve
 * prompts and backward passes.  Exported from the same library as include/vptq_b200.h; the inference ABI (its
 * symbols, VPTQ_B200_ABI_VERSION, vptq_linear_desc) is unchanged by them.  A library without these symbols fails at
 * symbol lookup.
 *
 * The dense weight is written from the lists with the packed dequant kernels' arithmetic,
 *   W[o][f] = fmaf(C + R, weight_scale[f], weight_bias[f]) in fp32, rounded once to the layer type
 * (scale 1, bias 0 without a norm), so it is bit-identical to what vptq_b200_dequant and the transposed dequant of
 * vptq_b200_quant_gemm(VPTQ_FLAG_TRANSPOSE) produce from the packed words of the same layer.  The GEMMs are the
 * prefill kernel of vptq_b200_quant_gemm: where that call takes its prep-free route (in_features % 64 == 0, x 16-byte
 * aligned with a row pitch that is a multiple of 8, VPTQ_B200_GEMM_PREP unset) and for every input gradient, results
 * are bit-identical to it.  Elsewhere they agree to within the prefill route's rounding (x is not pre-scaled here).
 *
 * Both list geometries are taken: vector_len 8 (the lists of vptq_b200_quant_gemv) and vector_len 16 (the lists of
 * vptq_b200_quant_gemv_lists16, include/vptq_b200_lists16.h: an index row covers 16 outputs, lists_tile_cols of
 * that header's geometry).  Either way one codebook group, no outliers, K = 4096 * (2..16) and Kr <= 256.  The
 * workspace layout is the same for both: W [out_features][in_features rounded up to 64] (Wt: [in_features][pitch of
 * the input-gradient GEMM]) after the zero-at-rest head, then the staged activation.  At vector_len 16 the last index
 * row's outputs past out_features are never part of W, and are zeros in Wt.
 *
 * Every call accepts a descriptor that carries index lists, decode-only or full (the packed words are then
 * ignored), and refuses one without them (VPTQ_ERR_UNSUPPORTED).  Conventions are those of include/vptq_b200.h: the
 * caller allocates outputs and workspace (zero-initialised once; kernels leave its head zeroed), no call allocates
 * or synchronises, every call is CUDA-graph capturable, errors come back as a negative vptq_status with
 * vptq_b200_last_error(), and nothing is launched on a refusal.
 */
#ifndef VPTQ_B200_LISTS_DENSE_H_
#define VPTQ_B200_LISTS_DENSE_H_

#include "vptq_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VPTQ_B200_LISTS_DENSE_VERSION 1

VPTQ_B200_API int vptq_b200_lists_dense_version(void);

/*
 * Bytes of workspace vptq_b200_lists_quant_gemm needs for this layer and token count (flags: 0 or
 * VPTQ_FLAG_TRANSPOSE, VPTQ_FLAG_PDL ignored); 0 with an error message when the call would be refused.
 */
VPTQ_B200_API size_t vptq_b200_lists_dense_workspace_bytes(const vptq_linear_desc* desc, int32_t tokens,
                                                           uint32_t flags);

/*
 * flags 0: W [out_features][ld] in original feature order, ld >= in_features, columns [in_features, ld) zero,
 * padding rows of a ragged out_features not written.  flags VPTQ_FLAG_TRANSPOSE: Wt [in_features][ld],
 * ld >= out_features, columns [out_features, ld) zero.  w 16-byte aligned, ld a multiple of 8.  No workspace.
 */
VPTQ_B200_API int vptq_b200_lists_dequant(const vptq_linear_desc* desc, void* w, int64_t ld, uint32_t flags,
                                          void* stream);

/*
 * flags 0: y [tokens][y_stride] = x [tokens][x_stride] . W^T + bias (x_stride >= in_features, y_stride >=
 * out_features).  VPTQ_FLAG_TRANSPOSE: the input gradient y = dX [tokens][in_features] = x . W with x = dY
 * [tokens][out_features], no bias (x_stride >= out_features, y_stride >= in_features).  Any tokens >= 1.
 * VPTQ_FLAG_PDL is accepted; these kernels launch without programmatic dependent launch.  Workspace:
 * vptq_b200_lists_dense_workspace_bytes(desc, tokens, flags).
 */
VPTQ_B200_API int vptq_b200_lists_quant_gemm(const vptq_linear_desc* desc, const void* x, int64_t x_stride, void* y,
                                             int64_t y_stride, int32_t tokens, void* workspace,
                                             size_t workspace_bytes, uint32_t flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_LISTS_DENSE_H_ */
