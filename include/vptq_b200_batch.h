/*
 * vptq_b200_batch.h  --  batched decode from the index lists: 1..8 tokens (several sequences, beams, speculative
 * verification) in one launch that reads only vptq_linear_desc::lists_*, never a dequantised weight.  Exported from
 * the same library as include/vptq_b200.h; the inference ABI (its symbols, VPTQ_B200_ABI_VERSION,
 * vptq_linear_desc) is unchanged by them.  A library without these symbols fails at symbol lookup.
 *
 * Arithmetic, per token t and output o (x' = x * weight_scale rounded to the layer's 16-bit type, in ORIGINAL
 * feature order; C, R the main / residual entries of a field):
 *   * the fields of an index row are summed per unit = (column tile, codebook slice, index row) in fp32 FMAs,
 *     x'_t * (C + R) with C + R in packed fp16 (fp16 layers) or fp32 (bf16 layers);
 *   * sum_f x_t[f] * weight_bias[f] over a column tile (fp32) is added to the tile's slice-0 unit;
 *   * each unit sum is rounded to 2^-30 fixed point and the Q = slices x tiles units of an output are added as
 *     64-bit integers (order-free), converted back to fp32, bias added, rounded once to the layer type.
 *   The fixed point costs at most Q * 2^-31 per output, absolute.  Unit sums that are not finite or too large to
 *   add without wrapping make the output +inf, -inf or NaN (the class of their sum); an fp16 output past 65504
 *   becomes +-inf.
 *
 * Token invariance: how a launch is cut into CTAs, warps and warp runs depends on the layers' shapes and the
 * device's SM count only, never on the token count.  Each token's sums see the same entries in the same order, so
 * a token's outputs are bit-identical whatever the other rows of x are, at whatever position, for any token count
 * from 1 to the maximum, and from run to run.  (They are not those of vptq_b200_quant_gemv: that kernel cuts
 * the same sums differently and may round them differently in the last place.)
 *
 * Conventions are those of include/vptq_b200.h: the caller allocates outputs and workspace (zero-initialised, the
 * size vptq_b200_workspace_bytes(desc, 1, VPTQ_OP_GEMV) gives, summed over the layers; kernels leave its head
 * zeroed), no call synchronises, every call is CUDA-graph capturable, and errors come back as a negative
 * vptq_status with vptq_b200_last_error().  There is no fall-back to another kernel.
 */
#ifndef VPTQ_B200_BATCH_H_
#define VPTQ_B200_BATCH_H_

#include "vptq_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VPTQ_B200_BATCH_VERSION 1

VPTQ_B200_API int vptq_b200_batch_version(void);

/*
 * The largest token count vptq_b200_quant_gemv_batch takes for these n (1..VPTQ_MAX_FUSED) layers on the current
 * device, or 0 when they are not eligible: a layer without index lists (or one the single-token list kernel does
 * not take: v != 8, groups, outliers, Kr > 256), layers that differ in dtype, in_features, num_centroids or in having
 * a residual codebook, n * slices * tiles > SM count, or index rows of all layers x 8 > 65536.  0 also sets the
 * error message.  Enqueues nothing.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_batch_max_tokens(int32_t n, const vptq_linear_desc* const* descs);

/*
 * ys[l] [tokens][y_strides[l]] = x [tokens][x_stride] . W_l^T + bias_l for n layers reading the same x, in one
 * launch.  1 <= tokens <= vptq_b200_quant_gemv_batch_max_tokens(n, descs); x_stride >= in_features, y_strides[l] >=
 * out_features, x 16-byte aligned.  Decode-only descriptors (indices == NULL) are accepted.  flags: 0 or
 * VPTQ_FLAG_PDL.  Returns VPTQ_ERR_UNSUPPORTED (not eligible, bad token count) or VPTQ_ERR_WORKSPACE (workspace
 * too small) with a message; nothing is launched then.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_batch(int32_t n, const vptq_linear_desc* const* descs, const void* x,
                                             int64_t x_stride, void* const* ys, const int64_t* y_strides,
                                             int32_t tokens, void* workspace, size_t workspace_bytes, uint32_t flags,
                                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_BATCH_H_ */
