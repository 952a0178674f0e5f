/*
 * vptq_b200_lists16.h  --  decode from the index lists for vector-length-16 layers (the v16-k65536 checkpoints,
 * 1.375-1.5 bits per weight): 1..4 tokens of up to VPTQ_MAX_FUSED layers reading the same x in one launch, without
 * materialising the weight.  Exported from the same library as include/vptq_b200.h; the inference ABI (its symbols,
 * VPTQ_B200_ABI_VERSION, vptq_linear_desc) is unchanged by them.  A library without these symbols fails at symbol
 * lookup.
 *
 * Lists.  The slice x tile lists of vptq_linear_desc::lists_stream / lists_tab / lists_tile_cols (entry word, tile
 * geometry, tab and padding exactly as at v = 8, see include/vptq_b200.h), but an index row covers 16 outputs:
 * Ro = ceil(out_features / 16) rows per combo.  Build them with vptq_b200_lists16_build_host (or the Python builder,
 * vptq_b200.lists.build_lists(vector_len=16)); vptq_b200_lists_deal_host applies unchanged.  Every other entry point
 * of the library treats a vector-length-16 descriptor that carries lists exactly as one without lists.
 *
 * Layers: vector_len 16, one codebook group, no outlier columns, num_centroids K = 4096 * (2..16), no residual or
 * num_res_centroids <= 256, 16-byte aligned lists_stream, weight_scale and weight_bias, and slices x column tiles
 * (K / 4096 * ceil(in_features / 4096)) * n <= the device's SM count.
 *
 * Arithmetic, per token t and output o (x' = x * weight_scale rounded to the layer's 16-bit type, in ORIGINAL
 * feature order; C, R the main / residual entries of a field): the list kernels' (include/vptq_b200_batch.h) --
 * fp32 FMAs of x'_t * (C + R) per unit (C + R in packed fp16 for fp16 layers, fp32 for bf16), sum x_t * weight_bias
 * of a column tile added to its slice-0 unit, unit sums rounded to 2^-30 fixed point and summed as 64-bit integers,
 * bias added after the conversion, one rounding to the layer type.  At most Q * 2^-31 per output from the fixed
 * point; unit sums that are not finite or too large make the output +inf, -inf or NaN (the class of their sum).
 *
 * Token invariance: the launch's CTAs, warps and warp runs depend on the layers' shapes and the SM count only, so a
 * token's outputs are bit-identical whatever the other rows of x are, at any position, for 1 to the maximum token
 * count.  (They are not those of vptq_b200_quant_gemv, which cuts the sums differently.)
 *
 * Conventions are those of include/vptq_b200.h: the caller allocates outputs and a zero-initialised workspace of at
 * least VPTQ_B200_LISTS16_WORKSPACE_BYTES (kernels leave it zeroed), no call synchronises, every call is CUDA-graph
 * capturable, errors come back as a negative vptq_status with vptq_b200_last_error().  No fall-back to another kernel.
 */
#ifndef VPTQ_B200_LISTS16_H_
#define VPTQ_B200_LISTS16_H_

#include "vptq_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VPTQ_B200_LISTS16_VERSION 1
/* zero-at-rest head a launch needs: row counters, class records, [row][token][16] 64-bit accumulators */
#define VPTQ_B200_LISTS16_WORKSPACE_BYTES ((size_t)65536 * 4 + (size_t)65536 * 64)

VPTQ_B200_API int vptq_b200_lists16_version(void);

/*
 * The largest token count (4, 2 or 1) vptq_b200_quant_gemv_lists16 takes for these n (1..VPTQ_MAX_FUSED) layers on
 * the current device, or 0 when they are not eligible (see above; also: layers that differ in dtype, in_features,
 * num_centroids or in having a residual codebook, or whose index rows times the token count exceed 32768, or no
 * shared-memory layout fits).  0 also sets the error message.  Enqueues nothing.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_lists16_max_tokens(int32_t n, const vptq_linear_desc* const* descs);

/*
 * ys[l] [tokens][y_strides[l]] = x [tokens][x_stride] . W_l^T + bias_l for n layers reading the same x, in one
 * launch.  1 <= tokens <= vptq_b200_quant_gemv_lists16_max_tokens(n, descs); x_stride >= in_features, y_strides[l] >=
 * out_features, x 16-byte aligned.  flags: 0 or VPTQ_FLAG_PDL.  Returns VPTQ_ERR_INVALID (NULL or bad argument),
 * VPTQ_ERR_UNSUPPORTED (not eligible, bad token count) or VPTQ_ERR_WORKSPACE (workspace too small) with a message;
 * nothing is launched then.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_lists16(int32_t n, const vptq_linear_desc* const* descs, const void* x,
                                               int64_t x_stride, void* const* ys, const int64_t* y_strides,
                                               int32_t tokens, void* workspace, size_t workspace_bytes, uint32_t flags,
                                               void* stream);

/*
 * Host (CPU) builder of the vector-length-16 lists: the arguments, sizing call (stream_out = NULL) and results of
 * vptq_b200_lists_build_host, with index rows of 16 outputs (indices_host holds ceil(out_features / 16) rows).
 * Byte-identical to vptq_b200.lists.build_lists(vector_len=16, deal=False); run vptq_b200_lists_deal_host after it.
 */
VPTQ_B200_API int vptq_b200_lists16_build_host(const int32_t* indices_host, int64_t index_stride_row,
                                               int32_t out_features, int32_t in_features, int32_t num_centroids,
                                               int32_t num_res_centroids, const uint16_t* perm_host, void* stream_out,
                                               size_t stream_capacity, uint32_t* tab_out, size_t* steps_out,
                                               int32_t* tile_cols_out);

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_LISTS16_H_ */
