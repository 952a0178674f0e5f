/*
 * vptq_b200_grad.h  --  training entry points of libvptq_b200.so: gradients of a VPTQ layer's codebooks,
 * weight_scale and weight_bias.  Exported from the same library as include/vptq_b200.h; the inference ABI
 * (its symbols, VPTQ_B200_ABI_VERSION, vptq_linear_desc, the vptq_op codes) is unchanged by them.  A library
 * without these symbols fails at symbol lookup.
 *
 * Notation (vptq_linear_desc): quantised column c, original feature f = perm[c], index row r, output
 * o = v r + e (e < v, o < O).  For c >= S: group g = (c - S) / gs and the field (k, kr) of row r, column
 * (c - S) mod gs.
 *   Wq[o][f] = C_g[k][e] + R_g[kr][e]       (fp32 from the 16-bit values, as the dequant kernels evaluate it)
 *   Wq[o][f] = Col[outlier_indices[o / vol][c]][o mod vol]          for an outlier column c < S
 *   W[o][f]  = Wq[o][f] * s_f + b_f         (s = weight_scale, b = weight_bias; 1 and 0 without them)
 * Given G[o][f] = dL/dW[o][f]:
 *   dC_g[k][e]        = sum over (r, c) of group g with main index k, o = v r + e < O, of  s_f G[o][f]
 *   dR_g[kr][e]       = the same sum over residual index kr
 *   dCol[oi][eo]      = sum over outlier columns c < S and rows with outlier index oi, o = vol rol + eo < O
 *   d weight_scale[f] = sum_o G[o][f] Wq[o][f]
 *   d weight_bias[f]  = sum_o G[o][f]
 * Padding outputs (o >= O) contribute nothing; indices and perm get no gradient.
 *
 * Method: terms are added as 64-bit fixed-point integers (red.global.add.u64), so every result is independent of
 * the order the GPU adds them in -- bit-identical from run to run and under CUDA-graph replay.  The unit is a
 * power of two chosen per call on the device from a cheap bound B of the sum of |terms| (unit >= B / 2^61), so
 * no partial sum can overflow.  Every term is rounded to the unit on its own, and each gradient element is rounded
 * once, correctly, from its integer sum to the layer's dtype.  If any value of x, dY or G is not finite (including an
 * fp32 element of G that overflows), or of weight_scale, or -- when d weight_scale is requested -- of any main,
 * residual or outlier codebook entry, used or not, every requested gradient is NaN (fixed point carries no inf; a
 * loss-scaling loop sees the overflow).  Without d weight_scale the codebook values are not read, and weight_bias
 * and bias never are: non-finite values there change no bit.  A sum past the largest finite value gives +-inf with
 * its sign.
 *
 * Conventions are those of include/vptq_b200.h: the caller allocates outputs and workspace, no call
 * synchronises, every call is CUDA-graph capturable, decode-only descriptors (indices == NULL) are refused, and
 * errors come back as a negative vptq_status with vptq_b200_last_error().  The workspace needs no zeroing and
 * may be the one the inference calls use: these calls never touch its zero-at-rest head.
 */
#ifndef VPTQ_B200_GRAD_H_
#define VPTQ_B200_GRAD_H_

#include "vptq_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define VPTQ_B200_GRAD_VERSION 1

typedef enum vptq_grad_op {
  VPTQ_GRAD_OP_WGRAD = 0,            /* vptq_b200_quant_gemm_wgrad                            */
  VPTQ_GRAD_OP_DEQUANT_BACKWARD = 1, /* vptq_b200_dequant_backward                            */
  VPTQ_GRAD_OP_WGRAD_GENERIC = 2     /* vptq_b200_quant_gemm_wgrad with VPTQ_GRAD_FLAG_GENERIC */
} vptq_grad_op;

/* vptq_b200_quant_gemm_wgrad only: take the generic route (G in fp32 in the workspace, then a scatter kernel) also
   for a layer the fused route covers.  Both routes give bit-identical gradients; the flag exists so that one can
   be checked against the other.  Workspace: VPTQ_GRAD_OP_WGRAD_GENERIC. */
#define VPTQ_GRAD_FLAG_GENERIC 1u

/* Output of one gradient call: one pointer per gradient, in the layer's dtype and in the layout of the matching
   vptq_linear_desc tensor (centroids [G][centroid_stride], res_centroids [G][res_centroid_stride], outlier
   centroids [Kol * vol], weight_scale / weight_bias [I]).  NULL = not wanted: nothing is computed for it.  Every
   element of a requested gradient is written (zero where no term lands). */
typedef struct vptq_linear_grads {
  uint32_t struct_size; /* = sizeof(vptq_linear_grads) */
  uint32_t reserved;    /* 0 */
  void* centroids;
  void* res_centroids;
  void* outlier_centroids;
  void* weight_scale;
  void* weight_bias;
} vptq_linear_grads;

VPTQ_B200_API int vptq_b200_grad_version(void);

/* Bytes of workspace `op` (vptq_grad_op) needs for this layer and token count (tokens is ignored by
   VPTQ_GRAD_OP_DEQUANT_BACKWARD).  0 on an invalid descriptor or op. */
VPTQ_B200_API size_t vptq_b200_grad_workspace_bytes(const vptq_linear_desc* desc, int32_t tokens, int32_t op);

/*
 * Weight gradients of y = x W^T + bias for G = dY^T x: x [tokens][x_stride] (x_stride >= I), dy [tokens][dy_stride]
 * (dy_stride >= O), tokens >= 1.  G is formed by the wgmma GEMM with fp32 accumulators.
 *   fused route   (v = 8, one codebook group, no outlier columns, Kr <= 256 -- every Llama shape): the GEMM's
 *                 epilogue adds every accumulator straight into the fixed-point sums; G is never stored.
 *   generic route (every other layer, or VPTQ_GRAD_FLAG_GENERIC): the GEMM stores G in fp32 in the workspace
 *                 (O * I * 4 bytes) and a scatter kernel reduces it.
 * flags: 0 or VPTQ_GRAD_FLAG_GENERIC.
 */
VPTQ_B200_API int vptq_b200_quant_gemm_wgrad(const vptq_linear_desc* desc, const void* x, int64_t x_stride,
                                             const void* dy, int64_t dy_stride, int32_t tokens,
                                             const vptq_linear_grads* grads, void* workspace, size_t workspace_bytes,
                                             uint32_t flags, void* stream);

/*
 * Backward of vptq_b200_dequant: G = dw [O][dw_stride] (dw_stride >= I, the layer's dtype, original feature
 * order) is the incoming gradient of W.  flags must be 0.
 */
VPTQ_B200_API int vptq_b200_dequant_backward(const vptq_linear_desc* desc, const void* dw, int64_t dw_stride,
                                             const vptq_linear_grads* grads, void* workspace, size_t workspace_bytes,
                                             uint32_t flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_GRAD_H_ */
