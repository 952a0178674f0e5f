/*
 * vptq_b200.h  --  C ABI of libvptq_b200.so: the H100 (sm_90a) VPTQ quantized-linear hot path.
 *
 * This is the drop-in boundary.  It replaces the three pybind11 entry points the reference
 * registers in csrc/ops.cc:44-55 (module `vptq.libvptq`, bound by vptq/ops/quant_gemm.py:22-26):
 *
 *   reference (pybind11, torch::Tensor in / out)          this library (plain pointers, sizes)
 *   ---------------------------------------------------   -----------------------------------------
 *   quant_gemv   = vptq::wquant_act16_gemv                 vptq_b200_quant_gemv
 *                  csrc/ops.cc:20-30,49  quant_gemv.cu:241
 *   dequant      = vptq::dequant                           vptq_b200_dequant
 *                  csrc/ops.cc:9-18,47   dequant.cu:227
 *   dequant + torch F.linear (vptq/ops/quant_gemm.py:231-275)
 *                                                          vptq_b200_quant_gemm   (fused, wgmma)
 *   quant_gemv_v2 = vptq::quant_gemv_v2                    vptq_b200_quant_gemv_v2
 *                  csrc/ops.cc:32-38,53  quant_gemv_v2.cu:25
 *
 * Conventions (differences from the reference boundary are deliberate, see INTEGRATION.md):
 *   - No torch types.  All tensors are raw DEVICE pointers described by vptq_linear_desc.
 *   - The CALLER allocates outputs and workspace (the reference allocates with at::empty inside:
 *     quant_gemv.cu:203-206, dequant.cu:186).  The library never allocates or frees device
 *     memory, never synchronises, and only enqueues work on `stream` (a cudaStream_t passed as
 *     void*; NULL = legacy default stream).  Every call is CUDA-graph capturable.
 *   - Errors: return 0 on success, a negative vptq_status otherwise; vptq_b200_last_error()
 *     returns a thread-local message (the reference throws through TORCH_CHECK,
 *     quant_gemv.cu:252-282).  There is no CPU fallback and no silent fallback of any kind:
 *     unsupported configurations return VPTQ_ERR_UNSUPPORTED.
 *   - `perm` has the reference's meaning: perm[c] = original input feature of quantised column c
 *     (csrc/kernels/quant_gemv.cuh:53-54).  The reference passes perm to quant_gemv and
 *     argsort(perm) to dequant (vptq/ops/quant_gemm.py:208-211,222,239); here both entry points
 *     take `perm` and derive what they need on the device.
 *   - The workspace must be zero-filled ONCE by the caller before its first use (cudaMemset /
 *     torch.zeros).  Kernels leave it zeroed again on completion, so it can be reused by every
 *     subsequent call on the same stream without clearing.
 */
#ifndef VPTQ_B200_H_
#define VPTQ_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VPTQ_B200_ABI_VERSION 7

#if defined(__GNUC__)
#define VPTQ_B200_API __attribute__((visibility("default")))
#else
#define VPTQ_B200_API
#endif

typedef enum vptq_dtype {
  VPTQ_FP16 = 0, /* IEEE binary16 (torch.float16) */
  VPTQ_BF16 = 1  /* bfloat16 (torch.bfloat16)     */
} vptq_dtype;

typedef enum vptq_status {
  VPTQ_OK = 0,
  VPTQ_ERR_INVALID = -1,     /* NULL / misaligned pointer, inconsistent sizes              */
  VPTQ_ERR_UNSUPPORTED = -2, /* well-formed but not implemented (message says what)        */
  VPTQ_ERR_WORKSPACE = -3,   /* workspace smaller than vptq_b200_workspace_bytes()         */
  VPTQ_ERR_CUDA = -4,        /* a CUDA runtime call failed (message carries the CUDA text) */
  VPTQ_ERR_DEVICE = -5       /* current device is not compute capability 9.0               */
} vptq_status;

/* launch flags (bit-or) */
#define VPTQ_FLAG_PDL 1u /* launch with programmatic dependent launch: the kernel prefetches
                            weights/codebooks/indices before griddepcontrol.wait and only then
                            reads x; legal whenever x is produced by the preceding kernel on
                            the same stream */
#define VPTQ_FLAG_TRANSPOSE 2u /* vptq_b200_quant_gemm only: compute the layer's INPUT GRADIENT
                                  y[tokens][in_features] = x[tokens][out_features] . W instead of
                                  x W^T + bias (bias is not applied; x_stride >= out_features,
                                  y_stride >= in_features).  Workspace: VPTQ_OP_GEMM_DGRAD.  Any
                                  tokens >= 1.  Libraries before ABI 7 ignore this flag. */

/*
 * One VQuantLinear layer: exactly the tensors the reference module owns
 * (vptq/layers/vqlinear.py:89-240) in their checkpoint layout.  16-bit float tensors are
 * `dtype`; index tensors are the reference's uint16-viewed-as-int16 / packed int32 words.
 */
typedef struct vptq_linear_desc {
  uint32_t struct_size; /* = sizeof(vptq_linear_desc); guards ABI drift */
  int32_t dtype;        /* vptq_dtype of x, y, centroids, scale, bias  */

  int32_t in_features;           /* I                                                        */
  int32_t out_features;          /* O                                                        */
  int32_t vector_len;            /* v   = vector_lens[1]   (even, 2..16)                     */
  int32_t num_centroids;         /* K   = num_centroids[1] (power of two, <= 65536)          */
  int32_t num_res_centroids;     /* Kr  (power of two >= 2; <= 0: no residual codebook)      */
  int32_t num_codebooks;         /* G   = group_num                                          */
  int32_t group_size;            /* gs  columns per codebook group; S + G*gs == I            */
  int32_t outlier_size;          /* S   leading outlier columns (0: none)                    */
  int32_t outlier_vector_len;    /* vol = vector_lens[0]                                     */
  int32_t num_outlier_centroids; /* Kol = num_centroids[0]                                   */

  /* packed indices, int32 words [G][Ro][Wd], Ro = ceil(O/v), Wd = ceil(gs*(ib+rb)/32);
     field j of a row = bits [j*b, (j+1)*b) of its little-endian bit stream,
     field = idx | ridx << ib   (vptq/utils/pack.py:41-67).  Strides in 32-bit words. */
  const int32_t* indices; /* may be NULL when lists_stream / lists_tab are given (decode-only descriptor: the packed
                             words were dropped after the lists were built; only single-token GEMV calls work) */
  int64_t index_stride_codebook;
  int64_t index_stride_row;

  const void* centroids;     /* [G][K][v]   */
  int64_t centroid_stride;   /* elements between codebooks (>= K*v) */
  const void* res_centroids; /* [G][Kr][v]  or NULL */
  int64_t res_centroid_stride;

  const uint16_t* outlier_indices; /* [ceil(O/vol)][S] or NULL */
  const void* outlier_centroids;   /* [Kol][vol] or NULL       */

  const uint16_t* perm;     /* [I] or NULL (identity) */
  const void* weight_scale; /* [I] or NULL; scale and bias are both present or both NULL */
  const void* weight_bias;  /* [I] or NULL */
  const void* bias;         /* [O] or NULL */

  /* Optional load-time derivatives (NULL = not provided; results are identical either way):
     weight_scale / weight_bias gathered into QUANTISED column order, i.e. element c holds
     weight_scale[perm[c]] -- lets the decode kernel load them without waiting for perm. */
  const void* weight_scale_q; /* [I] or NULL */
  const void* weight_bias_q;  /* [I] or NULL */

  /* Optional second load-time derivative: the SAME indices re-bucketed into slice x tile lists for the
     decode kernel that keeps 64 KiB slices of a large main codebook in each SM's shared memory
     (NULL = not provided: the packed words above are decoded directly).  With the lists, single-token
     results round x * weight_scale to the layer's 16-bit type and, for fp16 layers, c + r to fp16, as
     the reference's kernel does, and sum in fp32 per unit, then in 2^-30 fixed point over the Q = NS * NT
     units of an output: an absolute error of up to Q * 2^-31 per output whatever its size.  By default
     the fixed point holds |output| < 2^33 only and carries no inf or NaN: with non-finite inputs or layer
     tensors, or unit sums past that range, these results are not defined.  With the environment variable
     VPTQ_B200_LISTS_CHECKED=1 (read at each launch) the kernel keeps such sums out of the fixed point and
     returns +inf, -inf or NaN for them (NaN for finite sums past 2^33 / 2^ceil(log2 Q)), like the other
     routes, at a cost of about 2 % of decode throughput.
     Eligible layers: vector_len 8, one codebook group, no outlier columns, K = NS * 4096 with
     2 <= NS <= 16, Kr <= 256; used for single-token calls.  Geometry:
       NT  = ceil(I / 4096) column tiles over the ORIGINAL input features,
       TCW = lists_tile_cols = ceil(ceil(I / NT) / 8) * 8 features per tile,
       combo = tile * NS + slice,  unit u = combo * Ro + r  (U = NS * NT * Ro units).
     Unit u lists the fields of index row r whose main index lies in [4096 s, 4096 (s+1)) and whose
     original feature perm[c] lies in [TCW t, TCW (t+1)), in any order (the builders order them so
     that 8 consecutive entries hit 8 different 16-byte bank groups), as 32-bit entries
       (main index & 4095) | (perm[c] - TCW t) << 12 | residual index << 24,
     padded with zero words to whole steps of 32 entries; every unit has at least one step.
       lists_stream  uint32 [T][32], units in increasing u, 16-byte aligned
       lists_tab     uint32 [U + 1]: tab[u] = first step of unit u | (number of valid entries in the
                     unit's LAST step, 0..32) << 26;  tab[U] = T
     vptq_b200.native.make_desc(lists=True) (GPU, torch) and vptq_b200_lists_build_host (CPU) build
     them; perm is folded in, so the kernel never reads `perm`. */
  const uint32_t* lists_stream;
  const uint32_t* lists_tab;
  int32_t lists_tile_cols;
  int32_t lists_reserved;
} vptq_linear_desc;

typedef enum vptq_op {
  VPTQ_OP_GEMV = 0,    /* vptq_b200_quant_gemv    */
  VPTQ_OP_DEQUANT = 1, /* vptq_b200_dequant       */
  VPTQ_OP_GEMM = 2,    /* vptq_b200_quant_gemm    */
  VPTQ_OP_GEMV_V2 = 3, /* vptq_b200_quant_gemv_v2 */
  VPTQ_OP_GEMM_DGRAD = 4 /* vptq_b200_quant_gemm with VPTQ_FLAG_TRANSPOSE */
} vptq_op;

/* Developer aid (not needed by any caller): when given a device buffer of 32 uint64, every GEMV
   launched afterwards records %globaltimer stamps of its phases (first and last CTA) there;
   NULL switches it off again.  See tools/profile_gemv.py --phases. */
VPTQ_B200_API void vptq_b200_debug_phase_stamps(void* device_buffer);

/* Library / device probing.  No GPU work. */
VPTQ_B200_API int vptq_b200_abi_version(void);
VPTQ_B200_API const char* vptq_b200_last_error(void);
/* Bytes of zero-initialised device workspace `op` needs for this layer and token count. */
VPTQ_B200_API size_t vptq_b200_workspace_bytes(const vptq_linear_desc* desc, int32_t tokens, int32_t op);

/*
 * Decode path: y[t][o] = sum_f x[t][f] * W[o][f] + bias[o], W never materialised.
 * Replaces vptq::wquant_act16_gemv (csrc/quant_gemv.cu:241-294) + its `sum(-1)` epilogue
 * (:235).  x: [tokens][x_stride] elements, y: [tokens][y_stride] elements (strides >= I / O).
 * Any tokens >= 1 is accepted (processed in passes of <= 4); the reference routes
 * tokens < 3 here (vptq/ops/quant_gemm.py:213).
 */
VPTQ_B200_API int vptq_b200_quant_gemv(const vptq_linear_desc* desc, const void* x, int64_t x_stride, void* y,
                         int64_t y_stride, int32_t tokens, void* workspace,
                         size_t workspace_bytes, uint32_t flags, void* stream);

/*
 * Host-side builder of the slice x tile lists of ONE layer (vptq_linear_desc::lists_stream / ::lists_tab)
 * for hosts that do not use vptq_b200.native: plain CPU code, no GPU work.  Reads the packed index
 * words [Ro][index_stride_row] of a one-codebook layer and its perm (uint16 [I], NULL = identity) from
 * HOST memory and writes HOST buffers the caller uploads (stream 16-byte aligned on the device).
 * tab_out must hold (K / 4096) * ceil(I / tile_cols) * ceil(O / 8) + 1 words; *tile_cols_out receives
 * lists_tile_cols.  With stream_out == NULL only tab_out, *steps_out and *tile_cols_out are produced
 * (sizing call: stream bytes = *steps_out * 128).  Byte-identical to vptq_b200.lists.build_lists.
 */
VPTQ_B200_API int vptq_b200_lists_build_host(const int32_t* indices_host, int64_t index_stride_row,
                                             int32_t out_features, int32_t in_features, int32_t num_centroids,
                                             int32_t num_res_centroids, const uint16_t* perm_host,
                                             void* stream_out, size_t stream_capacity, uint32_t* tab_out,
                                             size_t* steps_out, int32_t* tile_cols_out);

/*
 * Optional second load-time pass over built lists (HOST memory, in place; CPU threads, 0 = all cores):
 * re-orders the entries INSIDE every list -- the kernel's result does not depend on that order, its
 * shared-memory bank conflicts do.  Per 32-entry step the entries are chosen so that each quarter-warp
 * reads 8 different 16-byte codebook bank groups (index & 7) and, as far as a bipartite matching
 * allows, the 32 lanes read 32 different x' banks ((column >> 1) & 31).  vptq_b200.lists.build_lists
 * applies it by default (VPTQ_B200_LISTS_DEAL=0 skips it); a host using vptq_b200_lists_build_host
 * calls it on (stream_out, tab_out) before uploading.  units = number of lists (tab has units + 1 words).
 */
VPTQ_B200_API int vptq_b200_lists_deal_host(uint32_t* stream_host, const uint32_t* tab_host, int64_t units,
                                            int32_t threads);

/*
 * Decode path, horizontally fused: up to 4 layers that read the SAME x (q/k/v, gate/up of a
 * decoder layer) in ONE launch -- y_l = x W_l^T + bias_l for every l.  No reference counterpart
 * (the reference launches each VQuantLinear separately); identical results to n separate
 * vptq_b200_quant_gemv calls.  tokens <= 2, vector_len 8.  Returns VPTQ_ERR_UNSUPPORTED when the
 * layers do not admit one launch configuration: the caller then launches them one by one.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_multi(int32_t n, const vptq_linear_desc* const* descs, const void* x,
                                             int64_t x_stride, void* const* ys, const int64_t* y_strides,
                                             int32_t tokens, uint32_t flags, void* stream);

/* Same, with a workspace (zero-initialised once, size >= the sum of vptq_b200_workspace_bytes(desc_l,
 * tokens, VPTQ_OP_GEMV) over the layers).  Needed for the list-based decode kernel (layers carrying
 * lists_stream reduce their per-combo partial sums through it); without a workspace such layers run the
 * generic kernel.  Same results up to fp32 summation order. */
VPTQ_B200_API int vptq_b200_quant_gemv_multi_ws(int32_t n, const vptq_linear_desc* const* descs, const void* x,
                                                int64_t x_stride, void* const* ys, const int64_t* y_strides,
                                                int32_t tokens, void* workspace, size_t workspace_bytes,
                                                uint32_t flags, void* stream);

/*
 * Tensor-parallel decode with the exchange fused into the kernel (no NCCL call, no memset):
 * every rank passes pointers to the SAME y slice inside every rank's full-width output buffer
 * (peer-mapped device memory: CUDA IPC / symmetric memory, peer access enabled by the caller).
 * The kernel stores each output value locally and into all peers over NVLink; the last CTA
 * publishes this launch's epoch in every peer's flag array; a launch with wait_slot >= 0 polls
 * the flags of the launch that produced its x before reading it.  All ranks must issue the same
 * sequence of launches; `slot` identifies a launch position within one token (static under CUDA
 * graphs: the epochs live in device memory).  `workspace` as for vptq_b200_quant_gemv_multi_ws (may be NULL:
 * layers carrying index lists then run the generic kernel).  A flag wait that does not complete within ~2 s
 * sets *error (the outputs of that token are then undefined; later waits return at once): the host must check
 * it.  No reference counterpart.
 *
 * Checked before any descriptor (VPTQ_ERR_INVALID): 0 <= slot < num_slots and -1 <= wait_slot < num_slots for both
 * formats (epoch, done and the flag arrays hold num_slots entries); VPTQ_TP_TAGGED: ys[l] and every non-NULL
 * peer_y[l][r] 16-byte aligned; VPTQ_TP_PLAIN: every non-NULL peer_y[l][r] at the same address modulo 16 bytes as
 * ys[l] (the kernels store 16-byte vectors to peer_y[l][r] + o wherever ys[l] + o is aligned).
 * world == 1 is an exchange like any other: the launch stores its tagged words (into peer_y[l][0]), advances its
 * epochs and is refused on the generic route in the tagged format exactly as rank 0 of a larger world, so the same
 * chain, vptq_b200_tp_untag included, runs on one GPU.
 * The epoch counters wrap at 2^32: flag waits compare serial numbers (int32_t(flag - want) < 0), and the tags are
 * uint32 arithmetic, so a chain may run indefinitely.
 *
 * Two wire formats (vptq_tp_exchange::format):
 *   VPTQ_TP_PLAIN   16-bit outputs stored as they are + one epoch flag per (launch, source rank); the producer
 *                   needs two system-scope fences per launch (data before flag), ~8 us per dependent launch.
 *   VPTQ_TP_TAGGED  every pair of 16-bit outputs travels in one 8-byte word {2 values, 32-bit tag}, tag =
 *                   run * num_slots + slot + 1 of the producing launch; an aligned 8-byte store is atomic, so the
 *                   consumer simply re-reads a word until its tag is the one it expects: no fence, no flag, one
 *                   NVLink one-way latency (the idea of NCCL's LL protocol).  peer_y[l][r] then points at THIS
 *                   rank's slice inside rank r's TAGGED buffer (4 bytes per output; entry [rank] = the local
 *                   one, also written), and a launch with wait_slot >= 0 takes `x` = its local tagged buffer
 *                   (in_features / 2 words).  ys[l] still receives the plain local slice.  Only for launches
 *                   whose layers all carry index lists (list kernel), one token, out_features % 8 == 0.
 *                   Buffer reuse is safe without any handshake as long as every launch of the chain waits for
 *                   the launch that produced its x (wait_slot) and a buffer written by slot n is read only by
 *                   slot n + 1: a rank that is about to overwrite the buffer (at slot n + k, k >= 2, of the same
 *                   or the next token) has waited for the outputs of slot n + k - 1 >= n + 1 of EVERY rank, and
 *                   a rank produces those only after its own launch n + 1 -- the reader -- has completed.
 */
#define VPTQ_TP_PLAIN 0
#define VPTQ_TP_TAGGED 1
#define VPTQ_MAX_FUSED 4
#define VPTQ_MAX_RANKS 8
typedef struct vptq_tp_exchange {
  uint32_t struct_size;
  int32_t world, rank;
  int32_t slot;      /* this launch's position in the token, 0 <= slot < num_slots */
  int32_t wait_slot; /* launch whose outputs are this launch's x; -1: x is local (replicated) */
  void* peer_y[VPTQ_MAX_FUSED][VPTQ_MAX_RANKS]; /* [layer][rank]: start of THIS rank's slice in rank r's y */
  uint32_t* peer_flags[VPTQ_MAX_RANKS];         /* rank r's flag array, uint32 [num_slots][world] */
  uint32_t* epoch;   /* local uint32 [num_slots], zero-initialised once */
  uint32_t* done;    /* local uint32 [num_slots], zero-initialised once */
  uint32_t* error;   /* local uint32, set to 1 when a flag wait timed out (~2 s) */
  int32_t format;    /* VPTQ_TP_PLAIN or VPTQ_TP_TAGGED */
  int32_t num_slots; /* launches per token: entries of epoch / done / the flag arrays; tag arithmetic */
} vptq_tp_exchange;

VPTQ_B200_API int vptq_b200_quant_gemv_multi_tp(int32_t n, const vptq_linear_desc* const* descs, const void* x,
                                                int64_t x_stride, void* const* ys, const int64_t* y_strides,
                                                int32_t tokens, const vptq_tp_exchange* tp, void* workspace,
                                                size_t workspace_bytes, uint32_t flags, void* stream);

/*
 * VPTQ_TP_TAGGED only: copy the full-width output of the launch described by `tp` (its exchange struct) from this
 * rank's tagged buffer (n outputs, 4 bytes each) into plain 16-bit values y[n], waiting until every rank's words
 * of that launch's latest run have arrived.  Enqueue it behind the producing launch on the same stream: this is
 * how the LAST activation of a tensor-parallel chain (which no tagged consumer reads) becomes an ordinary tensor.
 */
VPTQ_B200_API int vptq_b200_tp_untag(const void* tagged, void* y, int32_t n, const vptq_tp_exchange* tp, void* stream);

/*
 * W[o][f] (row-major [O][I], `dtype`), scale/bias/perm applied -- what the reference's dequant
 * returns (csrc/dequant.cu:227-287, Return_OUF_x_INF=true; python spec
 * vptq/ops/quant_gemm.py:43-158).
 */
VPTQ_B200_API int vptq_b200_dequant(const vptq_linear_desc* desc, void* w_out, void* workspace,
                      size_t workspace_bytes, void* stream);

/*
 * Prefill path: y = x W^T + bias for many tokens (replaces dequant + torch F.linear,
 * vptq/ops/quant_gemm.py:231-275): the quantised weight is dequantised once into the workspace (16-bit,
 * quantised column order, scale / bias / perm kept out of it) and fed by TMA to a wgmma tensor-core
 * GEMM with register accumulators.
 * With VPTQ_FLAG_TRANSPOSE: the input gradient dX = dY . W of the layer (x = dY [tokens][out_features],
 * y = dX [tokens][in_features], no bias) through a transposed dequant W^T[in][out] in the workspace (original
 * feature order, scale / bias folded in, bit-identical to the transpose of vptq_b200_dequant's W) and the same
 * GEMM.  Gradients of the codebooks, scale and bias vectors: include/vptq_b200_grad.h.
 */
VPTQ_B200_API int vptq_b200_quant_gemm(const vptq_linear_desc* desc, const void* x, int64_t x_stride, void* y,
                         int64_t y_stride, int32_t tokens, void* workspace,
                         size_t workspace_bytes, uint32_t flags, void* stream);

/*
 * The reference's second GEMV op with UNPACKED indices (csrc/quant_gemv_v2.cu:25-180; layout
 * pinned by tests/test_quant_gemv.py:86-105): indices u16 [Ro][I], residual_indices u8
 * (res_index_bytes == 1) or u16 (== 2) [Ro][I] or NULL, scale_weights/scale_bias [I] or NULL,
 * one codebook, no perm, no outliers.
 */
VPTQ_B200_API int vptq_b200_quant_gemv_v2(int32_t dtype, const void* x, void* y, int32_t tokens,
                            int32_t in_features, int32_t out_features, int32_t vector_len,
                            int32_t num_centroids, int32_t num_res_centroids,
                            const uint16_t* indices, const void* centroids,
                            const void* residual_indices, int32_t res_index_bytes,
                            const void* residual_centroids, const void* scale_weights,
                            const void* scale_bias, const void* bias, void* workspace,
                            size_t workspace_bytes, uint32_t flags, void* stream);

/*
 * End-to-end helper used by the `e2e` measurement: x_host -> (H2D) -> GEMV/GEMM -> (D2H) ->
 * y_host on `stream`, then a stream synchronise.  x_dev / y_dev are caller-provided device
 * staging buffers ([tokens][I] / [tokens][O]); host buffers should be pinned.
 */
VPTQ_B200_API int vptq_b200_linear_host(const vptq_linear_desc* desc, const void* x_host, void* y_host,
                          int32_t tokens, void* x_dev, void* y_dev, void* workspace,
                          size_t workspace_bytes, uint32_t flags, void* stream);

/* Workspace helpers for hosts that capture CUDA graphs: include/vptq_b200_graph.h. */

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_H_ */
