/*
 * vptq_b200_graph.h  --  CUDA-graph helpers of libvptq_b200.so, exported from the same library as
 * include/vptq_b200.h.  The inference ABI (its symbols, VPTQ_B200_ABI_VERSION, vptq_linear_desc) is unchanged by
 * them.  A library without these symbols fails at symbol lookup.
 *
 * Why a host needs them: every entry point of include/vptq_b200.h takes a workspace whose head must be zero when a
 * kernel starts, and kernels leave it zeroed.  A workspace allocated and zero-filled INSIDE a stream capture is
 * zeroed only when that graph replays its recorded fill, so it must stay private to that one graph: no eager call
 * and no other capture may use it.  Telling captures apart needs the capture's id, which this header provides.
 */
#ifndef VPTQ_B200_GRAPH_H_
#define VPTQ_B200_GRAPH_H_

#include "vptq_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * Is `stream` (a cudaStream_t passed as void*; NULL = legacy default stream) capturing a CUDA graph right now?
 * Returns 1 and sets *id to the capture's id (unique in the process, cudaStreamGetCaptureInfo) when it is, 0 and
 * *id = 0 when it is not, and a negative vptq_status on error (VPTQ_ERR_INVALID for id == NULL, VPTQ_ERR_CUDA when
 * the CUDA runtime fails, e.g. without a device).  Enqueues nothing and does not synchronise.
 */
VPTQ_B200_API int vptq_b200_stream_capture_id(void* stream, uint64_t* id);

#ifdef __cplusplus
}
#endif
#endif /* VPTQ_B200_GRAPH_H_ */
