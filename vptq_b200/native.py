"""ctypes binding of libvptq_b200.so (the C ABI declared in include/vptq_b200.h).

This is the only bridge between the Python surface and the CUDA kernels.  There is no other
implementation behind it: if the shared library is missing or a call fails, a RuntimeError is
raised -- no CPU path, no torch fallback (the reference silently falls back to a torch
implementation when its extension is absent, vptq/ops/quant_gemm.py:20-40; this package does not).
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional

import torch

from . import lists as _lists

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VPTQ_B200_LIB") or os.path.join(_HERE, "libvptq_b200.so")   # (env: developer builds)

VPTQ_FP16, VPTQ_BF16 = 0, 1
OP_GEMV, OP_DEQUANT, OP_GEMM, OP_GEMV_V2, OP_GEMM_DGRAD = 0, 1, 2, 3, 4
FLAG_PDL, FLAG_TRANSPOSE = 1, 2
TP_PLAIN, TP_TAGGED = 0, 1
ABI_VERSION = 7
LISTS_DEFAULT = "1"   # VPTQ_B200_LISTS when unset

EXPORTS = (
    "vptq_b200_abi_version", "vptq_b200_last_error", "vptq_b200_workspace_bytes", "vptq_b200_quant_gemv",
    "vptq_b200_dequant", "vptq_b200_quant_gemm", "vptq_b200_quant_gemv_v2", "vptq_b200_linear_host",
    "vptq_b200_debug_phase_stamps", "vptq_b200_quant_gemv_multi", "vptq_b200_quant_gemv_multi_tp",
    "vptq_b200_lists_build_host", "vptq_b200_quant_gemv_multi_ws", "vptq_b200_tp_untag", "vptq_b200_lists_deal_host",
)

# CUDA-graph helpers (include/vptq_b200_graph.h), exported from the same library
GRAPH_EXPORTS = ("vptq_b200_stream_capture_id",)

# training entry points (include/vptq_b200_grad.h), exported from the same library
GRAD_EXPORTS = ("vptq_b200_grad_version", "vptq_b200_grad_workspace_bytes", "vptq_b200_quant_gemm_wgrad",
                "vptq_b200_dequant_backward")
GRAD_VERSION = 1
GRAD_OP_WGRAD, GRAD_OP_DEQUANT_BACKWARD, GRAD_OP_WGRAD_GENERIC = 0, 1, 2
GRAD_FLAG_GENERIC = 1

# batched decode from the index lists (include/vptq_b200_batch.h), exported from the same library
BATCH_EXPORTS = ("vptq_b200_batch_version", "vptq_b200_quant_gemv_batch_max_tokens", "vptq_b200_quant_gemv_batch")
BATCH_VERSION = 1

# prefill, dequant and input gradient from the index lists (include/vptq_b200_lists_dense.h), same library
LISTS_DENSE_EXPORTS = ("vptq_b200_lists_dense_version", "vptq_b200_lists_dense_workspace_bytes",
                       "vptq_b200_lists_dequant", "vptq_b200_lists_quant_gemm")
LISTS_DENSE_VERSION = 1

# decode from the index lists of vector-length-16 layers (include/vptq_b200_lists16.h), same library
LISTS16_EXPORTS = ("vptq_b200_lists16_version", "vptq_b200_quant_gemv_lists16_max_tokens",
                   "vptq_b200_quant_gemv_lists16", "vptq_b200_lists16_build_host")
LISTS16_VERSION = 1
LISTS16_WORKSPACE_BYTES = 65536 * 4 + 65536 * 64

MAX_FUSED, MAX_RANKS = 4, 8


class TpExchange(ctypes.Structure):
    """struct vptq_tp_exchange (include/vptq_b200.h)."""
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("world", ctypes.c_int32), ("rank", ctypes.c_int32),
        ("slot", ctypes.c_int32), ("wait_slot", ctypes.c_int32),
        ("peer_y", (ctypes.c_void_p * MAX_RANKS) * MAX_FUSED), ("peer_flags", ctypes.c_void_p * MAX_RANKS),
        ("epoch", ctypes.c_void_p), ("done", ctypes.c_void_p), ("error", ctypes.c_void_p),
        ("format", ctypes.c_int32), ("num_slots", ctypes.c_int32),
    ]


class LinearDesc(ctypes.Structure):
    """struct vptq_linear_desc (include/vptq_b200.h)."""
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("dtype", ctypes.c_int32),
        ("in_features", ctypes.c_int32), ("out_features", ctypes.c_int32),
        ("vector_len", ctypes.c_int32), ("num_centroids", ctypes.c_int32),
        ("num_res_centroids", ctypes.c_int32), ("num_codebooks", ctypes.c_int32),
        ("group_size", ctypes.c_int32), ("outlier_size", ctypes.c_int32),
        ("outlier_vector_len", ctypes.c_int32), ("num_outlier_centroids", ctypes.c_int32),
        ("indices", ctypes.c_void_p), ("index_stride_codebook", ctypes.c_int64),
        ("index_stride_row", ctypes.c_int64),
        ("centroids", ctypes.c_void_p), ("centroid_stride", ctypes.c_int64),
        ("res_centroids", ctypes.c_void_p), ("res_centroid_stride", ctypes.c_int64),
        ("outlier_indices", ctypes.c_void_p), ("outlier_centroids", ctypes.c_void_p),
        ("perm", ctypes.c_void_p), ("weight_scale", ctypes.c_void_p), ("weight_bias", ctypes.c_void_p),
        ("bias", ctypes.c_void_p), ("weight_scale_q", ctypes.c_void_p), ("weight_bias_q", ctypes.c_void_p),
        ("lists_stream", ctypes.c_void_p), ("lists_tab", ctypes.c_void_p),
        ("lists_tile_cols", ctypes.c_int32), ("lists_reserved", ctypes.c_int32),
    ]


class LinearGrads(ctypes.Structure):
    """struct vptq_linear_grads (include/vptq_b200_grad.h): one output pointer per gradient, NULL = not wanted."""
    _fields_ = [
        ("struct_size", ctypes.c_uint32), ("reserved", ctypes.c_uint32),
        ("centroids", ctypes.c_void_p), ("res_centroids", ctypes.c_void_p), ("outlier_centroids", ctypes.c_void_p),
        ("weight_scale", ctypes.c_void_p), ("weight_bias", ctypes.c_void_p),
    ]


GRAD_FIELDS = ("centroids", "res_centroids", "outlier_centroids", "weight_scale", "weight_bias")

_lib = None
_lock = threading.Lock()


def lib() -> ctypes.CDLL:
    """Load the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m vptq_b200.build` "
                "(vptq_b200 has no CPU or torch fallback)")
        L = ctypes.CDLL(LIB_PATH)
        L.vptq_b200_abi_version.restype = ctypes.c_int
        L.vptq_b200_last_error.restype = ctypes.c_char_p
        L.vptq_b200_workspace_bytes.restype = ctypes.c_size_t
        L.vptq_b200_workspace_bytes.argtypes = [ctypes.POINTER(LinearDesc), ctypes.c_int32, ctypes.c_int32]
        vp, i64, i32, u32, sz = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_uint32, ctypes.c_size_t
        dp = ctypes.POINTER(LinearDesc)
        L.vptq_b200_quant_gemv.argtypes = [dp, vp, i64, vp, i64, i32, vp, sz, u32, vp]
        L.vptq_b200_quant_gemm.argtypes = [dp, vp, i64, vp, i64, i32, vp, sz, u32, vp]
        L.vptq_b200_dequant.argtypes = [dp, vp, vp, sz, vp]
        L.vptq_b200_quant_gemv_v2.argtypes = [i32, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, i32, vp, vp,
                                              vp, vp, vp, sz, u32, vp]
        L.vptq_b200_linear_host.argtypes = [dp, vp, vp, i32, vp, vp, vp, sz, u32, vp]
        L.vptq_b200_quant_gemv_multi.argtypes = [i32, ctypes.POINTER(dp), vp, i64, ctypes.POINTER(vp),
                                                 ctypes.POINTER(i64), i32, u32, vp]
        L.vptq_b200_quant_gemv_multi.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_multi_ws.argtypes = [i32, ctypes.POINTER(dp), vp, i64, ctypes.POINTER(vp),
                                                    ctypes.POINTER(i64), i32, vp, sz, u32, vp]
        L.vptq_b200_quant_gemv_multi_ws.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_multi_tp.argtypes = [i32, ctypes.POINTER(dp), vp, i64, ctypes.POINTER(vp),
                                                    ctypes.POINTER(i64), i32, ctypes.POINTER(TpExchange), vp, sz, u32, vp]
        L.vptq_b200_quant_gemv_multi_tp.restype = ctypes.c_int
        L.vptq_b200_lists_build_host.argtypes = [vp, i64, i32, i32, i32, i32, vp, vp, sz, vp, ctypes.POINTER(sz),
                                                 ctypes.POINTER(i32)]
        L.vptq_b200_lists_build_host.restype = ctypes.c_int
        L.vptq_b200_lists_deal_host.argtypes = [vp, vp, i64, i32]
        L.vptq_b200_lists_deal_host.restype = ctypes.c_int
        L.vptq_b200_tp_untag.argtypes = [vp, vp, i32, ctypes.POINTER(TpExchange), vp]
        L.vptq_b200_tp_untag.restype = ctypes.c_int
        L.vptq_b200_debug_phase_stamps.argtypes = [vp]
        L.vptq_b200_debug_phase_stamps.restype = None
        for f in GRAPH_EXPORTS:
            if not hasattr(L, f):
                raise RuntimeError(f"{LIB_PATH} lacks {f} (include/vptq_b200_graph.h): rebuild it")
        L.vptq_b200_stream_capture_id.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64)]
        L.vptq_b200_stream_capture_id.restype = ctypes.c_int
        for f in ("vptq_b200_quant_gemv", "vptq_b200_quant_gemm", "vptq_b200_dequant", "vptq_b200_quant_gemv_v2",
                  "vptq_b200_linear_host"):
            getattr(L, f).restype = ctypes.c_int
        if L.vptq_b200_abi_version() != ABI_VERSION:
            raise RuntimeError(f"libvptq_b200.so ABI {L.vptq_b200_abi_version()} != expected {ABI_VERSION}")
        for f in GRAD_EXPORTS:
            if not hasattr(L, f):
                raise RuntimeError(f"{LIB_PATH} lacks {f} (include/vptq_b200_grad.h): rebuild it")
        gp = ctypes.POINTER(LinearGrads)
        L.vptq_b200_grad_version.restype = ctypes.c_int
        L.vptq_b200_grad_workspace_bytes.restype = ctypes.c_size_t
        L.vptq_b200_grad_workspace_bytes.argtypes = [dp, i32, i32]
        L.vptq_b200_quant_gemm_wgrad.argtypes = [dp, vp, i64, vp, i64, i32, gp, vp, sz, u32, vp]
        L.vptq_b200_quant_gemm_wgrad.restype = ctypes.c_int
        L.vptq_b200_dequant_backward.argtypes = [dp, vp, i64, gp, vp, sz, u32, vp]
        L.vptq_b200_dequant_backward.restype = ctypes.c_int
        if L.vptq_b200_grad_version() != GRAD_VERSION:
            raise RuntimeError(f"libvptq_b200.so grad interface {L.vptq_b200_grad_version()} != expected {GRAD_VERSION}")
        for f in BATCH_EXPORTS:
            if not hasattr(L, f):
                raise RuntimeError(f"{LIB_PATH} lacks {f} (include/vptq_b200_batch.h): rebuild it")
        L.vptq_b200_batch_version.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_batch_max_tokens.argtypes = [i32, ctypes.POINTER(dp)]
        L.vptq_b200_quant_gemv_batch_max_tokens.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_batch.argtypes = [i32, ctypes.POINTER(dp), vp, i64, ctypes.POINTER(vp), ctypes.POINTER(i64),
                                                 i32, vp, sz, u32, vp]
        L.vptq_b200_quant_gemv_batch.restype = ctypes.c_int
        if L.vptq_b200_batch_version() != BATCH_VERSION:
            raise RuntimeError(f"libvptq_b200.so batch interface {L.vptq_b200_batch_version()} != expected {BATCH_VERSION}")
        for f in LISTS_DENSE_EXPORTS:
            if not hasattr(L, f):
                raise RuntimeError(f"{LIB_PATH} lacks {f} (include/vptq_b200_lists_dense.h): rebuild it")
        L.vptq_b200_lists_dense_version.restype = ctypes.c_int
        L.vptq_b200_lists_dense_workspace_bytes.argtypes = [dp, i32, u32]
        L.vptq_b200_lists_dense_workspace_bytes.restype = ctypes.c_size_t
        L.vptq_b200_lists_dequant.argtypes = [dp, vp, i64, u32, vp]
        L.vptq_b200_lists_dequant.restype = ctypes.c_int
        L.vptq_b200_lists_quant_gemm.argtypes = [dp, vp, i64, vp, i64, i32, vp, sz, u32, vp]
        L.vptq_b200_lists_quant_gemm.restype = ctypes.c_int
        if L.vptq_b200_lists_dense_version() != LISTS_DENSE_VERSION:
            raise RuntimeError(f"libvptq_b200.so lists-dense interface {L.vptq_b200_lists_dense_version()} != expected "
                               f"{LISTS_DENSE_VERSION}")
        for f in LISTS16_EXPORTS:
            if not hasattr(L, f):
                raise RuntimeError(f"{LIB_PATH} lacks {f} (include/vptq_b200_lists16.h): rebuild it")
        L.vptq_b200_lists16_version.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_lists16_max_tokens.argtypes = [i32, ctypes.POINTER(dp)]
        L.vptq_b200_quant_gemv_lists16_max_tokens.restype = ctypes.c_int
        L.vptq_b200_quant_gemv_lists16.argtypes = [i32, ctypes.POINTER(dp), vp, i64, ctypes.POINTER(vp),
                                                   ctypes.POINTER(i64), i32, vp, sz, u32, vp]
        L.vptq_b200_quant_gemv_lists16.restype = ctypes.c_int
        L.vptq_b200_lists16_build_host.argtypes = L.vptq_b200_lists_build_host.argtypes
        L.vptq_b200_lists16_build_host.restype = ctypes.c_int
        if L.vptq_b200_lists16_version() != LISTS16_VERSION:
            raise RuntimeError(f"libvptq_b200.so lists16 interface {L.vptq_b200_lists16_version()} != expected "
                               f"{LISTS16_VERSION}")
        _lib = L
    return _lib


def last_error() -> str:
    return lib().vptq_b200_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (status {rc}): {last_error()}")


def dtype_code(dt: torch.dtype) -> int:
    if dt == torch.float16:
        return VPTQ_FP16
    if dt == torch.bfloat16:
        return VPTQ_BF16
    raise RuntimeError(f"vptq_b200 supports float16 and bfloat16 tensors only, got {dt}")


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def require_cuda(name: str, t: Optional[torch.Tensor], contiguous: bool = True) -> None:
    """The reference's CHECK_INPUT (csrc/util/common.h:11-19): CUDA + contiguous."""
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (vptq_b200 has no CPU path)")
    if contiguous and not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")


_sm_counts: dict = {}


def _sm_count(device: torch.device) -> int:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _sm_counts:
        _sm_counts[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _sm_counts[idx]


def make_desc(*, dtype: torch.dtype, in_features: int, out_features: int, vector_len: int, num_centroids: int,
              num_res_centroids: int, num_codebooks: int, group_size: int, outlier_size: int,
              outlier_vector_len: int, num_outlier_centroids: int, indices: torch.Tensor,
              centroids: torch.Tensor, res_centroids: Optional[torch.Tensor],
              outlier_indices: Optional[torch.Tensor], outlier_centroids: Optional[torch.Tensor],
              perm: Optional[torch.Tensor], weight_scale: Optional[torch.Tensor],
              weight_bias: Optional[torch.Tensor], bias: Optional[torch.Tensor],
              derive: bool = True, lists: Optional[bool] = None, drop_packed: bool = False,
              lists16: bool = False, lists_prefill: bool = False) -> LinearDesc:
    """Describe one layer's tensors for the C ABI.  Tensors are borrowed: keep them alive.

    With `derive` (default) the load-time derivatives the ABI accepts are built here, once:
    weight_scale / weight_bias in quantised column order (`t[perm]`).  They hang off the returned
    descriptor (`desc._keep`) so they live as long as it does.

    `lists`: also build the slice x tile index lists (vptq_b200.lists) that let single-token calls of
    large-codebook layers gather from shared memory; costs 4 bytes per index (+ ~6 % padding) on top
    of the packed words (3 bytes per index for the 65536+256 configuration).  None = the
    VPTQ_B200_LISTS environment variable (default on); ignored for layers the list kernel does not cover.

    `lists16`: build the index lists of a vector-length-16 layer (index rows of 16 outputs) for
    include/vptq_b200_lists16.h: 4.25 bytes per index on top of the packed words.  Opt-in only
    (VQuantLinear.set_list_decode); ignored for layers that kernel does not cover.

    `drop_packed`: decode-only descriptor -- once the lists are built the descriptor forgets the packed words
    (`indices` = NULL), so the caller may free them: 4.2 instead of 7.2 bytes per index.  Multi-token calls,
    dequant and prefill then return VPTQ_ERR_UNSUPPORTED.  Refused for layers without lists.  A vector-length-16
    layer (`lists16`) becomes decode-only only with `lists_prefill` (VQuantLinear.set_lists_prefill), whose routes
    (include/vptq_b200_lists_dense.h) serve every call its list kernel does not: 4.25 instead of 7.25 bytes per
    index.  Refused when its lists take no token count (lists16_max_tokens 0).
    """
    if indices.dtype != torch.int32:
        raise RuntimeError("`indices` must be packed int32 words (is_indice_packed=True); "
                           "see vptq_b200.pack.pack_index")
    for n, t in (("indices", indices), ("centroids", centroids), ("res_centroids", res_centroids),
                 ("outlier_indices", outlier_indices), ("outlier_centroids", outlier_centroids), ("perm", perm),
                 ("weight_scale", weight_scale), ("weight_bias", weight_bias), ("bias", bias)):
        require_cuda(n, t)
    if indices.dim() != 3:
        raise RuntimeError(f"indices must be [num_codebooks, num_indices, packed_groupsize], got {tuple(indices.shape)}")
    use_outlier = outlier_indices is not None and outlier_centroids is not None and outlier_size > 0
    d = LinearDesc()
    d.struct_size = ctypes.sizeof(LinearDesc)
    d.dtype = dtype_code(dtype)
    d.in_features, d.out_features = int(in_features), int(out_features)
    d.vector_len, d.num_centroids = int(vector_len), int(num_centroids)
    d.num_res_centroids = int(num_res_centroids) if res_centroids is not None else -1
    d.num_codebooks, d.group_size = int(num_codebooks), int(group_size)
    d.outlier_size = int(outlier_size) if use_outlier else 0
    d.outlier_vector_len = int(outlier_vector_len)
    d.num_outlier_centroids = int(num_outlier_centroids)
    d.indices = _ptr(indices)
    d.index_stride_codebook, d.index_stride_row = indices.stride(0), indices.stride(1)
    d.centroids = _ptr(centroids)
    d.centroid_stride = int(num_centroids) * int(vector_len)
    d.res_centroids = _ptr(res_centroids)
    d.res_centroid_stride = int(num_res_centroids) * int(vector_len) if res_centroids is not None else 0
    d.outlier_indices = _ptr(outlier_indices) if use_outlier else None
    d.outlier_centroids = _ptr(outlier_centroids) if use_outlier else None
    d.perm = _ptr(perm)
    d.weight_scale, d.weight_bias = _ptr(weight_scale), _ptr(weight_bias)
    d.bias = _ptr(bias)
    d._keep = ()
    if derive and perm is not None and weight_scale is not None and weight_bias is not None:
        # ordinary tensors even when built inside torch.inference_mode(): an optimizer step outside it refreshes them
        # in place (VQuantLinear._refresh_in_place)
        with torch.inference_mode(False), torch.no_grad():
            pidx = perm.view(torch.uint16).to(torch.int64) if perm.dtype in (torch.int16, torch.uint16) else perm.long()
            ws_q, wb_q = weight_scale[pidx].contiguous(), weight_bias[pidx].contiguous()
        d.weight_scale_q, d.weight_bias_q = ws_q.data_ptr(), wb_q.data_ptr()
        d._keep = (ws_q, wb_q)
    if lists is None:
        lists = os.environ.get("VPTQ_B200_LISTS", LISTS_DEFAULT) != "0"
    if lists and derive and _lists.eligible(
            vector_len=d.vector_len, num_centroids=d.num_centroids, num_res_centroids=d.num_res_centroids,
            num_codebooks=d.num_codebooks, outlier_size=d.outlier_size, in_features=d.in_features) and (
            weight_scale is None or (weight_scale.data_ptr() % 16 == 0 and weight_bias.data_ptr() % 16 == 0)) and (
            _lists.launchable(d.in_features, d.num_centroids, _sm_count(indices.device))):
        stream, tab, tcw = _lists.build_lists(indices, num_centroids=d.num_centroids,
                                              num_res_centroids=d.num_res_centroids, in_features=d.in_features,
                                              out_features=d.out_features, perm=perm)
        d.lists_stream, d.lists_tab, d.lists_tile_cols = stream.data_ptr(), tab.data_ptr(), int(tcw)
        d._keep = d._keep + (stream, tab)
    if lists16 and derive and d.vector_len == 16 and _lists.eligible(
            vector_len=d.vector_len, num_centroids=d.num_centroids, num_res_centroids=d.num_res_centroids,
            num_codebooks=d.num_codebooks, outlier_size=d.outlier_size, in_features=d.in_features,
            list_vector_len=16) and (
            weight_scale is None or (weight_scale.data_ptr() % 16 == 0 and weight_bias.data_ptr() % 16 == 0)) and (
            _lists.launchable(d.in_features, d.num_centroids, _sm_count(indices.device))):
        stream, tab, tcw = _lists.build_lists(indices, num_centroids=d.num_centroids,
                                              num_res_centroids=d.num_res_centroids, in_features=d.in_features,
                                              out_features=d.out_features, perm=perm, vector_len=16)
        d.lists_stream, d.lists_tab, d.lists_tile_cols = stream.data_ptr(), tab.data_ptr(), int(tcw)
        d._keep = d._keep + (stream, tab)
    if drop_packed:
        if d.vector_len != 8 and d.lists_stream and not lists_prefill:
            raise RuntimeError("drop_packed: decode-only descriptors exist for vector_len 8 only, unless a "
                               "vector-length-16 layer also opts in to prefill from its lists (set_lists_prefill): "
                               "its list kernel serves single- and few-token decode, not prefill or dequant")
        if not d.lists_stream or (d.vector_len == 16 and lists16_max_tokens(d) == 0):
            raise RuntimeError("drop_packed: this layer has no index lists (not eligible, its slices x column tiles "
                               "exceed the device's SM count, lists=False, or for vector_len 16 no set_list_decode or "
                               "lists its kernel takes at no token count)")
        d.indices = None
    return d


# Zero-initialised workspaces: kernels leave them zeroed (include/vptq_b200.h).  A CUDA graph keeps the addresses
# it was captured with, so no buffer a graph may use is freed before release_workspaces() (DESIGN.md section 1).
_workspaces: dict = {}   # (device, stream) -> the stream's current buffer, zeroed eagerly
_retired: list = []      # buffers replaced by bigger ones: graphs captured earlier still use them
_captured: dict = {}     # (device, stream, capture id) -> buffer allocated inside that capture, private to it


def _grown(old: Optional[torch.Tensor], nbytes: int) -> int:
    # at least doubling: everything retired stays below the size of the largest buffer
    return max(int(nbytes), 1 << 20, 2 * old.numel() if old is not None else 0)


def pick_workspace(key, nbytes: int, capture_id: int, alloc, current: dict, retired: list, captured: dict):
    """The bookkeeping of workspace(), free of CUDA so that it can be tested with fake buffers.

    key: (device, stream); capture_id: the stream's capture id, 0 when it is not capturing; alloc(n): a new
    zero-initialised buffer of n bytes (inside a capture its fill is recorded into the graph, so it runs only when
    that graph replays).  An eagerly zeroed buffer that is big enough serves everyone, captures included.  Otherwise
    a call outside capture replaces it, and a call inside a capture gets a buffer of that capture's own, which no
    eager call or other capture ever sees.  A replaced buffer is retired, never dropped."""
    ws = current.get(key)
    if ws is not None and ws.numel() >= nbytes:
        return ws
    if not capture_id:
        if ws is not None:
            retired.append(ws)
        ws = current[key] = alloc(_grown(ws, nbytes))
        return ws
    ckey = key + (capture_id,)
    pv = captured.get(ckey)
    if pv is not None and pv.numel() >= nbytes:
        return pv
    if pv is not None:
        retired.append(pv)
    pv = captured[ckey] = alloc(_grown(pv, nbytes))
    return pv


def capture_id(stream: int) -> int:
    """The id of the CUDA-graph capture running on `stream` (a cudaStream_t handle), 0 when it is not capturing."""
    cid = ctypes.c_uint64(0)
    rc = lib().vptq_b200_stream_capture_id(stream, ctypes.byref(cid))
    if rc < 0:
        check(rc, "vptq_b200_stream_capture_id")
    return int(cid.value)


def workspace(device: torch.device, nbytes: int) -> torch.Tensor:
    stream = torch.cuda.current_stream(device).cuda_stream
    key = (device.index if device.index is not None else torch.cuda.current_device(), stream)
    ws = _workspaces.get(key)
    if ws is not None and ws.numel() >= nbytes:
        return ws
    return pick_workspace(key, nbytes, capture_id(stream),
                          lambda n: torch.zeros(n, dtype=torch.uint8, device=device), _workspaces, _retired, _captured)


def release_workspaces() -> None:
    """Drop every cached workspace: the streams' current ones, the retired ones and those private to a capture (they
    only grow: a weight-gradient call can leave hundreds of MB).  The next call allocates a fresh zeroed one.  Not
    while a captured CUDA graph still lives: it may use any of them."""
    _workspaces.clear()
    _retired.clear()
    _captured.clear()


def workspace_bytes(desc: LinearDesc, tokens: int, op: int) -> int:
    return int(lib().vptq_b200_workspace_bytes(ctypes.byref(desc), int(tokens), int(op)))


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class _on_device:
    """`with torch.cuda.device(dev)` only when dev is not already current (the context manager costs microseconds on
    a path whose kernel takes ten)."""

    def __init__(self, dev: torch.device):
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        self.ctx = None if idx == torch.cuda.current_device() else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *a):
        if self.ctx is not None:
            self.ctx.__exit__(*a)


def _ws_bytes_cached(desc: LinearDesc, tokens: int, op: int) -> int:
    cache = desc.__dict__.setdefault("_ws_cache", {})
    key = (min(tokens, 4) if op == OP_GEMV else tokens, op)     # the GEMV plans passes of at most 4 tokens
    v = cache.get(key)
    if v is None:
        # ("grad", op): an op of vptq_b200_grad_workspace_bytes
        v = cache[key] = grad_workspace_bytes(desc, tokens, op[1]) if isinstance(op, tuple) else \
            workspace_bytes(desc, tokens, op)
    return v


def row_pitch(t: torch.Tensor) -> int:
    """Row pitch in elements for the C ABI: a one-row tensor may carry any row stride (0 after `expand`)."""
    return t.stride(0) if t.shape[0] > 1 else t.shape[1]


def quant_gemv(desc: LinearDesc, x2d: torch.Tensor, y2d: torch.Tensor, flags: int = 0) -> None:
    dev = x2d.device
    tokens = x2d.shape[0]
    with _on_device(dev):
        ws = workspace(dev, _ws_bytes_cached(desc, tokens, OP_GEMV))
        rc = lib().vptq_b200_quant_gemv(ctypes.byref(desc), x2d.data_ptr(), row_pitch(x2d), y2d.data_ptr(),
                                        row_pitch(y2d), tokens, ws.data_ptr(), ws.numel(), flags, _stream(dev))
    check(rc, "vptq_b200_quant_gemv")


class FusedGemv:
    """Prepared argument arrays for vptq_b200_quant_gemv_multi (layers sharing one input)."""

    def __init__(self, descs, ys):
        n = len(descs)
        if not 1 <= n <= MAX_FUSED or len(ys) != n:
            raise RuntimeError(f"FusedGemv takes 1..{MAX_FUSED} layers with one output each")
        if any(d.in_features != descs[0].in_features or d.dtype != descs[0].dtype for d in descs):
            raise RuntimeError("FusedGemv: the layers must read the same x (same in_features and dtype)")
        self.n, self.descs, self.ys = n, list(descs), list(ys)
        self.desc_arr = (ctypes.POINTER(LinearDesc) * n)(*[ctypes.pointer(d) for d in descs])
        self.y_arr = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
        self.stride_arr = (ctypes.c_int64 * n)(*[y.stride(0) for y in ys])
        self.separate = False
        self.ws_bytes = None

    def __call__(self, x2d: torch.Tensor, flags: int = 0) -> None:
        dev = x2d.device
        if not self.separate:
            with torch.cuda.device(dev):
                if self.ws_bytes is None:
                    self.ws_bytes = sum(workspace_bytes(d, x2d.shape[0], OP_GEMV) for d in self.descs)
                ws = workspace(dev, self.ws_bytes)   # the list kernel reduces its partial sums through it
                rc = lib().vptq_b200_quant_gemv_multi_ws(self.n, self.desc_arr, x2d.data_ptr(), row_pitch(x2d),
                                                         self.y_arr, self.stride_arr, x2d.shape[0], ws.data_ptr(),
                                                         ws.numel(), flags, _stream(dev))
            if rc != -2:                      # VPTQ_ERR_UNSUPPORTED: these layers cannot share one launch
                check(rc, "vptq_b200_quant_gemv_multi")
                return
            self.separate = True              # same kernels, one launch per layer (identical results)
        for d, y in zip(self.descs, self.ys):
            quant_gemv(d, x2d, y, flags)


def _desc_array(descs):
    return (ctypes.POINTER(LinearDesc) * len(descs))(*[ctypes.pointer(d) for d in descs])


def batch_max_tokens(descs) -> int:
    """vptq_b200_quant_gemv_batch_max_tokens: the largest token count the batched list route takes for these layers
    (one descriptor or a list of 1..MAX_FUSED reading the same x) on the current device, 0 when they are not eligible.
    Cached on the first descriptor (the answer depends on the shapes and the device only)."""
    descs = [descs] if isinstance(descs, LinearDesc) else list(descs)
    if not descs or not all(d.lists_stream for d in descs):
        return 0
    idx = torch.cuda.current_device()
    cache = descs[0].__dict__.setdefault("_batch_max", {})
    key = (idx,) + tuple(id(d) for d in descs)
    v = cache.get(key)
    if v is None:
        v = cache[key] = int(lib().vptq_b200_quant_gemv_batch_max_tokens(len(descs), _desc_array(descs)))
    return v


def quant_gemv_batch(desc: LinearDesc, x2d: torch.Tensor, y2d: torch.Tensor, flags: int = 0) -> None:
    """y2d [tokens, O] = x2d [tokens, I] @ W^T + bias by the batched list kernel (vptq_b200_quant_gemv_batch),
    1 <= tokens <= batch_max_tokens(desc)."""
    FusedGemvBatch([desc], [y2d])(x2d, flags)


class FusedGemvBatch:
    """Prepared argument arrays for vptq_b200_quant_gemv_batch (1..MAX_FUSED layers sharing one input, 1..8 tokens).
    No fall-back: a refusal raises."""

    def __init__(self, descs, ys):
        n = len(descs)
        if not 1 <= n <= MAX_FUSED or len(ys) != n:
            raise RuntimeError(f"FusedGemvBatch takes 1..{MAX_FUSED} layers with one output each")
        self.n, self.descs, self.ys = n, list(descs), list(ys)
        self.desc_arr = _desc_array(self.descs)
        self.y_arr = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
        self.stride_arr = (ctypes.c_int64 * n)(*[row_pitch(y) for y in ys])
        self.ws_bytes = None

    def __call__(self, x2d: torch.Tensor, flags: int = 0) -> None:
        dev = x2d.device
        with _on_device(dev):
            if self.ws_bytes is None:
                self.ws_bytes = sum(_ws_bytes_cached(d, 1, OP_GEMV) for d in self.descs)
            ws = workspace(dev, self.ws_bytes)
            rc = lib().vptq_b200_quant_gemv_batch(self.n, self.desc_arr, x2d.data_ptr(), row_pitch(x2d), self.y_arr,
                                                  self.stride_arr, x2d.shape[0], ws.data_ptr(), ws.numel(), flags,
                                                  _stream(dev))
        check(rc, "vptq_b200_quant_gemv_batch")


def lists16_max_tokens(descs) -> int:
    """vptq_b200_quant_gemv_lists16_max_tokens: the largest token count (4, 2 or 1) the vector-length-16 list kernel
    takes for these layers (one descriptor or a list of 1..MAX_FUSED reading the same x) on the current device, 0 when
    they are not eligible.  Cached on the first descriptor (the answer depends on the shapes and the device only)."""
    descs = [descs] if isinstance(descs, LinearDesc) else list(descs)
    if not descs or not all(d.lists_stream and d.vector_len == 16 for d in descs):
        return 0
    idx = torch.cuda.current_device()
    cache = descs[0].__dict__.setdefault("_lists16_max", {})
    key = (idx,) + tuple(id(d) for d in descs)
    v = cache.get(key)
    if v is None:
        v = cache[key] = int(lib().vptq_b200_quant_gemv_lists16_max_tokens(len(descs), _desc_array(descs)))
    return v


def quant_gemv_lists16(desc: LinearDesc, x2d: torch.Tensor, y2d: torch.Tensor, flags: int = 0) -> None:
    """y2d [tokens, O] = x2d [tokens, I] @ W^T + bias by the vector-length-16 list kernel
    (vptq_b200_quant_gemv_lists16), 1 <= tokens <= lists16_max_tokens(desc)."""
    FusedGemvLists16([desc], [y2d])(x2d, flags)


class FusedGemvLists16:
    """Prepared argument arrays for vptq_b200_quant_gemv_lists16 (1..MAX_FUSED vector-length-16 layers sharing one
    input, 1..4 tokens).  No fall-back: a refusal raises."""

    def __init__(self, descs, ys):
        n = len(descs)
        if not 1 <= n <= MAX_FUSED or len(ys) != n:
            raise RuntimeError(f"FusedGemvLists16 takes 1..{MAX_FUSED} layers with one output each")
        self.n, self.descs, self.ys = n, list(descs), list(ys)
        self.desc_arr = _desc_array(self.descs)
        self.y_arr = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
        self.stride_arr = (ctypes.c_int64 * n)(*[row_pitch(y) for y in ys])

    def __call__(self, x2d: torch.Tensor, flags: int = 0) -> None:
        dev = x2d.device
        with _on_device(dev):
            ws = workspace(dev, LISTS16_WORKSPACE_BYTES)
            rc = lib().vptq_b200_quant_gemv_lists16(self.n, self.desc_arr, x2d.data_ptr(), row_pitch(x2d), self.y_arr,
                                                    self.stride_arr, x2d.shape[0], ws.data_ptr(), ws.numel(), flags,
                                                    _stream(dev))
        check(rc, "vptq_b200_quant_gemv_lists16")


class FusedGemvTP:
    """vptq_b200_quant_gemv_multi_tp: fused layers + the tensor-parallel exchange inside the kernel."""

    def __init__(self, descs, ys, exchange: TpExchange):
        n = len(descs)
        self.n, self.descs, self.ys, self.ex = n, list(descs), list(ys), exchange
        self.desc_arr = (ctypes.POINTER(LinearDesc) * n)(*[ctypes.pointer(d) for d in descs])
        self.y_arr = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
        self.stride_arr = (ctypes.c_int64 * n)(*[y.stride(0) for y in ys])
        self.ws_bytes = None

    def __call__(self, x2d: torch.Tensor, flags: int = 0) -> None:
        dev = x2d.device
        with torch.cuda.device(dev):
            if self.ws_bytes is None:
                self.ws_bytes = sum(workspace_bytes(d, x2d.shape[0], OP_GEMV) for d in self.descs)
            ws = workspace(dev, self.ws_bytes)
            rc = lib().vptq_b200_quant_gemv_multi_tp(self.n, self.desc_arr, x2d.data_ptr(), row_pitch(x2d), self.y_arr,
                                                     self.stride_arr, x2d.shape[0], ctypes.byref(self.ex), ws.data_ptr(),
                                                     ws.numel(), flags, _stream(dev))
        check(rc, "vptq_b200_quant_gemv_multi_tp")


def tp_untag(tagged: torch.Tensor, y: torch.Tensor, exchange: TpExchange) -> None:
    """vptq_b200_tp_untag: the full-width output of the (VPTQ_TP_TAGGED) launch `exchange` -> plain values in y."""
    dev = y.device
    with torch.cuda.device(dev):
        rc = lib().vptq_b200_tp_untag(tagged.data_ptr(), y.data_ptr(), y.numel(), ctypes.byref(exchange), _stream(dev))
    check(rc, "vptq_b200_tp_untag")


def quant_gemm(desc: LinearDesc, x2d: torch.Tensor, y2d: torch.Tensor, flags: int = 0) -> None:
    dev = x2d.device
    tokens = x2d.shape[0]
    with _on_device(dev):
        ws = workspace(dev, _ws_bytes_cached(desc, tokens, OP_GEMM))
        rc = lib().vptq_b200_quant_gemm(ctypes.byref(desc), x2d.data_ptr(), row_pitch(x2d), y2d.data_ptr(),
                                        row_pitch(y2d), tokens, ws.data_ptr(), ws.numel(), flags, _stream(dev))
    check(rc, "vptq_b200_quant_gemm")


def quant_gemm_dgrad(desc: LinearDesc, dy2d: torch.Tensor, dx2d: torch.Tensor) -> None:
    """dx2d [tokens, in_features] = dy2d [tokens, out_features] @ W: the layer's input gradient
    (vptq_b200_quant_gemm with VPTQ_FLAG_TRANSPOSE).  Any token count."""
    tokens = dy2d.shape[0]
    if dy2d.stride(-1) != 1 or (tokens > 1 and dy2d.stride(0) < dy2d.shape[1]):
        dy2d = dy2d.contiguous()      # autograd hands over expanded (zero-stride) gradients, e.g. from y.sum()
    dev = dy2d.device
    with _on_device(dev):
        ws = workspace(dev, _ws_bytes_cached(desc, tokens, OP_GEMM_DGRAD))
        rc = lib().vptq_b200_quant_gemm(ctypes.byref(desc), dy2d.data_ptr(), row_pitch(dy2d), dx2d.data_ptr(),
                                        row_pitch(dx2d), tokens, ws.data_ptr(), ws.numel(), FLAG_TRANSPOSE, _stream(dev))
    check(rc, "vptq_b200_quant_gemm (transpose)")


def lists_dense_workspace_bytes(desc: LinearDesc, tokens: int, flags: int = 0) -> int:
    return int(lib().vptq_b200_lists_dense_workspace_bytes(ctypes.byref(desc), int(tokens), int(flags)))


def lists_quant_gemm(desc: LinearDesc, x2d: torch.Tensor, y2d: torch.Tensor, flags: int = 0) -> None:
    """vptq_b200_lists_quant_gemm: y2d = x2d @ W^T + bias (flags 0) or the input gradient y2d = x2d @ W with x2d = dY
    (FLAG_TRANSPOSE), the weight written from the index lists.  Any token count >= 1."""
    x2d = _dense_rows(x2d)
    tokens = x2d.shape[0]
    dev = x2d.device
    with _on_device(dev):
        cache = desc.__dict__.setdefault("_lists_ws", {})
        key = (tokens, flags & FLAG_TRANSPOSE)
        nbytes = cache.get(key)
        if nbytes is None:
            nbytes = cache[key] = lists_dense_workspace_bytes(desc, tokens, flags)
        ws = workspace(dev, max(nbytes, 1))
        rc = lib().vptq_b200_lists_quant_gemm(ctypes.byref(desc), x2d.data_ptr(), row_pitch(x2d), y2d.data_ptr(),
                                              row_pitch(y2d), tokens, ws.data_ptr(), ws.numel(), int(flags),
                                              _stream(dev))
    check(rc, "vptq_b200_lists_quant_gemm" + (" (transpose)" if flags & FLAG_TRANSPOSE else ""))


def lists_dequant(desc: LinearDesc, w: torch.Tensor, ld: int, flags: int = 0) -> None:
    """vptq_b200_lists_dequant into the buffer starting at w: W [out_features][ld] (flags 0) or Wt [in_features][ld]
    (FLAG_TRANSPOSE), written from the index lists; ld a multiple of 8, columns past the weight's zero."""
    dev = w.device
    with _on_device(dev):
        rc = lib().vptq_b200_lists_dequant(ctypes.byref(desc), w.data_ptr(), int(ld), int(flags), _stream(dev))
    check(rc, "vptq_b200_lists_dequant")


def lists_dense_weight(desc: LinearDesc, dtype: torch.dtype, device) -> torch.Tensor:
    """The layer's dense weight [out_features, in_features] from the index lists (a view into rows padded to a
    multiple of 8 elements when in_features is not one)."""
    I, O = desc.in_features, desc.out_features
    ld = (I + 7) // 8 * 8
    buf = torch.empty(O, ld, dtype=dtype, device=device)
    lists_dequant(desc, buf, ld)
    return buf if ld == I else buf[:, :I]


def grad_workspace_bytes(desc: LinearDesc, tokens: int, op: int) -> int:
    return int(lib().vptq_b200_grad_workspace_bytes(ctypes.byref(desc), int(tokens), int(op)))


def make_grads(grads: dict) -> LinearGrads:
    """{field of GRAD_FIELDS: output tensor} -> struct vptq_linear_grads (missing fields = not wanted)."""
    unknown = set(grads) - set(GRAD_FIELDS)
    if unknown:
        raise RuntimeError(f"unknown gradient outputs {sorted(unknown)}; expected some of {GRAD_FIELDS}")
    g = LinearGrads()
    g.struct_size = ctypes.sizeof(LinearGrads)
    for k, t in grads.items():
        if t is not None:
            require_cuda(k, t)
            setattr(g, k, t.data_ptr())
    return g


def _dense_rows(t: torch.Tensor) -> torch.Tensor:
    # autograd hands over expanded (zero-stride) gradients, e.g. from y.sum(): the kernels need pitch >= columns
    if t.stride(-1) != 1 or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
        return t.contiguous()
    return t


def quant_gemm_wgrad(desc: LinearDesc, x2d: torch.Tensor, dy2d: torch.Tensor, grads: dict, flags: int = 0) -> None:
    """Weight gradients of y = x W^T + bias into the tensors of `grads` (vptq_b200_quant_gemm_wgrad):
    x2d [tokens, in_features], dy2d [tokens, out_features].  flags=GRAD_FLAG_GENERIC takes the generic route (G in
    the workspace + scatter kernel) also where the fused GEMM epilogue applies; the results are bit-identical."""
    x2d, dy2d = _dense_rows(x2d), _dense_rows(dy2d)
    tokens = x2d.shape[0]
    if dy2d.shape[0] != tokens:
        raise RuntimeError(f"x has {tokens} rows but dy has {dy2d.shape[0]}")
    g = make_grads(grads)
    dev = dy2d.device
    with _on_device(dev):
        op = GRAD_OP_WGRAD_GENERIC if flags & GRAD_FLAG_GENERIC else GRAD_OP_WGRAD
        ws = workspace(dev, _ws_bytes_cached(desc, tokens, ("grad", op)))
        rc = lib().vptq_b200_quant_gemm_wgrad(ctypes.byref(desc), x2d.data_ptr(), row_pitch(x2d), dy2d.data_ptr(),
                                              row_pitch(dy2d), tokens, ctypes.byref(g), ws.data_ptr(), ws.numel(),
                                              int(flags), _stream(dev))
    check(rc, "vptq_b200_quant_gemm_wgrad")


def dequant_backward(desc: LinearDesc, dw: torch.Tensor, grads: dict) -> None:
    """Gradients of the layer's tensors from the gradient dw [out_features, in_features] of dequant()'s output
    (vptq_b200_dequant_backward)."""
    dw = _dense_rows(dw)
    g = make_grads(grads)
    dev = dw.device
    with _on_device(dev):
        ws = workspace(dev, _ws_bytes_cached(desc, 1, ("grad", GRAD_OP_DEQUANT_BACKWARD)))
        rc = lib().vptq_b200_dequant_backward(ctypes.byref(desc), dw.data_ptr(), row_pitch(dw), ctypes.byref(g),
                                              ws.data_ptr(), ws.numel(), 0, _stream(dev))
    check(rc, "vptq_b200_dequant_backward")


def dequant(desc: LinearDesc, w_out: torch.Tensor) -> None:
    dev = w_out.device
    with torch.cuda.device(dev):
        ws = workspace(dev, workspace_bytes(desc, 1, OP_DEQUANT))
        rc = lib().vptq_b200_dequant(ctypes.byref(desc), w_out.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev))
    check(rc, "vptq_b200_dequant")
