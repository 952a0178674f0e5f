"""`vptq.ops` operator surface on the H100 CUDA path.

Function names, argument order and argument meaning are the reference's
(vptq/ops/quant_gemm.py: `dequant` :43-69, `quant_gemm` :161-187, `quant_gemv_v2` :278-292), so
`VQuantLinear.forward` and the reference's tests can call them unchanged.  What differs:

* every op runs hand-written sm_90a CUDA through the C ABI (vptq_b200.native); there is no
  torch implementation to fall back to -- CPU tensors raise;
* routing: fewer than 3 tokens -> fused GEMV (the reference's rule, :213); otherwise the fused
  dequant->wgmma GEMM instead of `dequant` + `F.linear` (:231-275);
* `argsort(perm)` is not recomputed on every call (the reference does, :208-211).
"""
from __future__ import annotations

from typing import Optional

import torch

from . import native

__all__ = ["dequant", "quant_gemm", "quant_gemv_v2"]


def _desc(*, dtype, indices, centroids, outlier_indices, outlier_centroids, residual_centroids, perm,
          weight_scale, weight_bias, bias, vector_len, outlier_vector_len, num_codebooks, num_centroids,
          num_outlier_centroids, num_res_centroids, group_size, outlier_size, in_features, out_features,
          derive=True, lists=None, drop_packed=False):
    if perm is not None and perm.dtype not in (torch.int16, torch.uint16):
        # unpacked checkpoints keep perm as int64 (vqlinear.py:191-196)
        perm = perm.to(torch.int64).to(torch.uint16).contiguous()
    return native.make_desc(
        dtype=dtype, in_features=in_features, out_features=out_features, vector_len=vector_len,
        num_centroids=num_centroids, num_res_centroids=num_res_centroids if residual_centroids is not None else -1,
        num_codebooks=num_codebooks, group_size=group_size, outlier_size=outlier_size,
        outlier_vector_len=outlier_vector_len, num_outlier_centroids=num_outlier_centroids, indices=indices,
        centroids=centroids, res_centroids=residual_centroids, outlier_indices=outlier_indices,
        outlier_centroids=outlier_centroids, perm=perm, weight_scale=weight_scale, weight_bias=weight_bias,
        bias=bias, derive=derive, lists=lists, drop_packed=drop_packed), perm


def dequant(
    indices: torch.Tensor,
    centroids: torch.Tensor,
    outlier_indices: Optional[torch.Tensor],
    outlier_centroids: Optional[torch.Tensor],
    res_indices: Optional[torch.Tensor],
    res_centroids: Optional[torch.Tensor],
    perm: Optional[torch.Tensor],
    weight_scale: Optional[torch.Tensor],
    weight_bias: Optional[torch.Tensor],
    is_indice_packed: bool,
    enable_outlier: bool,
    enable_residual: bool,
    enable_perm: bool,
    enable_norm: bool,
    num_centroids: int,
    num_outlier_centroids: int,
    num_res_centroids: int,
    padding: int,
    outlier_padding: int,
    num_codebooks: int,
    group_size: int,
    outlier_size: int,
    vector_len: int,
    outlier_vector_len: int,
    vector_quant_dim: str = "out",
) -> torch.Tensor:
    """Dense weight [out_features, in_features] (reference: vptq/ops/quant_gemm.py:43-158)."""
    if vector_quant_dim == "in":
        raise ValueError("Not implemented yet.")
    if not is_indice_packed:
        raise RuntimeError("vptq_b200.ops.dequant needs packed int32 indices (vptq_b200.pack.pack_index)")
    if res_indices is not None:
        raise RuntimeError("packed layers carry the residual index inside `indices`; res_indices must be None")
    num_indices = indices.shape[1]
    out_features = num_indices * vector_len - padding
    in_features = num_codebooks * group_size + (outlier_size if enable_outlier else 0)
    desc, perm_ = _desc(
        dtype=centroids.dtype, indices=indices, centroids=centroids,
        outlier_indices=outlier_indices if enable_outlier else None,
        outlier_centroids=outlier_centroids if enable_outlier else None,
        residual_centroids=res_centroids if enable_residual else None, perm=perm if enable_perm else None,
        weight_scale=weight_scale if enable_norm else None, weight_bias=weight_bias if enable_norm else None,
        bias=None, vector_len=vector_len, outlier_vector_len=outlier_vector_len, num_codebooks=num_codebooks,
        num_centroids=num_centroids, num_outlier_centroids=num_outlier_centroids,
        num_res_centroids=num_res_centroids, group_size=group_size, outlier_size=outlier_size,
        in_features=in_features, out_features=out_features, derive=False, lists=False)
    w = torch.empty(out_features, in_features, dtype=centroids.dtype, device=centroids.device)
    native.dequant(desc, w)
    return w


def quant_gemm(
    x: torch.Tensor,
    bias: Optional[torch.Tensor],
    indices: torch.Tensor,
    centroids: torch.Tensor,
    outlier_indices: Optional[torch.Tensor],
    outlier_centroids: Optional[torch.Tensor],
    residual_indices: Optional[torch.Tensor],
    residual_centroids: Optional[torch.Tensor],
    perm: Optional[torch.Tensor],
    weight_scale: Optional[torch.Tensor],
    weight_bias: Optional[torch.Tensor],
    vector_len: int,
    outlier_vector_len: int,
    num_codebooks: int,
    num_centroids: int,
    num_outlier_centroids: int,
    num_res_centroids: int,
    is_indice_packed: bool,
    group_size: int,
    outlier_size: int,
    in_features: int,
    out_features: int,
    padding: int,
    outlier_padding: int,
    vector_quant_dim: str = "out",
    _desc_cache: Optional[list] = None,
    _drop_packed: bool = False,
) -> torch.Tensor:
    """y = x @ W^T + bias for one VPTQ layer (reference: vptq/ops/quant_gemm.py:161-275)."""
    if vector_quant_dim == "in":
        raise ValueError("Not implemented yet.")
    if not is_indice_packed:
        raise RuntimeError("vptq_b200.ops.quant_gemm needs packed int32 indices (vptq_b200.pack.pack_index)")
    if residual_indices is not None:
        raise RuntimeError("packed layers carry the residual index inside `indices`; residual_indices must be None")
    native.require_cuda("x", x, contiguous=False)
    if x.dtype != centroids.dtype:
        raise RuntimeError(f"x is {x.dtype} but the codebooks are {centroids.dtype}")
    if x.shape[-1] != in_features:
        raise RuntimeError(f"x has {x.shape[-1]} features, layer expects {in_features}")
    if _desc_cache is not None and _desc_cache:
        desc = _desc_cache[0]
    else:
        desc, perm_ = _desc(
            dtype=x.dtype, indices=indices, centroids=centroids, outlier_indices=outlier_indices,
            outlier_centroids=outlier_centroids, residual_centroids=residual_centroids, perm=perm,
            weight_scale=weight_scale, weight_bias=weight_bias, bias=bias, vector_len=vector_len,
            outlier_vector_len=outlier_vector_len, num_codebooks=num_codebooks, num_centroids=num_centroids,
            num_outlier_centroids=num_outlier_centroids, num_res_centroids=num_res_centroids,
            group_size=group_size, outlier_size=outlier_size, in_features=in_features, out_features=out_features,
            # a one-off descriptor (reference-style direct call) must not pay for re-bucketing the whole layer:
            # the slice x tile lists are built only when the caller keeps the descriptor (VQuantLinear does)
            lists=None if _desc_cache is not None else False, drop_packed=_drop_packed)
        if _desc_cache is not None:
            _desc_cache.extend([desc, perm_])   # keep the converted perm alive with the descriptor
    x2d = x.reshape(-1, in_features)
    if x2d.stride(-1) != 1:
        x2d = x2d.contiguous()
    tokens = x2d.shape[0]
    y = torch.empty(tokens, out_features, dtype=x.dtype, device=x.device)
    if tokens == 0:
        return y.reshape(*x.shape[:-1], out_features)
    if tokens < 3:
        native.quant_gemv(desc, x2d, y)
    else:
        native.quant_gemm(desc, x2d, y)
    return y.reshape(*x.shape[:-1], out_features)


def quant_gemv_v2(
    x: torch.Tensor,
    bias: Optional[torch.Tensor],
    indices: torch.Tensor,
    centroids: torch.Tensor,
    residual_indices: Optional[torch.Tensor],
    residual_centroids: Optional[torch.Tensor],
    scale_weights: Optional[torch.Tensor],
    scale_bias: Optional[torch.Tensor],
    vector_len: int,
    num_codebooks: int,
    num_centroids: int,
    num_residual_centroids: int,
    out_features: int,
) -> torch.Tensor:
    """GEMV with unpacked indices (reference: vptq/ops/quant_gemm.py:278-356; csrc/quant_gemv_v2.cu:25)."""
    for n, t in (("x", x), ("indices", indices), ("centroids", centroids), ("residual_indices", residual_indices),
                 ("residual_centroids", residual_centroids), ("scale_weights", scale_weights),
                 ("scale_bias", scale_bias), ("bias", bias)):
        native.require_cuda(n, t)
    if x.dim() != 3:
        raise RuntimeError("x must be (batch_size, sequence_length, in_features)")
    if num_codebooks != 1:
        raise RuntimeError("Only support one codebook.")
    tokens = x.shape[0] * x.shape[1]
    if tokens >= 16:   # same guard as the reference (quant_gemm.py:338-344, quant_gemv_v2.cu:58)
        raise RuntimeError("The input tensor is too large for GEMV to achieve good performance. "
                           "Please use quant_gemm instead.")
    if indices.dtype not in (torch.uint16, torch.int16):
        raise RuntimeError("indices must be uint16")
    in_features = x.shape[-1]
    res_bytes = 0
    if residual_centroids is not None:
        if residual_indices is None:
            raise RuntimeError("residual_centroids given without residual_indices")
        res_bytes = residual_indices.element_size()
    import ctypes
    y = torch.empty(x.shape[0], x.shape[1], out_features, dtype=x.dtype, device=x.device)
    p = lambda t: None if t is None else t.data_ptr()
    with torch.cuda.device(x.device):
        rc = native.lib().vptq_b200_quant_gemv_v2(
            native.dtype_code(x.dtype), x.data_ptr(), y.data_ptr(), tokens, in_features, out_features, vector_len,
            num_centroids, num_residual_centroids if residual_centroids is not None else 0, indices.data_ptr(),
            centroids.data_ptr(), p(residual_indices), res_bytes, p(residual_centroids), p(scale_weights),
            p(scale_bias), p(bias), None, 0, 0, torch.cuda.current_stream(x.device).cuda_stream)
    native.check(rc, "vptq_b200_quant_gemv_v2")
    return y
