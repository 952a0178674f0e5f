"""`vptq.ops` operator surface on the H100 CUDA path.

Function names, argument order and argument meaning are the reference's
(vptq/ops/quant_gemm.py: `dequant` :43-69, `quant_gemm` :161-187, `quant_gemv_v2` :278-292), so
`VQuantLinear.forward` and the reference's tests can call them unchanged.  What differs:

* every op runs hand-written sm_90a CUDA through the C ABI (vptq_b200.native); there is no
  torch implementation to fall back to -- CPU tensors raise;
* routing: `route` alone decides which kernel takes a call -- of one layer, of a fused group of layers
  (vptq_b200.fuse) or of an input gradient -- from the token count, the alignment of x, the descriptor and the layer's
  opt-ins (`OptIns`: VQuantLinear.set_batched_decode / set_lists_prefill / set_list_decode).  Without opt-ins it is
  the reference's rule (fewer than 3 tokens -> fused GEMV, :213), with the fused dequant->wgmma GEMM instead of
  `dequant` + `F.linear` (:231-275) for larger calls;
* `argsort(perm)` is not recomputed on every call (the reference does, :208-211).
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch
from torch.autograd.function import once_differentiable

from . import native

__all__ = ["dequant", "quant_gemm", "quant_gemv_v2"]


class OptIns(NamedTuple):
    """A VQuantLinear's routing opt-ins: set_batched_decode, set_lists_prefill and set_list_decode."""
    batched_decode: bool = False
    lists_prefill: bool = False
    list_decode: bool = False


NO_OPT_INS = OptIns()

# the routes `route` returns
EMPTY, LISTS16, BATCH, LISTS_GEMM, GEMV, GEMM, DGRAD = (
    "empty", "lists16", "batch", "lists_gemm", "gemv", "gemm", "dgrad")


def route(descs, tokens: int, aligned: bool, opt_ins, vector_len: int = 0, dgrad: bool = False) -> Optional[str]:
    """The kernel that takes a call of `tokens` rows of x; `aligned`: x starts on a 16-byte boundary.

    One call: `descs` is the layer's descriptor and `opt_ins` its OptIns.  The first rule that holds wins:
      1. no tokens: EMPTY, no launch;
      2. list_decode, v = 16, index lists, x aligned or a decode-only descriptor (no packed words; the caller runs it
         on an aligned copy of x), tokens <= lists16_max_tokens: LISTS16, the v = 16 list kernel;
      3. batched_decode, 2+ tokens, index lists, x aligned, tokens <= batch_max_tokens: BATCH, the batched list kernel;
      4. lists_prefill, 2+ tokens, a decode-only descriptor: LISTS_GEMM, the GEMM with the weight from the lists;
      5. fewer than 3 tokens: GEMV;
      6. GEMM.
    A max-token query runs only when every other condition of its rule holds (its answer is cached per descriptor).

    `dgrad`: the route of the input gradient instead: DGRAD (the transposed GEMM) while the descriptor has its packed
    words, LISTS_GEMM (transposed) for a decode-only one with lists_prefill, None for a decode-only one without.

    A fused group (vptq_b200.fuse): `descs` is a function returning the members' descriptors, called only once a rule
    needs them (it rebuilds stale ones), `opt_ins` one OptIns per member and `vector_len` the members'.  The rules
    above apply to the group as one layer: batched_decode and list_decode when every member opted in, "lists_prefill
    and decode-only" when some member is both, max-token queries for all the descriptors together, and x is never
    copied.  The group gets GEMV or BATCH (v = 8) or LISTS16 (v = 16) -- the routes that launch the group as one --
    and None for every other route: each member then runs its own call."""
    group = not isinstance(opt_ins, OptIns)
    if group:
        batched = all(o.batched_decode for o in opt_ins)
        list_decode = all(o.list_decode for o in opt_ins)
        lists_prefill = any(o.lists_prefill for o in opt_ins)
        d = None
    else:
        batched, lists_prefill, list_decode = opt_ins
        d, vector_len = descs, descs.vector_len
        if dgrad:
            return DGRAD if d.indices else LISTS_GEMM if lists_prefill else None
    if tokens == 0:
        return None if group else EMPTY
    if list_decode and vector_len == 16:
        d = d or descs()
        # a group's query answers 0 when some member has no lists
        if (group or d.lists_stream) and (aligned or not (group or d.indices)) and \
                tokens <= native.lists16_max_tokens(d):
            return LISTS16
    if group and vector_len == 16:
        return None           # a v = 16 group launches nothing else as one
    if batched and tokens >= 2 and aligned:
        d = d or descs()
        if (group or d.lists_stream) and tokens <= native.batch_max_tokens(d):
            return BATCH
    if group and tokens >= 3:
        return None           # past the batched kernel a v = 8 group has only the GEMV of 1..2 tokens
    if lists_prefill and tokens >= 2:
        d = d or descs()
        if any(o.lists_prefill and not m.indices for o, m in zip(opt_ins, d)) if group else not d.indices:
            return None if group else LISTS_GEMM
    return GEMV if tokens < 3 else GEMM


def _desc(*, dtype, indices, centroids, outlier_indices, outlier_centroids, residual_centroids, perm,
          weight_scale, weight_bias, bias, vector_len, outlier_vector_len, num_codebooks, num_centroids,
          num_outlier_centroids, num_res_centroids, group_size, outlier_size, in_features, out_features,
          derive=True, lists=None, drop_packed=False, lists16=False, lists_prefill=False):
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
        bias=bias, derive=derive, lists=lists, drop_packed=drop_packed, lists16=lists16,
        lists_prefill=lists_prefill), perm


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
    _quant_grad: bool = False,
) -> torch.Tensor:
    """Dense weight [out_features, in_features] (reference: vptq/ops/quant_gemm.py:43-158).

    `_quant_grad` (VQuantLinear.set_quant_grad): under grad mode the result is differentiable with respect to the
    codebooks, weight_scale and weight_bias that require grad (vptq_b200_dequant_backward)."""
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
    if _quant_grad and torch.is_grad_enabled():
        slots = _quant_slots(centroids, res_centroids if enable_residual else None,
                             outlier_centroids if enable_outlier else None, weight_scale if enable_norm else None,
                             weight_bias if enable_norm else None)
        if any(t.requires_grad for _, t in slots):
            others = [t for t in (indices, outlier_indices if enable_outlier else None,
                                  perm if enable_perm else None) if t is not None]
            return _DequantFn.apply([desc, perm_], out_features, tuple(n for n, _ in slots),
                                    *[t for _, t in slots], *others)
    w = torch.empty(out_features, in_features, dtype=centroids.dtype, device=centroids.device)
    native.dequant(desc, w)
    return w


def _quant_slots(centroids, residual_centroids, outlier_centroids, weight_scale, weight_bias):
    """(gradient name of vptq_linear_grads, tensor) for the layer's floating-point tensors that are present."""
    pairs = (("centroids", centroids), ("res_centroids", residual_centroids), ("outlier_centroids", outlier_centroids),
             ("weight_scale", weight_scale), ("weight_bias", weight_bias))
    return [(n, t) for n, t in pairs if t is not None]


def _quant_grads(ctx, first: int, names, tensors) -> dict:
    """Output tensors for the quantizer gradients autograd asks for; input slot `first + i` holds tensors[i]."""
    return {n: torch.empty_like(t, memory_format=torch.contiguous_format)
            for i, (n, t) in enumerate(zip(names, tensors)) if ctx.needs_input_grad[first + i]}


class _DequantFn(torch.autograd.Function):
    """W = dequant(layer), differentiable with respect to the codebooks, weight_scale and weight_bias.

    backward: vptq_b200_dequant_backward reduces dL/dW into each requested tensor (64-bit fixed point: bit-identical
    from run to run).  The packed indices, outlier indices and perm are saved too, only for autograd's version
    check; they get no gradient."""

    @staticmethod
    def forward(ctx, keep, out_features, names, *layer):
        ctx.keep, ctx.names = keep, names
        ctx.save_for_backward(*layer)
        desc = keep[0]
        w = torch.empty(out_features, desc.in_features, dtype=layer[0].dtype, device=layer[0].device)
        native.dequant(desc, w)
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, dw):
        saved = ctx.saved_tensors
        quant = saved[:len(ctx.names)]
        want = _quant_grads(ctx, 3, ctx.names, quant)
        if want:
            native.dequant_backward(ctx.keep[0], dw, want)
        return (None, None, None) + tuple(want.get(n) for n in ctx.names) + (None,) * (len(saved) - len(quant))


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
    _quant_grad: bool = False,
    _opt_ins: OptIns = NO_OPT_INS,
) -> torch.Tensor:
    """y = x @ W^T + bias for one VPTQ layer (reference: vptq/ops/quant_gemm.py:161-275).

    `_quant_grad` (VQuantLinear.set_quant_grad): under grad mode the codebooks, weight_scale and weight_bias that
    require grad get gradients too, also when x does not require grad (vptq_b200_quant_gemm_wgrad).

    `_opt_ins` (VQuantLinear.set_batched_decode / set_lists_prefill / set_list_decode): the routes `route` may
    choose besides the default ones.  With list_decode a kept descriptor of a vector-length-16 layer carries index lists;
    with lists_prefill as well, `_drop_packed` may make it decode-only."""
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
            lists=None if _desc_cache is not None else False, drop_packed=_drop_packed,
            lists16=_opt_ins.list_decode and _desc_cache is not None, lists_prefill=_opt_ins.lists_prefill)
        if _desc_cache is not None:
            _desc_cache.extend([desc, perm_])   # keep the converted perm alive with the descriptor
    x2d = x.reshape(-1, in_features)
    if x2d.stride(-1) != 1 or (x2d.shape[0] > 1 and x2d.stride(0) < in_features):
        x2d = x2d.contiguous()    # broadcast rows (expand, overlapping unfold windows): the kernels need pitch >= I
    if torch.is_grad_enabled():
        slots = _quant_slots(centroids, residual_centroids, outlier_centroids, weight_scale, weight_bias) \
            if _quant_grad else []
        quant = any(t.requires_grad for _, t in slots)
        if x.requires_grad or quant:
            # keeps the descriptor (and the uint16 perm it points to) alive until backward, also for a one-off
            # descriptor
            keep = _desc_cache[:2] if _desc_cache is not None else [desc, perm_]
            if not quant:
                layer = (indices, centroids, residual_centroids, outlier_indices, outlier_centroids, perm,
                         weight_scale, weight_bias)
                y = _QuantLinearFn.apply(x2d, bias, keep, out_features, _opt_ins, *[t for t in layer if t is not None])
            else:
                others = [t for t in (indices, outlier_indices, perm) if t is not None]
                y = _QuantLinearWgradFn.apply(x2d, bias, keep, out_features, _opt_ins, tuple(n for n, _ in slots),
                                              *[t for _, t in slots], *others)
            return y.reshape(*x.shape[:-1], out_features)
    return _forward(desc, x2d, out_features, _opt_ins).reshape(*x.shape[:-1], out_features)


def _forward(desc, x2d: torch.Tensor, out_features: int, opt_ins: OptIns = NO_OPT_INS) -> torch.Tensor:
    tokens = x2d.shape[0]
    y = torch.empty(tokens, out_features, dtype=x2d.dtype, device=x2d.device)
    aligned = x2d.data_ptr() % 16 == 0
    r = route(desc, tokens, aligned, opt_ins)
    if r is LISTS16:
        # a decode-only descriptor has no other route for these calls: a misaligned x runs on an aligned copy (each
        # token's outputs do not depend on where x lives)
        native.quant_gemv_lists16(desc, x2d if aligned else x2d.clone(memory_format=torch.contiguous_format), y)
    elif r is BATCH:
        native.quant_gemv_batch(desc, x2d, y)
    elif r is LISTS_GEMM:
        native.lists_quant_gemm(desc, x2d, y)
    elif r is GEMV:
        native.quant_gemv(desc, x2d, y)
    elif r is GEMM:
        native.quant_gemm(desc, x2d, y)
    return y


class _QuantLinearFn(torch.autograd.Function):
    """y = x W^T + bias with gradients for x and bias.

    forward: the no-grad routing above, so values are bit-identical to a call under torch.no_grad().
    backward: dX = dY W through the transposed dequant + wgmma GEMM (vptq_b200_quant_gemm with VPTQ_FLAG_TRANSPOSE)
    for any token count; dbias = dY summed over tokens in fp32.  The codebooks, weight_scale and weight_bias get no
    gradient (the reference's CUDA path does not give them one either).  The layer tensors are saved so that an
    in-place update between forward and backward fails autograd's version check instead of using new weights."""

    @staticmethod
    def forward(ctx, x2d, bias, keep, out_features, opt_ins, *layer):
        ctx.keep, ctx.opt_ins = keep, opt_ins
        ctx.save_for_backward(*layer)
        return _forward(keep[0], x2d, out_features, opt_ins)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        ctx.saved_tensors            # version check of the layer tensors
        dx, dbias = _input_grads(ctx, ctx.keep[0], dy)
        return (dx, dbias, None, None, None) + (None,) * len(ctx.saved_tensors)


def _input_grads(ctx, desc, dy):
    """(dX, dbias) of y = x W^T + bias for the slots 0 and 1 that need them."""
    r = route(desc, dy.shape[0], True, ctx.opt_ins, dgrad=True)
    if r is None:
        raise RuntimeError("backward through a decode-only VQuantLinear (prepare(drop_packed=True)): the input "
                           "gradient needs the packed index words, which were freed; reload the checkpoint")
    dx = dbias = None
    if ctx.needs_input_grad[0]:
        dx = torch.empty(dy.shape[0], desc.in_features, dtype=dy.dtype, device=dy.device)
        if dy.shape[0]:
            if r is LISTS_GEMM:   # Wt written from the index lists
                native.lists_quant_gemm(desc, dy, dx, native.FLAG_TRANSPOSE)
            else:
                native.quant_gemm_dgrad(desc, dy, dx)
    if ctx.needs_input_grad[1]:
        dbias = dy.float().sum(0).to(dy.dtype)
    return dx, dbias


class _QuantLinearWgradFn(torch.autograd.Function):
    """_QuantLinearFn plus the gradients of the codebooks, weight_scale and weight_bias (VQuantLinear.set_quant_grad).

    forward: the same no-grad routing (bit-identical values); x is saved for the weight gradient.
    backward: dX and dbias as _QuantLinearFn; the quantizer tensors autograd asks for through
    vptq_b200_quant_gemm_wgrad (G = dY^T x by the wgmma GEMM, reduced in 64-bit fixed point: bit-identical from run
    to run).  `layer` = the quantizer tensors named by `names`, then the index tensors and perm (saved only for
    autograd's version check)."""

    @staticmethod
    def forward(ctx, x2d, bias, keep, out_features, opt_ins, names, *layer):
        ctx.keep, ctx.names, ctx.opt_ins = keep, names, opt_ins
        ctx.save_for_backward(x2d, *layer)
        return _forward(keep[0], x2d, out_features, opt_ins)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        saved = ctx.saved_tensors
        x2d, quant = saved[0], saved[1:1 + len(ctx.names)]
        desc = ctx.keep[0]
        dx, dbias = _input_grads(ctx, desc, dy)
        want = _quant_grads(ctx, 6, ctx.names, quant)
        if want:
            if dy.shape[0]:
                native.quant_gemm_wgrad(desc, x2d, dy, want)
            else:
                for t in want.values():
                    t.zero_()
        return (dx, dbias, None, None, None, None) + tuple(want.get(n) for n in ctx.names) + \
            (None,) * (len(saved) - 1 - len(quant))


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
