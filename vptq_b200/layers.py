"""`VQuantLinear`: the VPTQ quantized linear module on the H100 CUDA path.

Drop-in for the reference module (vptq/layers/vqlinear.py:17-240): same constructor signature
(:56-75), same parameter / sub-module names, shapes and storage dtypes -- i.e. the same
state_dict, so Hugging Face `transformers.integrations.vptq.replace_with_vptq_linear` and the
public VPTQ-community checkpoints load unchanged:

    centroids.weight          [G, K*v]                       fp16/bf16   (nn.Embedding)
    res_centroids.weight      [G, Kr*v]                      fp16/bf16   (nn.Embedding, if Kr > 0)
    outlier_centroids.weight  [1, Kol*vol]                   fp16/bf16   (nn.Embedding, if outliers)
    indices                   [G, ceil(O/v), ceil(gs*b/32)]  int32 packed | [G, ceil(O/v), gs] int16
    res_indices               [G, ceil(O/v), gs]             int16       (unpacked + residual only)
    outlier_indices           [1, ceil(O/vol), S]            int16 / fp16 view of uint16
    perm                      [I]                            int16 view of uint16 (packed) | int64
    weight_scale, weight_bias [I],   bias [O]

`forward` hands these tensors to `vptq_b200.ops.quant_gemm`, which runs the sm_90a kernels.
The constructor is meta-device safe (HF builds the module under `torch.device("meta")`).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn
from torch.nn.parameter import Parameter

from . import ops
from .pack import pack_index

__all__ = ["VQuantLinear"]


def _frozen(shape, dtype, device) -> Parameter:
    return Parameter(torch.empty(shape, dtype=dtype, device=device), requires_grad=False)


def _version(t: torch.Tensor) -> int:
    """t._version, or 0 for an inference tensor: it has no version counter (reading it raises), and writes to it are
    only possible inside torch.inference_mode(), where the caches cannot see them (prepare(rebuild=True))."""
    return 0 if t.is_inference() else t._version


class VQuantLinear(nn.Module):
    """VPTQ quantized linear layer (see the module docstring for the tensors it holds).

    Autograd: when grad mode is on and `x.requires_grad`, `forward` records a backward that gives `x` its gradient
    (dX = dY W: a transposed dequant feeding the wgmma GEMM) and `bias` its gradient -- what adapters (LoRA / PEFT)
    trained on top of a frozen quantized model need.

    Fine-tuning the quantized layer itself is opt-in: after `set_quant_grad(True)` the codebooks (`centroids`,
    `res_centroids`, `outlier_centroids`), `weight_scale` and `weight_bias` get gradients too, through `forward`
    (also when x does not require grad) and through `dequant()` / `proxy_error_forward`.  Their `requires_grad`
    (see `set_centroids_grad`) decides which ones are computed; they come out in the parameter's dtype, summed in
    64-bit fixed point and rounded once, bit-identical from run to run (include/vptq_b200_grad.h).  Without the
    opt-in they get no gradient, as with the reference's CUDA extension.  Indices and perm never get one.  There is
    no double backward, and the backward of a decode-only module (`prepare(drop_packed=True)`) raises."""

    def __init__(
        self,
        in_features: int,
        out_features: int,
        vector_lens: Tuple[int, int],
        num_centroids: Tuple[int, int],
        num_res_centroids: Tuple[int, int],
        group_num: int,
        group_size: int,
        outlier_size: int,
        indices_as_float: bool,
        enable_norm: bool = False,
        enable_perm: bool = False,
        is_indice_packed: bool = False,
        bias: bool = False,
        vector_quant_dim: str = "out",
        device=None,
        dtype=None,
        enable_proxy_error=True,
    ):
        super().__init__()
        if vector_quant_dim not in ("in", "out"):
            raise ValueError("vector_quant_dim must be 'in' or 'out'.")
        if vector_quant_dim == "in":
            raise RuntimeError("Not implemented yet.")
        fk = {"device": device, "dtype": dtype}

        # ---- plain attributes (names are part of the surface: HF and user code read them) ----
        self.vector_quant_dim = vector_quant_dim
        self.in_features, self.out_features = in_features, out_features
        self.enable_proxy_error = enable_proxy_error
        self.outlier_vector_len, self.vector_len = vector_lens[0], vector_lens[1]
        self.num_outlier_centroids, self.num_centroids = num_centroids[0], num_centroids[1]
        self.outlier_num_res_centroids, self.num_res_centroids = num_res_centroids[0], num_res_centroids[1]
        self.group_num = self.num_codebooks = group_num
        self.group_size = group_size
        self.outlier_size = outlier_size
        self.indices_as_float = indices_as_float
        self.is_indice_packed = is_indice_packed
        self.enable_norm, self.enable_perm = enable_norm, enable_perm
        if self.num_res_centroids == 1:
            # 0 index bits: the packed format has no field that could tell one residual entry from none
            raise ValueError("num_res_centroids = 1 is not supported: use -1 (no residual) or a power of two >= 2")
        self.enable_residual = self.num_res_centroids > 0
        self.enable_outlier = bool(self.outlier_vector_len > 1 and self.num_outlier_centroids > 0)
        self.padding = (-out_features) % self.vector_len
        self.num_indices = (out_features + self.padding) // self.vector_len
        self.outlier_padding = 0
        self.ouliter_num_indices = 0          # (sic) attribute name kept from the reference

        # uint16 payloads are stored behind an int16 / float16 view (safetensors and NCCL have no uint16)
        u16_view = torch.float16 if indices_as_float else torch.int16

        if bias:
            self.bias = Parameter(torch.empty(out_features, **fk))
        else:
            self.register_parameter("bias", None)

        # ---- main codebook ----
        self.centroids = nn.Embedding(self.num_codebooks, self.num_centroids * self.vector_len, **fk)

        # ---- outlier columns: their own codebook, vector length vector_lens[0] ----
        self.outlier_centroids = None
        self.outlier_indices = None
        if self.enable_outlier:
            if self.outlier_num_res_centroids != -1:
                raise ValueError("Current implementation does not support residual quantization on outliers yet.")
            self.outlier_padding = (-out_features) % self.outlier_vector_len
            self.ouliter_num_indices = (out_features + self.outlier_padding) // self.outlier_vector_len
            self.outlier_centroids = nn.Embedding(1, self.num_outlier_centroids * self.outlier_vector_len, **fk)
            self.outlier_indices = _frozen((1, self.ouliter_num_indices, outlier_size), u16_view, device)

        # ---- residual codebook ----
        if self.enable_residual:
            self.res_indices = None
            self.res_centroids = nn.Embedding(self.num_codebooks, self.num_res_centroids * self.vector_len, **fk)
            if not is_indice_packed:
                self.res_indices = _frozen((self.num_codebooks, self.num_indices, group_size), u16_view, device)
        else:
            self.register_parameter("res_centroids", None)
            self.register_parameter("res_indices", None)

        # ---- column permutation and per-column affine ----
        if enable_perm:
            pdt = torch.int16 if is_indice_packed else torch.int64
            self.perm = Parameter(torch.arange(in_features, device=device, dtype=pdt), requires_grad=False)
        self.weight_scale = self.weight_bias = None
        if enable_norm:
            self.weight_scale = Parameter(torch.empty(in_features, **fk), requires_grad=True)
            self.weight_bias = Parameter(torch.empty(in_features, **fk), requires_grad=True)

        # ---- indices ----
        if is_indice_packed:
            self.index_bits = int(math.log2(self.num_centroids))
            self.res_index_bits = int(math.log2(self.num_res_centroids)) if self.enable_residual else 0
            self.total_index_bits = self.index_bits + self.res_index_bits
            words = math.ceil(group_size * self.total_index_bits / 32)
            self.indices = _frozen((self.num_codebooks, self.num_indices, words), torch.int32, device)
        else:
            self.indices = _frozen((self.num_codebooks, self.num_indices, group_size), torch.int16, device)

        self._desc_cache: list = []      # [LinearDesc, perm16] built on first forward
        self._desc_key = None
        self._packed = None              # lazily packed indices for unpacked checkpoints
        self._quant_grad = False         # set_quant_grad

    # ------------------------------------------------------------------------------------------
    def _tensors(self):
        resc = self.res_centroids.weight if self.res_centroids is not None else None
        outc = self.outlier_centroids.weight if self.enable_outlier else None
        return (self.indices, self.centroids.weight, resc, self.outlier_indices, outc, getattr(self, "perm", None),
                self.weight_scale, self.weight_bias, self.bias)

    def _packed_indices(self) -> torch.Tensor:
        if self.is_indice_packed:
            return self.indices
        key = tuple((a.data_ptr(), _version(a)) if a is not None else None for a in (self.indices, self.res_indices))
        if self._packed is None or self._packed[0] != key:
            ib = int(math.log2(self.num_centroids))
            rb = int(math.log2(self.num_res_centroids)) if self.enable_residual else 0
            packed = pack_index(self.indices, ib, self.res_indices if self.enable_residual else None, rb)
            self._packed = (key, packed.contiguous())
        return self._packed[1]

    def _cache_key(self, t, dtype, device):
        # data_ptr catches .to() / re-assignment, _version catches in-place updates (load_state_dict, copy_);
        # res_indices (unpacked checkpoints) is packed into the words the descriptor points to
        return tuple((a.data_ptr(), a.dtype, _version(a)) if a is not None else None
                     for a in t + (self.res_indices,)) + (dtype, device)

    # positions in _tensors() of the floating-point tensors the descriptor only points to (codebooks, scale, bias):
    # an in-place update of them (an optimizer step) keeps the descriptor and its index lists
    _FLOAT_SLOTS = (1, 2, 4, 6, 7, 8)

    def _refresh_in_place(self, key) -> bool:
        """Only floating-point tensors changed, in place (same storage): re-derive the quantised-order copies of
        weight_scale / weight_bias into their buffers and keep the descriptor.  False: rebuild everything."""
        old = self._desc_key
        if not self._desc_cache or old is None or len(old) != len(key) or old[-2:] != key[-2:]:
            return False
        for i, (a, b) in enumerate(zip(old[:-2], key[:-2])):
            if a is None or b is None:
                if a is not b:
                    return False
            elif a[:2] != b[:2] or (i not in self._FLOAT_SLOTS and a[2] != b[2]):
                return False
        desc = self._desc_cache[0]
        if desc._keep[:2] and desc.weight_scale_q:
            ws_q, wb_q = desc._keep[0], desc._keep[1]
            perm = self._desc_cache[1]
            pidx = perm.view(torch.uint16).to(torch.int64) if perm.dtype in (torch.int16, torch.uint16) else perm.long()
            with torch.no_grad():
                torch.index_select(self.weight_scale, 0, pidx, out=ws_q)
                torch.index_select(self.weight_bias, 0, pidx, out=wb_q)
        return True

    def set_quant_grad(self, enabled: bool = True) -> "VQuantLinear":
        """Opt in to gradients for the codebooks, weight_scale and weight_bias (see the class docstring).  The
        tensors' `requires_grad` decides which are computed.  A decode-only module refuses: its packed index words,
        which every weight gradient reads, were freed."""
        if enabled:
            self._check_quant_grad_possible()
        self._quant_grad = bool(enabled)
        return self

    def _check_quant_grad_possible(self) -> None:
        if getattr(self, "_drop_packed", False) and self.indices.numel() == 0:
            raise RuntimeError("set_quant_grad: this VQuantLinear is decode-only (prepare(drop_packed=True)); the "
                               "packed index words the weight gradients need were freed; reload the checkpoint")

    def _quant_grad_needed(self) -> bool:
        """Opted in and some quantizer tensor requires grad: a forward under grad mode records a node."""
        if not getattr(self, "_quant_grad", False):
            return False
        _, cent, resc, _, outc, _, ws, wb, _ = self._tensors()
        return any(t is not None and t.requires_grad for t in (cent, resc, outc, ws, wb))

    def prepare(self, dtype: Optional[torch.dtype] = None, drop_packed: bool = False,
                rebuild: bool = False) -> "VQuantLinear":
        """Build the C-ABI descriptor and its load-time derivatives (scale/bias in quantised order, the
        slice x tile index lists of the decode kernel) now instead of inside the first forward: call once
        after loading the checkpoint, before capturing CUDA graphs.

        The descriptor is kept as long as the parameters' storage and version counters say nothing changed.  After an
        in-place update of the parameters (an optimizer step, `mul_`, `copy_`), call `prepare()` again before
        replaying a captured CUDA graph: it refreshes the quantised-order copies of weight_scale / weight_bias, which
        only `forward` does otherwise.  Writes the version counters cannot see -- through `.data`, or to inference
        tensors inside torch.inference_mode() -- need `rebuild=True`: it drops the descriptor, the index lists and
        the packed words of an unpacked checkpoint and builds them again from the tensors.  Graphs captured before
        a rebuild point to the dropped buffers: capture them again.

        drop_packed=True makes the module DECODE-ONLY: once the index lists exist the packed `indices` are freed
        (4.2 instead of 7.2 bytes per index resident).  Calls with more than one token, `dequant()` and saving the
        state_dict are no longer possible; reloading a checkpoint restores them."""
        if rebuild:
            if getattr(self, "_drop_packed", False) and self.indices.numel() == 0:
                raise RuntimeError("prepare(rebuild=True): this VQuantLinear is decode-only (prepare(drop_packed="
                                   "True)); its index lists cannot be rebuilt without the packed index words, which "
                                   "were freed; reload the checkpoint")
            self._desc_cache, self._desc_key, self._packed = [], None, None
        dtype = dtype or self.centroids.weight.dtype
        x = torch.zeros(1, self.in_features, dtype=dtype, device=self.centroids.weight.device)
        if drop_packed:
            if not self.is_indice_packed:
                raise RuntimeError("drop_packed needs a packed checkpoint (is_indice_packed=True)")
            if getattr(self, "_quant_grad", False):
                raise RuntimeError("prepare(drop_packed=True) on a module with set_quant_grad(True): the weight "
                                   "gradients need the packed index words; call set_quant_grad(False) first")
            self._desc_cache, self._desc_key = [], None
            self._drop_request = True
        try:
            self.forward(x)
        finally:
            self._drop_request = False
        if drop_packed:
            with torch.no_grad():
                self.indices.data = torch.empty(0, dtype=self.indices.dtype, device=self.indices.device)
            self._packed, self._drop_packed = None, True
        return self

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # a decode-only module (prepare(drop_packed=True)) freed its packed words: make room for the checkpoint's
        src = state_dict.get(prefix + "indices")
        if src is not None and self.indices.numel() == 0 and src.numel() > 0:
            with torch.no_grad():
                self.indices.data = torch.empty(src.shape, dtype=self.indices.dtype, device=self.indices.device)
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def __getstate__(self):
        # the cached descriptor holds raw pointers (ctypes): never pickled or deep-copied
        st = self.__dict__.copy()
        st["_desc_cache"], st["_desc_key"], st["_packed"] = [], None, None
        return st

    def __deepcopy__(self, memo):
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__getstate__().items():
            new.__dict__[k] = copy.deepcopy(v, memo)
        return new

    def forward(self, x, W=None, H=None):
        """x: [..., in_features] fp16/bf16 on the GPU -> [..., out_features]."""
        if self.enable_proxy_error:
            return self.proxy_error_forward(W, H)   # quantizer-side debugging aid
        t = self._tensors()
        key = self._cache_key(t, x.dtype, x.device)
        if getattr(self, "_drop_packed", False):
            if self.indices.numel() == 0 and self._desc_cache:
                key = self._desc_key                  # decode-only: the descriptor no longer depends on `indices`
            else:
                self._drop_packed = False             # a checkpoint was loaded again: a full module once more
        if key != self._desc_key:                    # parameters were moved / reloaded / updated in place
            if not self._refresh_in_place(key):
                self._desc_cache = []
            self._desc_key = key
        indices, cent, resc, outi, outc, perm, ws, wb, bias = t
        return ops.quant_gemm(
            x, bias=bias, indices=self._packed_indices(), centroids=cent, outlier_indices=outi,
            outlier_centroids=outc, residual_indices=None, residual_centroids=resc, perm=perm,
            weight_scale=ws, weight_bias=wb, vector_len=self.vector_len,
            outlier_vector_len=self.outlier_vector_len, num_codebooks=self.num_codebooks,
            num_centroids=self.num_centroids, num_outlier_centroids=self.num_outlier_centroids,
            num_res_centroids=self.num_res_centroids, is_indice_packed=True, group_size=self.group_size,
            outlier_size=self.outlier_size, in_features=self.in_features, out_features=self.out_features,
            padding=self.padding, outlier_padding=self.outlier_padding,
            vector_quant_dim=self.vector_quant_dim, _desc_cache=self._desc_cache,
            _drop_packed=getattr(self, "_drop_request", False), _quant_grad=getattr(self, "_quant_grad", False))

    def dequant(self) -> torch.Tensor:
        """Dense [out_features, in_features] weight through the CUDA dequant kernel."""
        if getattr(self, "_drop_packed", False) and self.indices.numel() == 0:
            raise RuntimeError("this VQuantLinear is decode-only (prepare(drop_packed=True)): the packed index words "
                               "dequant needs were freed; reload the checkpoint to get them back")
        indices, cent, resc, outi, outc, perm, ws, wb, _ = self._tensors()
        return ops.dequant(
            indices=self._packed_indices(), centroids=cent, outlier_indices=outi, outlier_centroids=outc,
            res_indices=None, res_centroids=resc, perm=perm, weight_scale=ws, weight_bias=wb,
            is_indice_packed=True, enable_outlier=self.enable_outlier, enable_residual=self.enable_residual,
            enable_perm=self.enable_perm, enable_norm=self.enable_norm, num_centroids=self.num_centroids,
            num_outlier_centroids=self.num_outlier_centroids, num_res_centroids=self.num_res_centroids,
            padding=self.padding, outlier_padding=self.outlier_padding, num_codebooks=self.num_codebooks,
            group_size=self.group_size, outlier_size=self.outlier_size, vector_len=self.vector_len,
            outlier_vector_len=self.outlier_vector_len, vector_quant_dim=self.vector_quant_dim,
            _quant_grad=getattr(self, "_quant_grad", False))

    def proxy_error_forward(self, W, H):
        """diff^T diff * H with diff = dequant() - W (the quantizer's layer-wise proxy loss)."""
        diff = self.dequant().to(W.dtype) - W
        return diff.T @ diff * H

    def set_centroids_grad(self, requires_grad: bool) -> None:
        """Sets `requires_grad` on the codebooks (reference surface).  They receive gradients once the module has
        opted in with `set_quant_grad(True)`; without it the CUDA path computes no codebook gradient."""
        self.centroids.weight.requires_grad = requires_grad
        if self.enable_outlier:
            self.outlier_centroids.weight.requires_grad = requires_grad
        if self.enable_residual:
            self.res_centroids.weight.requires_grad = requires_grad

    def init_parameters(self, centroids, indices, res_centroids=None, res_indices=None, weight_scale=None,
                        weight_bias=None, perm=None):
        """Load quantizer output (dicts keyed by codebook id; key 0 is the outlier block).

        Same contract as the reference (vptq/layers/vqlinear.py:242-342).  Indices are given
        unpacked; packed modules pack them here.
        """
        dev = self.centroids.weight.device
        u16_view = torch.float16 if self.indices_as_float else torch.int16

        def stack(d):
            return torch.stack([d[k] for k in sorted(d.keys())[1:]], dim=0)

        self.centroids.weight.data = stack(centroids).reshape(
            self.num_codebooks, self.num_centroids * self.vector_len).to(dev)
        main_idx = stack(indices).reshape(self.num_codebooks, self.num_indices, self.group_size).to(torch.int64)
        res_idx = None
        if self.enable_residual:
            self.res_centroids.weight.data = stack(res_centroids).reshape(
                self.num_codebooks, self.num_res_centroids * self.vector_len).to(dev)
            res_idx = stack(res_indices).reshape(self.num_codebooks, self.num_indices, self.group_size).to(torch.int64)
        if self.is_indice_packed:
            self.indices.data = pack_index(main_idx.to(dev), self.index_bits,
                                           res_idx.to(dev) if res_idx is not None else None, self.res_index_bits)
        else:
            self.indices.data = main_idx.to(torch.uint16).view(u16_view).to(dev)
            if res_idx is not None:
                self.res_indices.data = res_idx.to(torch.uint16).view(u16_view).to(dev)
        if self.enable_outlier:
            self.outlier_centroids.weight.data = centroids[0].clone().detach().reshape(
                1, self.num_outlier_centroids * self.outlier_vector_len).to(dev)
            oi = indices[0].clone().detach().to(torch.uint16).view(u16_view).to(dev)
            self.outlier_indices.data = oi.unsqueeze(0) if oi.dim() == 2 else oi
        if self.enable_norm:
            self.weight_scale.data = weight_scale.to(dev)
            self.weight_bias.data = weight_bias.to(dev)
        if self.enable_perm:
            p = perm.to(dev)
            self.perm.data = p.to(torch.uint16).view(torch.int16) if self.is_indice_packed else p.to(torch.int64)
        self._desc_cache, self._desc_key, self._packed = [], None, None

    def extra_repr(self) -> str:
        b = int(math.log2(self.num_centroids)) + (int(math.log2(self.num_res_centroids)) if self.enable_residual else 0)
        return (f"in_features={self.in_features}, out_features={self.out_features}, v={self.vector_len}, "
                f"K={self.num_centroids}, Kr={self.num_res_centroids}, index_bits/vector={b}, "
                f"groups={self.num_codebooks}, outliers={self.outlier_size if self.enable_outlier else 0}")
