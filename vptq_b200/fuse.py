"""Model-level adapter: horizontal fusion of sibling VQuantLinear layers, without touching the model code.

The reference launches every `VQuantLinear` on its own (vptq/layers/model_base.py:33-53 swaps the modules in,
Hugging Face then calls `self.q_proj(x)`, `self.k_proj(x)`, `self.v_proj(x)` one after the other).  The C ABI
can run layers that read the same x in ONE launch (`vptq_b200_quant_gemv_multi_ws`, SURVEY.md section 8 f-1);
this module makes that reachable from an unmodified model:

    import vptq_b200
    vptq_b200.fuse(model)            # after the checkpoint is loaded, before CUDA-graph capture

`fuse` walks the module tree; wherever a parent module owns a complete sibling group (`q_proj`/`k_proj`/
`v_proj`, `gate_proj`/`up_proj` -- configurable) of VQuantLinear layers with the same in_features and dtype,
it puts a `FusedMember` in place of each.  The FIRST member that is called with a new decode activation
(1..2 tokens) launches the whole group into one buffer and hands out its own slice; the following members see
the same tensor (same storage, same version) and only return theirs.  Anything else -- prefill token counts,
a member called alone, an activation that changed in between -- takes the member's own `forward`, so results
are those of the unfused model in every case.  `fuse` also builds every layer's descriptor and load-time
index lists (`VQuantLinear.prepare`), so nothing is allocated or re-bucketed inside the first forward.

After `set_batched_decode(model)` a group whose members all opted in also launches 2..8-token activations as one
batched list-kernel launch (include/vptq_b200_batch.h), with the same results as its members' own forwards.

After `set_list_decode(model)` a group of vector-length-16 layers that all opted in launches 1..4-token activations
as one launch of the v = 16 list kernel (include/vptq_b200_lists16.h).  Without it such a group is never fused: each
member takes its own forward.

`set_lists_prefill(model)` lets decode-only layers (`prepare(drop_packed=True)`) serve prompts from their index lists
(include/vptq_b200_lists_dense.h).  The generic fused launch cannot take 2-token calls of such a group, so those go to
each member's own forward.  A decode-only vector-length-16 group (set_list_decode too) only ever launches the v = 16
list kernel; every call it declines goes to each member's own forward, which never needs the packed words either.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import native
from .layers import VQuantLinear

__all__ = ["fuse", "unfuse", "set_quant_grad", "set_batched_decode", "set_lists_prefill", "set_list_decode", "FusedGroup",
           "FusedMember", "DEFAULT_GROUPS"]

DEFAULT_GROUPS: Tuple[Tuple[str, ...], ...] = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


def activation_key(x: torch.Tensor) -> tuple:
    """Identity of a decode activation for FusedGroup's output cache.  An inference tensor has no version counter:
    a write to x inside torch.inference_mode() between two members' calls goes unseen (a new activation at the same
    address does not: each member is served once)."""
    return (x.data_ptr(), 0 if x.is_inference() else x._version, tuple(x.shape), x.dtype, x.device)


class FusedGroup:
    """Shared state of one sibling group (not an nn.Module: the layers stay owned by their FusedMembers)."""

    def __init__(self, layers: Sequence[VQuantLinear], flags: int = 0):
        self.layers = list(layers)
        self.flags = flags
        self.widths = [l.out_features for l in self.layers]
        self._key = None          # identity of the activation the cached outputs belong to
        self._served = 0          # bit i: member i has already taken its slice of the cached outputs
        self._out: Optional[torch.Tensor] = None
        self._fused: Optional[native.FusedGemv] = None
        self._fused_key = None

    def _descs(self, x: torch.Tensor):
        for l in self.layers:     # (re)build stale descriptors through the layer's own cache logic
            t = l._tensors()
            key = l._cache_key(t, x.dtype, x.device)
            stale = key != l._desc_key
            if stale and l._decode_only() and l._desc_key is not None:
                # a decode-only layer's descriptor no longer follows `indices` (its forward keeps it the same way):
                # only another dtype or device makes it stale, and its forward then refuses the call
                stale = key[-2:] != l._desc_key[-2:]
            if stale or not l._desc_cache:
                l.prepare(x.dtype)
        return [l._desc_cache[0] for l in self.layers]

    def outputs(self, x: torch.Tensor, index: int) -> Optional[torch.Tensor]:
        """[tokens, sum(widths)] for a decode activation, None when this call must not be fused.

        The cached outputs are handed to every member at most once: an address + version match alone could be a
        NEW tensor the caching allocator placed where the previous activation lived."""
        if torch.is_grad_enabled() and (x.requires_grad or any(l._quant_grad_needed() for l in self.layers)):
            return None           # the member's own forward records the autograd graph (same values)
        x2 = x.reshape(-1, x.shape[-1])
        tokens = x2.shape[0]
        if not x.is_cuda or tokens < 1 or x2.stride(-1) != 1 or (tokens > 1 and x2.stride(0) < x2.shape[1]):
            return None
        if self.layers[0].vector_len == 16:
            return self._outputs16(x, x2, index)
        # 2..8 tokens: the batched list kernel when every member opted in (set_batched_decode) and it takes them
        batched = tokens >= 2 and all(getattr(l, "_batched_decode", False) for l in self.layers)
        if tokens > 2 and not batched:
            return None
        # decode-only members (set_lists_prefill) route 2-token calls the batched kernel does not take themselves
        lists_member = tokens == 2 and any(getattr(l, "_lists_prefill", False) and l._decode_only() for l in self.layers)
        if lists_member and not batched:
            return None
        key = activation_key(x)
        if key == self._key and self._out is not None and not (self._served >> index) & 1:
            self._served |= 1 << index
            if self._served == (1 << len(self.layers)) - 1:
                self._key = None
            return self._out
        descs = self._descs(x)
        if batched and (x2.data_ptr() % 16 or tokens > native.batch_max_tokens(descs)):
            if tokens > 2 or lists_member:
                return None       # each member routes its own call (its own batched launch where it is eligible)
            batched = False
        fkey = tuple(id(d) for d in descs) + (tokens, batched)
        if self._fused is None or fkey != self._fused_key:
            self._out = torch.empty(tokens, sum(self.widths), dtype=x.dtype, device=x.device)
            offs = [0]
            for w in self.widths:
                offs.append(offs[-1] + w)
            fused = native.FusedGemvBatch if batched else native.FusedGemv
            self._fused = fused(descs, [self._out[:, a:b] for a, b in zip(offs[:-1], offs[1:])])
            self._fused_key = fkey
        self._fused(x2, self.flags)
        self._key, self._served = key, 1 << index
        return self._out

    def _outputs16(self, x: torch.Tensor, x2: torch.Tensor, index: int) -> Optional[torch.Tensor]:
        """outputs() of a vector-length-16 group: one launch of the v = 16 list kernel when every member opted in
        (set_list_decode) and it takes the whole group at this token count, else None (each member's own forward)."""
        if not all(getattr(l, "_list_decode", False) for l in self.layers):
            return None
        tokens = x2.shape[0]
        key = activation_key(x)
        if key == self._key and self._out is not None and not (self._served >> index) & 1:
            self._served |= 1 << index
            if self._served == (1 << len(self.layers)) - 1:
                self._key = None
            return self._out
        descs = self._descs(x)
        if x2.data_ptr() % 16 or tokens > native.lists16_max_tokens(descs):
            return None
        fkey = tuple(id(d) for d in descs) + (tokens, "lists16")
        if self._fused is None or fkey != self._fused_key:
            self._out = torch.empty(tokens, sum(self.widths), dtype=x.dtype, device=x.device)
            offs = [0]
            for w in self.widths:
                offs.append(offs[-1] + w)
            self._fused = native.FusedGemvLists16(descs, [self._out[:, a:b] for a, b in zip(offs[:-1], offs[1:])])
            self._fused_key = fkey
        self._fused(x2, self.flags)
        self._key, self._served = key, 1 << index
        return self._out

    def invalidate(self) -> None:
        self._key = None


class FusedMember(nn.Module):
    """Stands where a VQuantLinear stood; `layer` is that VQuantLinear (state_dict keys gain no prefix: see
    `_save_to_state_dict` / `_load_from_state_dict` -- the wrapped layer's entries are stored at this level)."""

    def __init__(self, layer: VQuantLinear, group: FusedGroup, index: int):
        super().__init__()
        # in lists: plain python references, NOT registered sub-modules -- the wrapper must not add a
        # "layer." level to the state_dict keys, and nn.Module's loader must not recurse into it
        self._layer = [layer]
        self._group = [group]
        self._index = index
        self.in_features, self.out_features = layer.in_features, layer.out_features

    @property
    def layer(self) -> VQuantLinear:
        return self._layer[0]

    # the wrapper is transparent for checkpoints: "<name>.indices", not "<name>.layer.indices"
    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        return self.layer.state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        sub = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
        res = self.layer.load_state_dict(sub, strict=False)
        missing_keys.extend(prefix + k for k in res.missing_keys)
        unexpected_keys.extend(prefix + k for k in res.unexpected_keys)
        self._group[0].invalidate()

    def _apply(self, fn, recurse=True):   # .to() / .cuda() / .half() reach the wrapped layer too
        self.layer._apply(fn)
        self._group[0].invalidate()
        return super()._apply(fn, recurse)

    def named_parameters(self, prefix="", recurse=True, remove_duplicate=True):
        return self.layer.named_parameters(prefix=prefix, recurse=recurse, remove_duplicate=remove_duplicate)

    def parameters(self, recurse=True):
        return self.layer.parameters(recurse=recurse)

    def forward(self, x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        g = self._group[0]
        if args or kwargs or self.layer.enable_proxy_error:
            return self.layer(x, *args, **kwargs)
        out = g.outputs(x, self._index)
        if out is None:
            return self.layer(x)
        a = sum(g.widths[:self._index])
        return out[:, a:a + g.widths[self._index]].reshape(*x.shape[:-1], self.out_features)


def _eligible(layers: Iterable[nn.Module]) -> bool:
    layers = list(layers)
    if not layers or not all(isinstance(l, VQuantLinear) for l in layers):
        return False
    l0 = layers[0]
    return all(l.in_features == l0.in_features and l.centroids.weight.dtype == l0.centroids.weight.dtype and
               l.centroids.weight.device == l0.centroids.weight.device and l.vector_len == l0.vector_len and
               l.vector_len in (8, 16) and not l.enable_proxy_error for l in layers)


def fuse(model: nn.Module, groups: Sequence[Sequence[str]] = DEFAULT_GROUPS, pdl: bool = False,
         prepare: bool = True) -> List[FusedGroup]:
    """Fuse every complete sibling group found in `model` (in place).  Returns the groups created.

    pdl: launch the fused GEMVs with programmatic dependent launch (legal when each group's x is produced by
    the kernel enqueued just before it on the same stream; inside a captured CUDA graph it removes the launch
    gap).  prepare: also build the descriptors of ALL VQuantLinear layers of the model now."""
    made: List[FusedGroup] = []
    for parent in list(model.modules()):
        for names in groups:
            members = [getattr(parent, n, None) for n in names]
            if any(m is None for m in members) or not _eligible(members):
                continue
            g = FusedGroup(members, flags=native.FLAG_PDL if pdl else 0)
            for i, (n, m) in enumerate(zip(names, members)):
                setattr(parent, n, FusedMember(m, g, i))
            made.append(g)
    if prepare:
        for mod in model.modules():
            if isinstance(mod, VQuantLinear) and mod.centroids.weight.is_cuda and not mod.enable_proxy_error:
                mod.prepare()
    return made


def set_quant_grad(model: nn.Module, enabled: bool = True) -> int:
    """`VQuantLinear.set_quant_grad(enabled)` on every VQuantLinear of `model`, fused members included.  Returns how
    many layers it reached."""
    layers = [mod.layer if isinstance(mod, FusedMember) else mod for mod in model.modules()]
    layers = [l for l in layers if isinstance(l, VQuantLinear)]
    if enabled:
        for l in layers:          # refuse before any layer changes: all or nothing
            l._check_quant_grad_possible()
    for l in layers:
        l.set_quant_grad(enabled)
    return len(layers)


def set_batched_decode(model: nn.Module, enabled: bool = True) -> int:
    """`VQuantLinear.set_batched_decode(enabled)` on every VQuantLinear of `model`, fused members included.  Returns
    how many layers it reached."""
    layers = [mod.layer if isinstance(mod, FusedMember) else mod for mod in model.modules()]
    layers = [l for l in layers if isinstance(l, VQuantLinear)]
    for l in layers:
        l.set_batched_decode(enabled)
    return len(layers)


def set_lists_prefill(model: nn.Module, enabled: bool = True) -> int:
    """`VQuantLinear.set_lists_prefill(enabled)` on every VQuantLinear of `model`, fused members included.  Returns
    how many layers it reached."""
    layers = [mod.layer if isinstance(mod, FusedMember) else mod for mod in model.modules()]
    layers = [l for l in layers if isinstance(l, VQuantLinear)]
    for l in layers:
        l.set_lists_prefill(enabled)
    return len(layers)


def set_list_decode(model: nn.Module, enabled: bool = True) -> int:
    """`VQuantLinear.set_list_decode(enabled)` on every VQuantLinear of `model`, fused members included (it changes
    only vector-length-16 layers the v = 16 list kernel takes).  Returns how many layers it reached."""
    layers = [mod.layer if isinstance(mod, FusedMember) else mod for mod in model.modules()]
    layers = [l for l in layers if isinstance(l, VQuantLinear)]
    for l in layers:
        l.set_list_decode(enabled)
    return len(layers)


def unfuse(model: nn.Module) -> int:
    """Put the original VQuantLinear layers back.  Returns how many members were unwrapped."""
    n = 0
    for parent in list(model.modules()):
        for name, child in list(parent.named_children()):
            if isinstance(child, FusedMember):
                setattr(parent, name, child.layer)
                n += 1
    return n
