"""Tensor parallelism for VQuantLinear: out_features sharded over the ranks of one NVLink box.

The reference has no distributed code at all (SURVEY.md 2.2); this is new design, following
BASELINE.json's north_star: rank p owns index rows [p*Ro/P, (p+1)*Ro/P) -- whole rows of the
packed index tensor, so the wire format is untouched -- plus the matching slices of
`outlier_indices` and `bias`; codebooks, `perm`, `weight_scale`, `weight_bias` are indexed by
input column and are replicated.  Each rank computes its slice of y with the fused GEMV /
wgmma GEMM and ONE collective per layer completes y on every rank:

    mode "all_reduce" (north_star): write the slice into a zeroed full-width y, NCCL all-reduce(sum)
    mode "all_gather":              NCCL all-gather of the slices (same result, 1/P of the bytes)

`shard_tensors` / `combine` are plain tensor / torch.distributed code (tested on CPU with gloo,
tests/test_tp_gloo.py); `TPVQuantLinear` is the CUDA module.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .layers import VQuantLinear

__all__ = ["shard_bounds", "shard_tensors", "combine", "TPVQuantLinear", "shard_module"]


def shard_bounds(out_features: int, vector_len: int, outlier_vector_len: int, rank: int, world: int):
    """(row0, row1, o0, o1): index rows and output features owned by `rank`."""
    if out_features % vector_len:
        raise ValueError("tensor parallelism needs out_features to be a multiple of vector_len (no padding rows)")
    rows = out_features // vector_len
    if rows % world:
        raise ValueError(f"{rows} index rows do not divide over {world} ranks")
    per = rows // world
    o0, o1 = rank * per * vector_len, (rank + 1) * per * vector_len
    if outlier_vector_len > 1 and (o0 % outlier_vector_len or o1 % outlier_vector_len):
        raise ValueError("shard boundary splits an outlier vector")
    return rank * per, (rank + 1) * per, o0, o1


def shard_tensors(t: Dict[str, Optional[torch.Tensor]], *, out_features: int, vector_len: int,
                  outlier_vector_len: int, rank: int, world: int) -> Dict[str, Optional[torch.Tensor]]:
    """Slice one layer's state_dict-named tensors for `rank`.  Views where possible (no copy)."""
    r0, r1, o0, o1 = shard_bounds(out_features, vector_len, outlier_vector_len, rank, world)
    out = dict(t)
    out["indices"] = t["indices"][:, r0:r1, :]
    if t.get("res_indices") is not None:
        out["res_indices"] = t["res_indices"][:, r0:r1, :]
    if t.get("outlier_indices") is not None:
        vol = outlier_vector_len
        out["outlier_indices"] = t["outlier_indices"][:, o0 // vol:o1 // vol, :]
    if t.get("bias") is not None:
        out["bias"] = t["bias"][o0:o1]
    return out


def combine(y_local: torch.Tensor, out_features: int, rank: int, world: int, group=None,
            mode: str = "all_reduce", out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[tokens, O/world] slice on every rank -> [tokens, O] on every rank, one collective."""
    tokens, o_loc = y_local.shape
    if o_loc * world != out_features:
        raise ValueError("slice width * world != out_features")
    if world == 1:
        return y_local
    if mode == "all_reduce":
        y = out if out is not None else torch.empty(tokens, out_features, dtype=y_local.dtype, device=y_local.device)
        y.zero_()
        y[:, rank * o_loc:(rank + 1) * o_loc] = y_local
        dist.all_reduce(y, group=group)
        return y
    if mode == "all_gather":
        parts = torch.empty(world * tokens, o_loc, dtype=y_local.dtype, device=y_local.device)
        dist.all_gather_into_tensor(parts, y_local.contiguous(), group=group)   # rank-major concatenation
        return parts.view(world, tokens, o_loc).permute(1, 0, 2).reshape(tokens, out_features)
    raise ValueError(f"unknown mode {mode!r}")


class TPVQuantLinear(nn.Module):
    """A VQuantLinear whose out_features are sharded over `group`; forward returns the full y."""

    def __init__(self, shard: VQuantLinear, out_features: int, rank: int, world: int, group=None,
                 mode: str = "all_reduce"):
        super().__init__()
        self.shard, self.out_features, self.rank, self.world, self.group, self.mode = shard, out_features, rank, world, group, mode
        self.in_features = shard.in_features

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.in_features)
        if self.mode == "all_reduce" and self.world > 1:
            # the kernels write the rank's slice straight into the zeroed full-width buffer (strided y)
            from . import native
            y = torch.zeros(x2.shape[0], self.out_features, dtype=x.dtype, device=x.device)
            o_loc = self.out_features // self.world
            ys = y[:, self.rank * o_loc:(self.rank + 1) * o_loc]
            self.shard(x2[:0])  # builds / refreshes the cached descriptor without launching anything
            desc = self.shard._desc_cache[0]
            (native.quant_gemv if x2.shape[0] < 3 else native.quant_gemm)(desc, x2 if x2.stride(-1) == 1 else x2.contiguous(), ys)
            dist.all_reduce(y, group=self.group)
        else:
            y = combine(self.shard(x2), self.out_features, self.rank, self.world, self.group, self.mode)
        return y.reshape(*lead, self.out_features)


def shard_module(m: VQuantLinear, rank: int, world: int, group=None, mode: str = "all_reduce") -> TPVQuantLinear:
    """Build rank's shard of an (already loaded) VQuantLinear."""
    if m.padding:
        raise ValueError("tensor parallelism needs out_features to be a multiple of vector_len")
    r0, r1, o0, o1 = shard_bounds(m.out_features, m.vector_len, m.outlier_vector_len if m.enable_outlier else 1, rank, world)
    dev, dt = m.centroids.weight.device, m.centroids.weight.dtype
    s = VQuantLinear(m.in_features, o1 - o0, vector_lens=(m.outlier_vector_len, m.vector_len),
                     num_centroids=(m.num_outlier_centroids, m.num_centroids),
                     num_res_centroids=(m.outlier_num_res_centroids, m.num_res_centroids), group_num=m.group_num,
                     group_size=m.group_size, outlier_size=m.outlier_size, indices_as_float=m.indices_as_float,
                     enable_norm=m.enable_norm, enable_perm=m.enable_perm, is_indice_packed=m.is_indice_packed,
                     bias=m.bias is not None, device=dev, dtype=dt, enable_proxy_error=False)
    names = {k: v for k, v in m.state_dict().items()}
    t = shard_tensors({"indices": names["indices"], "res_indices": names.get("res_indices"),
                       "outlier_indices": names.get("outlier_indices"), "bias": names.get("bias")},
                      out_features=m.out_features, vector_len=m.vector_len,
                      outlier_vector_len=m.outlier_vector_len if m.enable_outlier else 1, rank=rank, world=world)
    with torch.no_grad():
        s.indices.data = t["indices"].contiguous()
        if t.get("res_indices") is not None:
            s.res_indices.data = t["res_indices"].contiguous()
        if t.get("outlier_indices") is not None:
            s.outlier_indices.data = t["outlier_indices"].contiguous()
            s.outlier_centroids.weight.data = m.outlier_centroids.weight.data
        if t.get("bias") is not None:
            s.bias.data = t["bias"].contiguous()
        s.centroids.weight.data = m.centroids.weight.data            # replicated (shared storage)
        if m.enable_residual:
            s.res_centroids.weight.data = m.res_centroids.weight.data
        if m.enable_perm:
            s.perm.data = m.perm.data
        if m.enable_norm:
            s.weight_scale.data, s.weight_bias.data = m.weight_scale.data, m.weight_bias.data
    return TPVQuantLinear(s.eval(), m.out_features, rank, world, group, mode)


# ---------------------------------------------------------------------------------------------------
# Exchange fused into the GEMV kernel: peer-mapped activation buffers + epoch flags (no NCCL call)
# ---------------------------------------------------------------------------------------------------
class PeerArena:
    """One symmetric byte arena per rank, mapped into every rank of the group (NVLink peer access).

    Sub-allocations are taken at identical offsets on every rank, so `peer_ptr(r, off)` is the address of
    the same object in rank r's arena.  Built on torch.distributed._symmetric_memory (CUDA VMM handles
    exchanged through the process group's store); nothing here is on the hot path.
    """

    def __init__(self, nbytes: int, device: torch.device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.nbytes = (int(nbytes) + 1023) // 1024 * 1024
        self.buf = symm_mem.empty(self.nbytes, dtype=torch.uint8, device=device)
        self.handle = symm_mem.rendezvous(self.buf, self.group)
        self.ptrs = [int(p) for p in self.handle.buffer_ptrs]
        self.buf.zero_()
        torch.cuda.synchronize(device)
        dist.barrier(self.group)
        self._top = 0

    def alloc(self, shape, dtype) -> "tuple[torch.Tensor, int]":
        """(local tensor view, byte offset) -- call in the same order with the same sizes on every rank."""
        n = 1
        for s in shape:
            n *= int(s)
        nb = n * torch.empty(0, dtype=dtype).element_size()
        off = (self._top + 255) // 256 * 256
        if off + nb > self.nbytes:
            raise RuntimeError("PeerArena exhausted")
        self._top = off + nb
        return self.buf[off:off + nb].view(dtype).view(*shape), off

    def peer_ptr(self, rank: int, offset: int) -> int:
        return self.ptrs[rank] + offset


def make_exchange(arena: PeerArena, *, slot: int, wait_slot: int, y_offsets, slice_bytes, flags_offset: int,
                  epoch: torch.Tensor, done: torch.Tensor, error: torch.Tensor, fmt: int = 0, num_slots: int = 0):
    """Fill a vptq_tp_exchange for one launch: y_offsets[l] = byte offset (in the arena) of layer l's FULL-width
    output buffer, slice_bytes[l] = byte offset of this rank's slice inside it.  fmt = native.TP_TAGGED: the
    buffers are tagged-word buffers (4 bytes per output, include/vptq_b200.h) and num_slots = launches per token."""
    from . import native
    ex = native.TpExchange()
    import ctypes
    ex.struct_size = ctypes.sizeof(native.TpExchange)
    ex.world, ex.rank, ex.slot, ex.wait_slot = arena.world, arena.rank, slot, wait_slot
    for l, (yo, sb) in enumerate(zip(y_offsets, slice_bytes)):
        for r in range(arena.world):
            ex.peer_y[l][r] = arena.peer_ptr(r, yo + sb)
    for r in range(arena.world):
        ex.peer_flags[r] = arena.peer_ptr(r, flags_offset)
    ex.epoch, ex.done, ex.error = epoch.data_ptr(), done.data_ptr(), error.data_ptr()
    ex.format, ex.num_slots = int(fmt), int(num_slots)
    return ex


def untag(buf: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Tagged-word buffer (uint8 view, 8 bytes per pair of outputs) -> the plain 16-bit values."""
    return buf.view(torch.int32).view(-1, 2)[:, 0].contiguous().view(dtype).view(1, -1)
