"""Load-time re-bucketing of a layer's packed indices into *slice x tile lists* for the decode kernel.

Format contract: include/vptq_b200.h (`vptq_linear_desc::lists_stream`, `::lists_tab`,
`::lists_tile_cols`); consumer: vptq_b200/csrc/gemv_lists.cu.

Why.  A main codebook of K = 65536 entries (1 MiB) cannot sit in one SM's shared memory, and gathering
it through L1/L2 is bound by the L1TEX tag stage.
A sum does not care about the order of its terms, so the fields of every index row are re-bucketed:

  * the codebook is cut into NS = K / 4096 slices of 64 KiB (a 12-bit index inside a slice);
  * the ORIGINAL input features are cut into NT = ceil(I / 4096) tiles of TCW columns (TCW a multiple of 8,
    <= 4096: a 12-bit column inside a tile).  The permutation is folded in here: an entry carries
    perm[c] - tile * TCW, so the kernel's x' tile is the coalesced x[f] * scale[f] -- no perm load, no
    dependent gather on the critical path (the idea of the reference's absorb_perm,
    vptq/utils/pack.py:284-394, without touching the checkpoint);
  * combo = tile * NS + slice; unit u = combo * Ro + r is the list of the fields of index row r that
    fall into that (tile, slice).  Entry = 32 bits: index & 4095 | column << 12 | residual index << 24
    -- 4 bytes per field instead of the 3 packed + 5 listed bytes of the round-1 format;
  * inside a list the entries are dealt round-robin over the eight 16-byte bank groups (index & 7), so the
    8 lanes of a quarter-warp read 8 different bank groups of the slice: conflict-free LDS.128; a second pass
    (`deal_lists`, C code in the shared library, CPU threads) re-orders every list so that the 32 lanes of a
    step also read distinct x' banks where a matching exists -- pure re-ordering, results unchanged;
  * lists are padded to whole steps of 32 entries (every list has >= 1 step); the padding words are 0 and
    the kernel masks them with the list's tail count, so no null column is needed.

Storage: `stream` int32 [T][32] (step-major, units in increasing u), `tab` int32 [U + 1] with
tab[u] = first step of unit u | (valid entries in the unit's LAST step) << 26, tab[U] = T.

Pure tensor code (argsort / scatter), runs on whatever device `indices` lives on; once per layer.  This is
host-side data layout, not a compute path: the kernel does all arithmetic.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Tuple

import torch

from .pack import unpack_index_tensor

SLICE_ENTRIES = 4096
TILE_MAX = 4096
STEP = 32
STEP_MASK = (1 << 26) - 1


def geometry(in_features: int, num_centroids: int) -> Tuple[int, int, int]:
    """-> (NS slices, NT column tiles, TCW columns per tile)."""
    ns = int(num_centroids) // SLICE_ENTRIES
    nt = (int(in_features) + TILE_MAX - 1) // TILE_MAX
    tcw = ((int(in_features) + nt - 1) // nt + 7) // 8 * 8
    return ns, nt, tcw


def eligible(*, vector_len: int, num_centroids: int, num_res_centroids: int, num_codebooks: int,
             outlier_size: int, in_features: int) -> bool:
    """Mirror of gemv_lists_eligible() (csrc/gemv_lists.cu) for the shape-only conditions."""
    K = int(num_centroids)
    return (vector_len == 8 and num_codebooks == 1 and outlier_size <= 0 and K >= 2 * SLICE_ENTRIES
            and K % SLICE_ENTRIES == 0 and K // SLICE_ENTRIES <= 16 and num_res_centroids <= 256
            and 8 <= in_features <= 65535)


DEAL_DEFAULT = "1"   # VPTQ_B200_LISTS_DEAL when unset


def deal_lists(stream: torch.Tensor, tab: torch.Tensor, threads: int = 0) -> torch.Tensor:
    """Bank-aware re-ordering of the entries inside every list (vptq_b200_lists_deal_host, include/vptq_b200.h).

    Runs on the host (C code, `threads` CPU threads, 0 = all): a device `stream` makes the round trip through
    host memory once, at load time.  Returns `stream` (re-ordered in place)."""
    from . import native
    host = stream.detach().to("cpu").contiguous()
    tab_h = tab.detach().to("cpu").contiguous()
    native.check(native.lib().vptq_b200_lists_deal_host(ctypes.c_void_p(host.data_ptr()), ctypes.c_void_p(tab_h.data_ptr()),
                                                        tab_h.numel() - 1, int(threads)), "lists_deal_host")
    if host.data_ptr() != stream.data_ptr():
        stream.copy_(host)
    return stream


def build_lists(indices: torch.Tensor, *, num_centroids: int, num_res_centroids: int, in_features: int,
                out_features: int, perm: Optional[torch.Tensor], deal: Optional[bool] = None
                ) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """packed int32 [1, >=Ro, W] (+ perm [I], uint16 payload) -> (stream int32 [T, 32], tab int32 [U+1], TCW).

    deal: run `deal_lists` on the result (None = VPTQ_B200_LISTS_DEAL, default on)."""
    K, Kr, I = int(num_centroids), int(num_res_centroids), int(in_features)
    Ro = (int(out_features) + 7) // 8
    ib = K.bit_length() - 1
    rb = (Kr.bit_length() - 1) if Kr > 0 else 0
    NS, NT, TCW = geometry(I, K)
    Q = NS * NT
    dev = indices.device
    idx, ridx = unpack_index_tensor(indices[0, :Ro], ib, I, rb)            # [Ro, I] int64
    if perm is None:
        feat = torch.arange(I, device=dev, dtype=torch.int64)
    elif perm.dtype in (torch.int16, torch.uint16):
        feat = perm.view(torch.uint16).to(torch.int64).to(dev)
    else:
        feat = perm.to(torch.int64).to(dev)
    tile = feat // TCW                                                     # [I]
    lcol = feat - tile * TCW
    low = idx & (SLICE_ENTRIES - 1)
    combo = tile[None, :] * NS + (idx >> 12)                               # [Ro, I]
    key1 = combo * 8 + (low & 7)                                           # (combo, bank group)
    order1 = torch.argsort(key1, dim=1, stable=True)
    k1s = torch.gather(key1, 1, order1)
    cnt = torch.zeros(Ro, Q * 8, dtype=torch.int64, device=dev)
    cnt.scatter_add_(1, key1, torch.ones_like(key1))
    start = cnt.cumsum(1) - cnt
    pos = torch.arange(I, device=dev, dtype=torch.int64)[None, :].expand(Ro, I)
    rank = pos - torch.gather(start, 1, k1s)                               # rank inside its (combo, bank) bucket
    key2 = ((k1s >> 3) * (I + 1) + rank) * 8 + (k1s & 7)                   # combo, then rank, then bank group
    order2 = torch.argsort(key2, dim=1)
    src = torch.gather(order1, 1, order2)                                  # quantised column of each sorted position
    combo_s = torch.gather(k1s >> 3, 1, order2)
    n_rc = cnt.view(Ro, Q, 8).sum(2)                                       # fields of (row, combo)
    row_start = n_rc.cumsum(1) - n_rc
    within = pos - torch.gather(row_start, 1, combo_s)
    steps_rc = torch.clamp((n_rc + STEP - 1) // STEP, min=1)               # every list has at least one step
    tail_rc = n_rc - STEP * (steps_rc - 1)                                 # valid entries of the last step (0..32)
    steps_u = steps_rc.t().contiguous().view(-1)                           # combo-major: u = combo * Ro + r
    first = torch.zeros(Q * Ro + 1, dtype=torch.int64, device=dev)
    first[1:] = steps_u.cumsum(0)
    T = int(first[-1].item())
    if T > STEP_MASK:
        raise RuntimeError(f"lists: {T} steps exceed the 26-bit step counter")
    rows = torch.arange(Ro, device=dev, dtype=torch.int64)[:, None].expand(Ro, I)
    dest = (first[combo_s * Ro + rows] * STEP + within).reshape(-1)
    word = torch.gather(low, 1, src) | (lcol[src] << 12)
    if Kr > 0:
        word = word | (torch.gather(ridx, 1, src) << 24)
    words = torch.zeros(T * STEP, dtype=torch.int64, device=dev)
    words[dest] = word.reshape(-1)
    words = torch.where(words >= (1 << 31), words - (1 << 32), words).to(torch.int32)
    tab = first.clone()
    tab[:-1] |= tail_rc.t().contiguous().view(-1) << 26
    tab = torch.where(tab >= (1 << 31), tab - (1 << 32), tab).to(torch.int32)
    stream, tab = words.view(T, STEP).contiguous(), tab.contiguous()
    if deal is None:
        deal = os.environ.get("VPTQ_B200_LISTS_DEAL", DEAL_DEFAULT) not in ("0", "off", "")
    if deal:
        deal_lists(stream, tab)
    return stream, tab, TCW


def emulate(stream: torch.Tensor, tab: torch.Tensor, *, num_centroids: int, num_res_centroids: int,
            in_features: int, out_features: int, centroids: torch.Tensor, res_centroids: Optional[torch.Tensor],
            xs: torch.Tensor) -> torch.Tensor:
    """float64 evaluation of sum_f xs[f] * (C[idx] + R[ridx]) straight from the lists, xs = x * scale in
    ORIGINAL feature order (test aid: validates the format without a GPU).  Returns [Ro * 8]."""
    K, Kr, I = int(num_centroids), int(num_res_centroids), int(in_features)
    Ro = (int(out_features) + 7) // 8
    NS, NT, TCW = geometry(I, K)
    U = NS * NT * Ro
    T = stream.shape[0]
    w = stream.to(torch.int64) & 0xFFFFFFFF                                                     # [T, 32]
    tb = tab.to(torch.int64) & 0xFFFFFFFF
    first, tail = tb & STEP_MASK, tb >> 26
    assert tb.shape[0] == U + 1 and int(first[-1]) == T
    unit = torch.bucketize(torch.arange(T), first[1:], right=True)                              # unit of each step
    combo, r_of = unit // Ro, unit % Ro
    t_of, s_of = combo // NS, combo % NS
    last = torch.arange(T) + 1 == first[unit + 1]
    valid = torch.arange(STEP)[None, :] < torch.where(last, tail[unit], torch.full_like(unit, STEP))[:, None]
    low, col, rix = w & 4095, (w >> 12) & 4095, w >> 24
    f = t_of[:, None] * TCW + col
    f = torch.where(valid, f, torch.zeros_like(f))
    assert bool((f < I).all())
    wt = centroids.reshape(K, 8).double()[s_of[:, None] * SLICE_ENTRIES + low]                  # [T, 32, 8]
    if Kr > 0:
        wt = wt + res_centroids.reshape(Kr, 8).double()[rix]
    xv = torch.where(valid, xs.double().reshape(-1)[f], torch.zeros(1, dtype=torch.float64))
    contrib = (wt * xv[:, :, None]).sum(1)                                                      # [T, 8]
    y = torch.zeros(Ro, 8, dtype=torch.float64)
    y.index_add_(0, r_of, contrib)
    return y.reshape(-1)
