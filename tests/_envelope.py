"""Oracle layers with chosen index data, and the list-shape statistics of the decode list kernel's work split.

`vo.make_layer` draws every main and residual index uniformly.  `layer_with(...)` builds the same layer and then
replaces `meta["idx"]` / `meta["ridx"]` by an index pattern of `PATTERNS` (or arrays given by the caller) and re-packs
them with `vo.pack_index`, so every field width b = ib + rb from 1 to 32 and every list shape the kernels can meet
is reachable.
"""
import math

import numpy as np

import vptq_oracle as vo

SLICE = 4096        # codebook entries per list-kernel slice (vptq_b200.lists.SLICE_ENTRIES)


def _width_pair(b):
    """one (K, Kr) pair of field width b (Kr = -1: no residual); residual codebooks grow with b above 16 bits"""
    if b == 1:
        return 2, -1
    if b <= 16:
        return (2 ** b, -1) if b % 2 == 0 else (2 ** (b - 1), 2)
    return 65536, 2 ** (b - 16)


# every width once, then the pairs where the codebooks' sizes matter: a tiny main codebook over a 65536-entry
# residual one, 65536 + 512 (the smallest residual over 8 bits at K = 65536), both codebooks 2^15 and 2^16 entries
WIDTH_PAIRS = [_width_pair(b) for b in range(1, 33)] + [
    (2, 2), (256, 65536), (4096, 65536), (65536, 512), (65536, 8192), (32768, 65536), (65536, 32768)]
WIDTH_PAIRS = list(dict.fromkeys(WIDTH_PAIRS))


def _bits(n):
    return int(math.log2(n)) if n > 0 else 0


def _zipf_ranks(rng, K, shape, a=1.1):
    """entry ranks 0..K-1 drawn with P(rank k) ~ (k + 1)^-a (rank 0 is the hottest)"""
    p = 1.0 / np.arange(1, K + 1, dtype=np.float64) ** a
    return rng.choice(K, size=shape, p=p / p.sum())


def pattern(kind, K, shape, rng, perm=None):
    """Main indices [G, Ro, gs] of pattern `kind`:
      uniform       every entry equally likely (what make_layer draws)
      ones          K - 1 everywhere: an all-ones field together with the residual's all-ones part
      zipf_hot0     Zipf over entries (exponent 1.1), the hottest entries are 0, 1, 2, ... (all in slice 0)
      zipf_spread   the same ranks scattered over the whole codebook by a fixed permutation
      row_slice     every field of index row r in slice r mod NS: the row's other lists are empty
      constant      one index everywhere
      ramp          row r takes a slice-0 entry with probability r / (Ro - 1), else a uniform one: empty units sit
                    next to units that hold a whole column tile
      col_slice     the slice depends on the ORIGINAL input feature of the column (given perm; identity if None)"""
    G, Ro, gs = shape
    NS = max(K // SLICE, 1)
    if kind == "uniform":
        return rng.integers(0, K, size=shape, dtype=np.int64)
    if kind == "ones":
        return np.full(shape, K - 1, dtype=np.int64)
    if kind == "zipf_hot0":
        return _zipf_ranks(rng, K, shape).astype(np.int64)
    if kind == "zipf_spread":
        scatter = np.random.default_rng(4242).permutation(K)
        return scatter[_zipf_ranks(rng, K, shape)].astype(np.int64)
    if kind == "row_slice":
        s = (np.arange(Ro) % NS)[None, :, None]
        return (s * SLICE + rng.integers(0, min(K, SLICE), size=shape)).astype(np.int64)
    if kind == "constant":
        return np.full(shape, min(K - 1, SLICE + 3), dtype=np.int64)
    if kind == "ramp":
        frac = (np.arange(Ro) / max(Ro - 1, 1))[None, :, None]
        hot = rng.random(shape) < frac
        return np.where(hot, rng.integers(0, min(K, SLICE), size=shape), rng.integers(0, K, size=shape))
    if kind == "col_slice":
        I = G * gs
        feat = np.arange(I) if perm is None else np.asarray(perm).astype(np.uint16).astype(np.int64)
        s = ((feat * NS) // I).reshape(G, 1, gs)   # contiguous feature ranges per slice
        return (s * SLICE + rng.integers(0, min(K, SLICE), size=shape)).astype(np.int64)
    raise ValueError(kind)


PATTERNS = ("uniform", "ones", "zipf_hot0", "zipf_spread", "row_slice", "constant", "ramp", "col_slice")


def layer_with(kind="uniform", res_kind=None, *, seed=1234, idx=None, ridx=None, **kw):
    """`vo.make_layer(**kw)` with the main indices of pattern `kind` (or `idx`) and the residual indices of
    `res_kind` (default: `ones` for `ones`, else uniform; or `ridx`), re-packed.  meta keeps the arrays."""
    L = vo.make_layer(seed=seed, **kw)
    K, Kr = L.num_centroids, L.num_res_centroids
    G, gs = L.num_codebooks, L.group_size
    Ro = (L.out_features + L.vector_len - 1) // L.vector_len
    rng = np.random.default_rng(seed + 17)
    if idx is None:
        idx = pattern(kind, K, (G, Ro, gs), rng, perm=L.perm if G == 1 and not L.enable_outlier else None)
    if Kr > 0 and ridx is None:
        rk = res_kind or ("ones" if kind == "ones" else "uniform")
        ridx = np.full((G, Ro, gs), Kr - 1, np.int64) if rk == "ones" else rng.integers(0, Kr, size=(G, Ro, gs))
    if Kr <= 0:
        ridx = None
    assert idx.min() >= 0 and idx.max() < K and (ridx is None or (ridx.min() >= 0 and ridx.max() < Kr))
    L.indices = vo.pack_index(idx, _bits(K), ridx, _bits(Kr))
    L.meta = dict(idx=idx, ridx=ridx, seed=seed)
    return L


# ----------------------------------------------------------------------------------------------------------------
# list shapes under the kernel's work split (csrc/gemv_lists.cu: units split evenly over CTAs, each CTA's steps
# split evenly over 16 warps, stages of 8 steps; the same arithmetic as test_lists_format._kernel_partition)
# ----------------------------------------------------------------------------------------------------------------
def list_shape_stats(first, tail, Ro, Q, ncta, warps=16, sps=8):
    """-> dict: max_warps_per_unit (warp runs a unit's steps touch), empty_cta_share (largest share of a CTA's units
    that are 1-step empty lists), max_ends_per_stage (unit ends inside one 8-step stage of one warp),
    max_steps_per_cta / mean_steps_per_cta."""
    U = Q * Ro
    n_valid = (np.diff(first) - 1) * 32 + tail[:-1]
    empty = (np.diff(first) == 1) & (n_valid == 0)
    max_warps, empty_share, max_ends, steps = 0, 0.0, 0, []
    for q in range(ncta):
        u0, u1 = U * q // ncta, U * (q + 1) // ncta
        T0, T1 = int(first[u0]), int(first[u1])
        TT = T1 - T0
        steps.append(TT)
        empty_share = max(empty_share, float(empty[u0:u1].mean()) if u1 > u0 else 0.0)
        # warp w runs steps [T0 + TT*w/warps, T0 + TT*(w+1)/warps)
        bounds = [T0 + TT * w // warps for w in range(warps + 1)]
        ends = first[u0 + 1:u1 + 1] - 1          # the last step of every unit of this CTA
        starts = first[u0:u1]
        for a, b in zip(starts, ends):
            wa = np.searchsorted(bounds, a, side="right") - 1
            wb = np.searchsorted(bounds, b, side="right") - 1
            max_warps = max(max_warps, int(wb - wa + 1))
        for w in range(warps):
            a, b = bounds[w], bounds[w + 1]
            for s in range(a, b, sps):
                e = np.count_nonzero((ends >= s) & (ends < min(s + sps, b)))
                max_ends = max(max_ends, int(e))
    return dict(max_warps_per_unit=max_warps, empty_cta_share=empty_share, max_ends_per_stage=max_ends,
                max_steps_per_cta=int(max(steps)), mean_steps_per_cta=float(np.mean(steps)))
