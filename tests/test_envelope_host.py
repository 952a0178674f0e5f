"""The index envelope on the host (no GPU needed): every field width b = 1..32, the list builders on skewed index
patterns, the refusal of a one-entry residual codebook, and a decode plan for every layer validate() accepts.

A decode plan exists for a layer when vptq_b200_workspace_bytes(desc, 1 | 2, VPTQ_OP_GEMV) > 0.  Without a device the
library plans for the H100 SXM geometry (132 SMs, 232448 bytes of opt-in shared memory).  The descriptors carry fake,
aligned addresses: nothing is launched or dereferenced.
"""
import ctypes

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _envelope import PATTERNS, layer_with, pattern
from vptq_b200 import lists, pack

from _envelope import WIDTH_PAIRS as PAIRS   # (K, Kr), Kr = -1 for none: b = ib + rb from 1 to 32


def _b(K, Kr):
    return int(np.log2(K)) + (int(np.log2(Kr)) if Kr > 0 else 0)


def test_pairs_cover_every_width():
    assert sorted({_b(K, Kr) for K, Kr in PAIRS}) == list(range(1, 33))


@pytest.mark.parametrize("K,Kr", PAIRS)
@pytest.mark.parametrize("kind", ["uniform", "ones"])
def test_packing_round_trip_at_every_width(K, Kr, kind):
    """vptq_b200.pack and the oracle's packer write the same words, and both unpack them to the fields packed"""
    rng = np.random.default_rng(_b(K, Kr))
    n, rows = 67, 5                                          # 67 fields: a ragged last word at every odd width
    idx = np.full((1, rows, n), K - 1) if kind == "ones" else rng.integers(0, K, size=(1, rows, n))
    ridx = None
    if Kr > 0:
        ridx = np.full((1, rows, n), Kr - 1) if kind == "ones" else rng.integers(0, Kr, size=(1, rows, n))
    ib, rb = int(np.log2(K)), (int(np.log2(Kr)) if Kr > 0 else 0)
    w_oracle = vo.pack_index(idx, ib, ridx, rb)
    w_torch = pack.pack_index(torch.from_numpy(idx), ib, None if ridx is None else torch.from_numpy(ridx), rb)
    assert w_torch.dtype == torch.int32 and w_torch.shape[-1] == (n * (ib + rb) + 31) // 32
    assert np.array_equal(np.asarray(w_oracle).astype(np.int64) & 0xFFFFFFFF, w_torch.numpy().astype(np.int64) & 0xFFFFFFFF)
    i2, r2 = pack.unpack_index_tensor(w_torch, ib, n, rb)
    assert np.array_equal(i2.numpy(), idx)
    assert (r2 is None) == (ridx is None) and (r2 is None or np.array_equal(r2.numpy(), ridx))
    i3, r3 = vo.unpack_index(w_oracle, ib, n, rb)
    assert np.array_equal(i3, idx) and (ridx is None or np.array_equal(r3, ridx))
    if kind == "ones" and (ib + rb) * n % 32 == 0:
        assert (w_torch == -1).all()                         # every bit set: the 32-bit field fills whole words


# ----------------------------------------------------------------------------------------------------------------
# list builders on the skewed patterns
# ----------------------------------------------------------------------------------------------------------------
def _c_build(ind, O, I, K, Kr):
    from vptq_b200 import native
    lib = native.lib()
    ind = np.ascontiguousarray(ind)
    NS, NT, _ = lists.geometry(I, K)
    tab = np.zeros(NS * NT * ((O + 7) // 8) + 1, dtype=np.uint32)
    steps, tcw = ctypes.c_size_t(0), ctypes.c_int32(0)
    args = (ind.ctypes.data, ind.shape[1], O, I, K, Kr, None)
    assert lib.vptq_b200_lists_build_host(*args, None, 0, tab.ctypes.data, ctypes.byref(steps), ctypes.byref(tcw)) == 0
    out = np.zeros(steps.value * 32, dtype=np.uint32)
    assert lib.vptq_b200_lists_build_host(*args, out.ctypes.data, out.nbytes, tab.ctypes.data, ctypes.byref(steps),
                                          ctypes.byref(tcw)) == 0, native.last_error()
    assert lib.vptq_b200_lists_deal_host(out.ctypes.data, tab.ctypes.data, len(tab) - 1, 0) == 0
    return out, tab


LIST_PATTERNS = [p for p in PATTERNS if p != "ones"] + ["ones"]


@pytest.mark.parametrize("kind", LIST_PATTERNS)
@pytest.mark.parametrize("Kr", [2, 256])
def test_list_builders_agree_on_skewed_patterns(kind, Kr):
    """The C host builder and the tensor builder give the same bytes, and the lists evaluate to the oracle's sum.
    col_slice runs without perm (the slice then follows the column); the others with perm."""
    I, O, K = 1536, 136, 16384
    L = layer_with(kind, in_features=I, out_features=O, num_centroids=K, num_res_centroids=Kr,
                   enable_perm=kind != "col_slice", seed=31)
    ind = torch.from_numpy(np.ascontiguousarray(L.indices))
    pt = None if L.perm is None else torch.from_numpy(np.asarray(L.perm).astype(np.uint16).astype(np.int64))
    stream, tab, _ = lists.build_lists(ind, num_centroids=K, num_res_centroids=Kr, in_features=I, out_features=O,
                                       perm=pt)
    if L.perm is None:      # the C builder with perm = NULL
        out, tab_c = _c_build(L.indices[0], O, I, K, Kr)
        assert np.array_equal(out, stream.numpy().reshape(-1).view(np.uint32))
        assert np.array_equal(tab_c.astype(np.int64), tab.numpy().astype(np.int64) & 0xFFFFFFFF)
    else:
        from vptq_b200 import native
        lib = native.lib()
        pp = np.ascontiguousarray(np.asarray(L.perm).astype(np.uint16))
        src = np.ascontiguousarray(L.indices[0])
        NS, NT, _ = lists.geometry(I, K)
        tab_c = np.zeros(NS * NT * ((O + 7) // 8) + 1, dtype=np.uint32)
        steps, tcw = ctypes.c_size_t(0), ctypes.c_int32(0)
        args = (src.ctypes.data, src.shape[1], O, I, K, Kr, pp.ctypes.data)
        assert lib.vptq_b200_lists_build_host(*args, None, 0, tab_c.ctypes.data, ctypes.byref(steps),
                                              ctypes.byref(tcw)) == 0
        out = np.zeros(steps.value * 32, dtype=np.uint32)
        assert lib.vptq_b200_lists_build_host(*args, out.ctypes.data, out.nbytes, tab_c.ctypes.data,
                                              ctypes.byref(steps), ctypes.byref(tcw)) == 0
        assert lib.vptq_b200_lists_deal_host(out.ctypes.data, tab_c.ctypes.data, len(tab_c) - 1, 0) == 0
        assert np.array_equal(out, stream.numpy().reshape(-1).view(np.uint32))
        assert np.array_equal(tab_c.astype(np.int64), tab.numpy().astype(np.int64) & 0xFFFFFFFF)
    x = vo.make_x(1, I, "fp16", seed=3)
    xf = vo.to_f32(x, "fp16").astype(np.float64).reshape(-1)
    sc = vo.to_f32(L.weight_scale, "fp16").astype(np.float64)
    wb = vo.to_f32(L.weight_bias, "fp16").astype(np.float64)
    y = lists.emulate(stream, tab, num_centroids=K, num_res_centroids=Kr, in_features=I, out_features=O,
                      centroids=torch.from_numpy(vo.to_f32(L.centroids, "fp16")),
                      res_centroids=torch.from_numpy(vo.to_f32(L.res_centroids, "fp16")),
                      xs=torch.from_numpy(xf * sc)).numpy()[:O] + float((xf * wb).sum())
    y_star = vo.quant_gemm(x, L).astype(np.float64).reshape(-1)
    assert np.max(np.abs(y - y_star)) <= 1e-5 * max(1.0, np.max(np.abs(y_star)))


def test_patterns_are_what_they_claim():
    rng = np.random.default_rng(0)
    K, shape = 65536, (1, 64, 4096)
    NS = K // 4096
    z0 = pattern("zipf_hot0", K, shape, rng)
    assert (z0 < 4096).mean() > 0.5                          # the hot entries sit in slice 0
    zs = pattern("zipf_spread", K, shape, rng)
    assert np.bincount(zs.reshape(-1) >> 12, minlength=NS).min() > 0
    rs = pattern("row_slice", K, shape, rng)
    assert ((rs[0] >> 12) == (np.arange(64) % NS)[:, None]).all()
    assert (pattern("constant", K, shape, rng) == 4099).all()
    rp = pattern("ramp", K, shape, rng)
    assert (rp[0, -1] < 4096).all() and (rp[0, 0] < 4096).mean() < 0.2
    cs = pattern("col_slice", K, shape, rng)
    assert ((cs[0] >> 12) == (np.arange(4096) * NS // 4096)[None, :]).all()


# ----------------------------------------------------------------------------------------------------------------
# descriptors with fake addresses: validation and planning only
# ----------------------------------------------------------------------------------------------------------------
def _desc(v, K, Kr, I=4096, O=4096, G=1):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    ib, rb = int(np.log2(K)), (int(np.log2(Kr)) if Kr > 1 else 0)
    gs = I // G
    words = (gs * (ib + rb) + 31) // 32
    vals = dict(dtype=0, in_features=I, out_features=O, vector_len=v, num_centroids=K, num_res_centroids=Kr,
                num_codebooks=G, group_size=gs, outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1,
                indices=0x1000_0000, index_stride_codebook=words * ((O + v - 1) // v), index_stride_row=words,
                centroids=0x2000_0000, centroid_stride=K * v,
                res_centroids=0x3000_0000 if Kr > 0 else None, res_centroid_stride=max(Kr, 0) * v,
                perm=0x4000_0000, weight_scale=0x5000_0000, weight_bias=0x5100_0000)
    for k, x in vals.items():
        setattr(d, k, x)
    return d


def test_one_residual_entry_is_refused():
    """Kr = 1 means 0 residual index bits: the packed format cannot carry it.  Refused without a device, also when
    the residual pointer is NULL (the check must not depend on it)."""
    from vptq_b200 import VQuantLinear, native
    OP_GEMV = native.OP_GEMV
    for res_ptr in (0x3000_0000, None):
        d = _desc(8, 4096, 1)
        d.res_centroids = res_ptr
        assert native.workspace_bytes(d, 1, OP_GEMV) == 0
        msg = native.last_error()
        assert "num_res_centroids 1" in msg and "[2,65536]" in msg, msg
    assert native.workspace_bytes(_desc(8, 4096, 2), 1, OP_GEMV) > 0           # the smallest legal residual
    assert native.workspace_bytes(_desc(8, 4096, -1), 1, OP_GEMV) > 0          # no residual
    with pytest.raises(ValueError, match="num_res_centroids = 1"):
        VQuantLinear(1024, 256, vector_lens=[-1, 8], num_centroids=[-1, 4096], num_res_centroids=[-1, 1], group_num=1,
                     group_size=1024, outlier_size=0, indices_as_float=False, is_indice_packed=True, device="meta")


VS = (2, 4, 6, 8, 10, 12, 16)
KS = tuple(2 ** k for k in range(1, 17))
KRS = (-1,) + tuple(2 ** k for k in range(1, 17))


@pytest.mark.parametrize("v", VS)
def test_every_accepted_layer_has_a_decode_plan(v):
    """1 and 2 tokens, every K and Kr with ib + rb <= 32 (4096 x 4096).  Before the residual codebook could be gathered
    through L1/L2, residual codebooks of 256 KiB and more had no plan."""
    from vptq_b200 import native
    missing = []
    for K in KS:
        for Kr in KRS:
            if _b(K, Kr) > 32:
                continue
            if (K * v * 2) % 16:
                continue            # validate() refuses a codebook that is not a whole number of 16-byte words
            d = _desc(v, K, Kr)
            for tokens in (1, 2):
                if native.workspace_bytes(d, tokens, native.OP_GEMV) == 0:
                    missing.append((K, Kr, tokens, native.last_error()))
    assert not missing, missing[:6]


def test_codebooks_past_65536_entries_are_refused():
    from vptq_b200 import native
    assert native.workspace_bytes(_desc(8, 65536, 65536), 1, native.OP_GEMV) > 0    # b = 32 exactly
    d = _desc(8, 65536, 65536)
    d.num_centroids = 131072
    assert native.workspace_bytes(d, 1, native.OP_GEMV) == 0 and "num_centroids" in native.last_error()
    d = _desc(8, 65536, 65536)
    d.num_res_centroids = 131072
    assert native.workspace_bytes(d, 1, native.OP_GEMV) == 0 and "num_res_centroids" in native.last_error()
