"""Prefill, dequant and input gradient from the index lists (include/vptq_b200_lists_dense.h), host-side checks.

* the header's symbol table: exactly LISTS_DENSE_EXPORTS, exported by the library, disjoint from every other header
  and export tuple; include/vptq_b200.h unchanged (15 functions, ABI 7);
* argument validation before any launch, with fake device addresses;
* an integer mirror of what the dense-from-lists kernel relies on, on lists built by vptq_b200_lists_build_host and
  dealt by vptq_b200_lists_deal_host: for every (index row, tile) the NS units hold every feature of the tile exactly
  once with the (main, residual) index of its packed field, and the padding entries are exactly the masked ones.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import vptq_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = ("vptq_b200.h", "vptq_b200_grad.h", "vptq_b200_graph.h", "vptq_b200_batch.h")


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", src)))


def test_lists_dense_header_declares_exactly_its_exports():
    from vptq_b200 import native
    L = native.lib()
    syms = _declared("vptq_b200_lists_dense.h")
    assert syms == sorted(native.LISTS_DENSE_EXPORTS)
    for s in syms:
        assert hasattr(L, s), s
    assert L.vptq_b200_lists_dense_version() == native.LISTS_DENSE_VERSION == 1
    src = open(os.path.join(ROOT, "include", "vptq_b200_lists_dense.h")).read()
    assert "#define VPTQ_B200_LISTS_DENSE_VERSION 1" in src


def test_lists_dense_symbols_are_disjoint_from_the_other_interfaces():
    from vptq_b200 import native
    mine = set(_declared("vptq_b200_lists_dense.h"))
    for h in HEADERS:
        assert not mine & set(_declared(h)), h
    for t in (native.EXPORTS, native.GRAD_EXPORTS, native.GRAPH_EXPORTS, native.BATCH_EXPORTS):
        assert not mine & set(t)


def test_inference_header_is_unchanged():
    from vptq_b200 import native
    assert len(_declared("vptq_b200.h")) == 15
    src = open(os.path.join(ROOT, "include", "vptq_b200.h")).read()
    assert "#define VPTQ_B200_ABI_VERSION 7" in src
    assert native.lib().vptq_b200_abi_version() == 7


def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    # Llama-3-8B gate/up, decode-only: lists, no packed words (fake, never dereferenced: every call below is refused
    # before anything is launched)
    base = dict(dtype=0, in_features=4096, out_features=14336, vector_len=8, num_centroids=65536,
                num_res_centroids=256, num_codebooks=1, group_size=4096, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=None, index_stride_codebook=0, index_stride_row=3072,
                centroids=0x20000, centroid_stride=65536 * 8, res_centroids=0x30000, res_centroid_stride=2048,
                lists_stream=0x40000, lists_tab=0x50000, lists_tile_cols=4096)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


ZERO = 65536 * 4 + 65536 * 64   # the zero-at-rest head every op leaves untouched


def _align(n, a=1024):
    return (n + a - 1) // a * a


def test_workspace_bytes():
    from vptq_b200 import native
    L = native.lib()
    ws = L.vptq_b200_lists_dense_workspace_bytes
    for tokens in (1, 3, 8192):
        # forward: W [14336][4096] + staged x [tokens][4096]
        assert ws(ctypes.byref(_desc()), tokens, 0) == ZERO + 14336 * 4096 * 2 + _align(tokens * 4096 * 2)
        assert ws(ctypes.byref(_desc()), tokens, native.FLAG_PDL) == ZERO + 14336 * 4096 * 2 + _align(tokens * 4096 * 2)
        # transposed: the layout of VPTQ_OP_GEMM_DGRAD
        assert ws(ctypes.byref(_desc()), tokens, native.FLAG_TRANSPOSE) == \
            ZERO + 4096 * 14336 * 2 + _align(tokens * 14336 * 2)
    # ragged shapes: K extents rounded up to whole 64-element blocks
    ragged = _desc(in_features=1000, out_features=1004, group_size=1000, lists_tile_cols=1000)
    assert ws(ctypes.byref(ragged), 5, 0) == ZERO + _align(1004 * 1024 * 2) + _align(5 * 1024 * 2)
    assert ws(ctypes.byref(ragged), 5, native.FLAG_TRANSPOSE) == ZERO + _align(1000 * 1024 * 2) + _align(5 * 1024 * 2)
    # refusals give 0 and a message
    assert ws(ctypes.byref(_desc(lists_stream=None, lists_tab=None, indices=0x10000)), 1, 0) == 0
    assert "no index lists" in native.last_error()
    assert ws(ctypes.byref(_desc()), 1, 4) == 0
    assert "unknown flags" in native.last_error()


def test_refusals_before_any_launch():
    from vptq_b200 import native
    L = native.lib()
    T = native.FLAG_TRANSPOSE
    gemm, deq = L.vptq_b200_lists_quant_gemm, L.vptq_b200_lists_dequant
    d = _desc()
    ws = 1 << 40
    # a descriptor without lists (full, packed words only): VPTQ_ERR_UNSUPPORTED with a message
    full = _desc(lists_stream=None, lists_tab=None, indices=0x10000)
    for flags in (0, T):
        assert gemm(ctypes.byref(full), 0x1000, 14336, 0x2000, 14336, 8, 0x3000, ws, flags, None) == -2
        assert "no index lists" in native.last_error()
        assert deq(ctypes.byref(full), 0x1000, 14336, flags, None) == -2
    # lists of a layer the list kernels do not take (tile width not the lists geometry's)
    assert deq(ctypes.byref(_desc(lists_tile_cols=2048)), 0x1000, 4096, 0, None) == -2
    # dequant: ld < columns, ld % 8, misaligned or NULL w, unknown flags
    for ld, flags in ((4095, 0), (4100, 0), (14335, T), (14340, T), (4096, T)):
        assert deq(ctypes.byref(d), 0x1000, ld, flags, None) == -1, (ld, flags)
        assert "ld" in native.last_error()
    assert deq(ctypes.byref(d), 0x1008, 4096, 0, None) == -1
    assert deq(ctypes.byref(d), None, 4096, 0, None) == -1
    assert deq(ctypes.byref(d), 0x1000, 4096, native.FLAG_PDL, None) == -1
    # GEMM: tokens < 1, short strides (swapped for the transposed call), NULL x / y, unknown flags
    assert gemm(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 0, 0x3000, ws, 0, None) == -1
    for xs, ys, flags in ((4095, 14336, 0), (4096, 14335, 0), (4096, 14336, T), (14336, 4095, T)):
        assert gemm(ctypes.byref(d), 0x1000, xs, 0x2000, ys, 8, 0x3000, ws, flags, None) == -1, (xs, ys, flags)
        assert "stride" in native.last_error()
    assert gemm(ctypes.byref(d), None, 4096, 0x2000, 14336, 8, 0x3000, ws, 0, None) == -1
    assert gemm(ctypes.byref(d), 0x1000, 4096, None, 14336, 8, 0x3000, ws, 0, None) == -1
    assert gemm(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, 0x3000, ws, 8, None) == -1
    assert "unknown flags" in native.last_error()
    assert gemm(None, 0x1000, 4096, 0x2000, 14336, 8, 0x3000, ws, 0, None) == -1
    if not torch.cuda.is_available():
        # well-formed arguments reach the device check, which fails on a host without an H100
        assert gemm(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, 0x3000, ws, 0, None) < 0
        assert deq(ctypes.byref(d), 0x1000, 4096, 0, None) < 0


# the shapes of the GPU tests (tests/test_gpu_lists.py CASES + the Llama-3-8B layers)
MIRROR = {
    "k65536_r256": dict(in_features=2048, out_features=1024, num_centroids=65536, num_res_centroids=256),
    "k65536_r16_ragged": dict(in_features=1000, out_features=1004, num_centroids=65536, num_res_centroids=16),
    "k65536_i1004": dict(in_features=1004, out_features=512, num_centroids=65536, num_res_centroids=256),
    "k16384_r256": dict(in_features=1536, out_features=512, num_centroids=16384, num_res_centroids=256),
    "k8192_r256": dict(in_features=1536, out_features=512, num_centroids=8192, num_res_centroids=256),
    "k32768_plain": dict(in_features=1024, out_features=256, num_centroids=32768, enable_perm=False, enable_norm=False),
    "k32768_noperm_r64": dict(in_features=1024, out_features=264, num_centroids=32768, num_res_centroids=64,
                              enable_perm=False),
    "k65536_one_row": dict(in_features=4096, out_features=8, num_centroids=65536, num_res_centroids=256),
    "k65536_wide_odd": dict(in_features=9000, out_features=72, num_centroids=65536, num_res_centroids=256),
    "k65536_many_rows": dict(in_features=512, out_features=16384, num_centroids=65536, num_res_centroids=256),
    "llama_4096x4096": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256),
    "llama_4096x14336": dict(in_features=4096, out_features=14336, num_centroids=65536, num_res_centroids=256),
    "llama_14336x4096": dict(in_features=14336, out_features=4096, num_centroids=65536, num_res_centroids=256),
}


def _host_lists(L):
    from vptq_b200 import native
    lib = native.lib()
    ind = np.ascontiguousarray(np.asarray(L.indices, dtype=np.int32)[0])
    pp = None if L.perm is None else np.ascontiguousarray(np.asarray(L.perm).astype(np.uint16))
    ns, nt = L.num_centroids // 4096, (L.in_features + 4095) // 4096
    ro = (L.out_features + 7) // 8
    tab = np.zeros(ns * nt * ro + 1, dtype=np.uint32)
    steps, tcw = ctypes.c_size_t(0), ctypes.c_int32(0)
    args = (ind.ctypes.data, ind.shape[1], L.out_features, L.in_features, L.num_centroids, L.num_res_centroids,
            None if pp is None else pp.ctypes.data)
    assert lib.vptq_b200_lists_build_host(*args, None, 0, tab.ctypes.data, ctypes.byref(steps), ctypes.byref(tcw)) == 0
    stream = np.zeros(steps.value * 32, dtype=np.uint32)
    assert lib.vptq_b200_lists_build_host(*args, stream.ctypes.data, stream.nbytes, tab.ctypes.data,
                                          ctypes.byref(steps), ctypes.byref(tcw)) == 0, native.last_error()
    assert lib.vptq_b200_lists_deal_host(stream.ctypes.data, tab.ctypes.data, len(tab) - 1, 0) == 0
    return stream.reshape(-1, 32), tab, ns, nt, ro, tcw.value


@pytest.mark.parametrize("name", sorted(MIRROR))
def test_integer_mirror_every_feature_once_padding_masked(name):
    L = vo.make_layer(vector_len=8, seed=41, **MIRROR[name])
    stream, tab, ns, nt, ro, tcw = _host_lists(L)
    I = L.in_features
    U = ns * nt * ro
    first, valid_last, end = tab[:U] & ((1 << 26) - 1), tab[:U] >> 26, tab[1:] & ((1 << 26) - 1)
    nsteps = (end - first).astype(np.int64)
    assert (nsteps >= 1).all() and (valid_last <= 32).all() and int(end[-1]) == stream.shape[0]
    assert (first[1:] == end[:-1]).all()
    step_unit = np.repeat(np.arange(U), nsteps)
    step_local = np.arange(stream.shape[0]) - np.repeat(first.astype(np.int64), nsteps)
    lane = np.arange(32)[None, :]
    # the kernel's mask: every lane of a non-final step, lanes < valid count of the final step
    live = (step_local[:, None] < nsteps[step_unit][:, None] - 1) | (lane < valid_last[step_unit][:, None])
    assert not stream[~live].any()                       # padding entries: zero words, masked by the count
    u = np.broadcast_to(step_unit[:, None], stream.shape)[live]
    e = stream[live].astype(np.int64)
    r, combo = u % ro, u // ro
    s, t = combo % ns, combo // ns
    col = (e >> 12) & 4095
    f = t * tcw + col
    assert (col < tcw).all() and (f < I).all()
    # every (index row, feature) exactly once: NS units of (r, t) partition the tile's features
    key = r * I + f
    assert key.size == ro * I and np.unique(key).size == ro * I
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    inv = np.arange(I) if L.perm is None else np.argsort(np.asarray(L.perm).astype(np.uint16).astype(np.int64))
    c = inv[f]
    assert np.array_equal((e & 4095) + 4096 * s, idx[0][r, c].astype(np.int64))
    want_r = ridx[0][r, c].astype(np.int64) if L.res_bits else np.zeros_like(e)
    assert np.array_equal(e >> 24, want_r)
