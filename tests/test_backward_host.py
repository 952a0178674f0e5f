"""Input gradient of the quantized linear layer, host-side checks (no GPU needed).

* the dX oracle (tests/_dgrad.py) against autograd through the CPU port of the reference's differentiable torch
  path (oracle/torch_port.py) on every golden fixture;
* the C ABI of VPTQ_FLAG_TRANSPOSE: workspace size of VPTQ_OP_GEMM_DGRAD and argument validation.
"""
import ctypes

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _dgrad import quant_gemm_dgrad
from _util import golden_names, load_golden


@pytest.mark.parametrize("name", golden_names())
def test_dgrad_oracle_matches_torch_port_autograd(name):
    import torch_port as tp
    L, x, ref = load_golden(name)
    f = (lambda a: None if a is None else (torch.from_numpy(np.asarray(a, dtype=np.float16).copy()) if L.dtype == "fp16"
         else torch.from_numpy(np.asarray(a, dtype=np.uint16).copy()).view(torch.bfloat16)))
    u = lambda a: None if a is None else torch.from_numpy(np.asarray(a, dtype=np.uint16).copy()).view(torch.int16)
    d = dict(in_features=L.in_features, out_features=L.out_features, vector_len=L.vector_len,
             num_centroids=L.num_centroids, num_res_centroids=L.num_res_centroids, num_codebooks=L.num_codebooks,
             group_size=L.group_size, outlier_size=L.outlier_size if L.enable_outlier else 0,
             outlier_vector_len=L.outlier_vector_len, num_outlier_centroids=L.num_outlier_centroids,
             indices=torch.from_numpy(L.indices.copy()), centroids=f(L.centroids), res_centroids=f(L.res_centroids),
             outlier_indices=u(L.outlier_indices), outlier_centroids=f(L.outlier_centroids), perm=u(L.perm),
             weight_scale=f(L.weight_scale), weight_bias=f(L.weight_bias), bias=f(L.bias))
    dy = vo.make_x(x.shape[0], L.out_features, L.dtype, seed=11)
    xt = f(x).float().requires_grad_()
    tp.quant_gemm(xt, d).backward(f(dy).float())
    want = quant_gemm_dgrad(dy, L)
    assert want.shape == (x.shape[0], L.in_features)
    err = np.abs(xt.grad.numpy() - want).max() / np.abs(want).max()
    assert err <= 1e-5, f"{name}: {err:.3e}"


def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    base = dict(dtype=0, in_features=4096, out_features=14336, vector_len=8, num_centroids=65536,
                num_res_centroids=256, num_codebooks=1, group_size=4096, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=0x10000, index_stride_codebook=1792 * 3072, index_stride_row=3072,
                centroids=0x20000, centroid_stride=65536 * 8, res_centroids=0x30000, res_centroid_stride=2048)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


ZERO = 65536 * 4 + 65536 * 64   # the zero-at-rest head every op leaves untouched


def _align(n, a=1024):
    return (n + a - 1) // a * a


def test_dgrad_workspace_bytes_without_gpu():
    from vptq_b200 import native
    L = native.lib()
    assert native.OP_GEMM_DGRAD == 4 and native.FLAG_TRANSPOSE == 2 and native.ABI_VERSION == 7
    # Llama-3-8B gate/up: W^T [4096][14336] + staged dY [tokens][14336] behind the head
    for tokens in (1, 3, 8192):
        assert L.vptq_b200_workspace_bytes(ctypes.byref(_desc()), tokens, native.OP_GEMM_DGRAD) == \
            ZERO + 4096 * 14336 * 2 + _align(tokens * 14336 * 2)
    # ragged out_features: the K extent is rounded up to whole 64-element blocks (1004 -> 1024)
    ragged = _desc(in_features=1000, out_features=1004, group_size=1000, index_stride_row=750,
                   index_stride_codebook=126 * 750)
    assert L.vptq_b200_workspace_bytes(ctypes.byref(ragged), 5, native.OP_GEMM_DGRAD) == \
        ZERO + _align(1000 * 1024 * 2) + _align(5 * 1024 * 2)
    # unknown op codes are still refused
    assert L.vptq_b200_workspace_bytes(ctypes.byref(_desc()), 1, 5) == 0
    assert "unknown op" in native.last_error()


def test_transpose_flag_validates_swapped_strides():
    from vptq_b200 import native
    L = native.lib()
    T = native.FLAG_TRANSPOSE
    gemm = L.vptq_b200_quant_gemm
    d = _desc()   # in 4096, out 14336: x = dY [tokens][14336], y = dX [tokens][4096]
    # strides that would be right for the forward call are wrong for the transposed one
    for xs, ys in ((4096, 14336), (14335, 4096), (14336, 4095)):
        assert gemm(ctypes.byref(d), 0x1000, xs, 0x2000, ys, 8, None, 0, T, None) == -1
        assert "transpose" in native.last_error() and "stride" in native.last_error()
    assert gemm(ctypes.byref(d), None, 14336, 0x2000, 4096, 8, None, 0, T, None) == -1
    assert gemm(ctypes.byref(d), 0x1000, 14336, 0x2000, 4096, 0, None, 0, T, None) == -1
    # decode-only descriptor (lists only, no packed words): refused before anything is launched
    dec = _desc(indices=None, lists_stream=0x40000, lists_tab=0x50000, lists_tile_cols=4096)
    assert gemm(ctypes.byref(dec), 0x1000, 14336, 0x2000, 4096, 8, None, 0, T, None) == -2
    assert "decode-only" in native.last_error()
    if not torch.cuda.is_available():
        # well-formed arguments reach the device check, which fails on a host without an H100
        rc = gemm(ctypes.byref(d), 0x1000, 14336, 0x2000, 4096, 8, None, 0, T, None)
        assert rc < 0 and native.last_error()
