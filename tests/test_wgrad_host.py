"""Weight gradients of the quantized linear layer, host-side checks (no GPU needed).

* the fp64 oracle (tests/_wgrad.py) against autograd through the CPU port of the reference's differentiable torch
  path (oracle/torch_port.py) on every golden fixture, from (x, dY) and from a given dL/dW;
* the C interface of include/vptq_b200_grad.h: symbols, struct layout, workspace sizes, argument validation; and
  that the inference ABI of include/vptq_b200.h is unchanged by it.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _util import golden_names, load_golden
from _wgrad import gamma_from_x_dy, grads_from_gamma

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("centroids", "res_centroids", "outlier_centroids", "weight_scale", "weight_bias")


def _port_layer(L):
    """torch_port layer dict with fp64 leaves (requires_grad) for the floating-point tensors."""
    f = lambda a: None if a is None else torch.from_numpy(vo.to_f32(a, L.dtype).astype(np.float64)).requires_grad_()
    u = lambda a: None if a is None else torch.from_numpy(np.asarray(a, dtype=np.uint16).copy()).view(torch.int16)
    return dict(in_features=L.in_features, out_features=L.out_features, vector_len=L.vector_len,
                num_centroids=L.num_centroids, num_res_centroids=L.num_res_centroids, num_codebooks=L.num_codebooks,
                group_size=L.group_size, outlier_size=L.outlier_size if L.enable_outlier else 0,
                outlier_vector_len=L.outlier_vector_len, num_outlier_centroids=L.num_outlier_centroids,
                indices=torch.from_numpy(L.indices.copy()), centroids=f(L.centroids),
                res_centroids=f(L.res_centroids) if L.res_bits else None,
                outlier_indices=u(L.outlier_indices) if L.enable_outlier else None,
                outlier_centroids=f(L.outlier_centroids) if L.enable_outlier else None, perm=u(L.perm),
                weight_scale=f(L.weight_scale), weight_bias=f(L.weight_bias), bias=None)


def _check(d, want, name):
    got = {n: d[n].grad.numpy().reshape(want[n].shape) for n in NAMES if d.get(n) is not None}
    assert sorted(got) == sorted(want), name
    for n in want:
        err = np.abs(got[n] - want[n]).max() / max(np.abs(want[n]).max(), 1e-30)
        assert err <= 1e-5, f"{name} {n}: {err:.3e}"


@pytest.mark.parametrize("name", golden_names())
def test_wgrad_oracle_matches_torch_port_autograd(name):
    """From (x, dY): v4 no-norm no-perm, v6 padding rows, v12, v16, outlier columns, two groups, bf16."""
    import torch_port as tp
    L, x, _ = load_golden(name)
    d = _port_layer(L)
    dy = vo.make_x(x.shape[0], L.out_features, L.dtype, seed=12)
    xt = torch.from_numpy(vo.to_f32(x, L.dtype).astype(np.float64))
    (tp.dequant(d).double() @ xt.T).T.backward(torch.from_numpy(vo.to_f32(dy, L.dtype).astype(np.float64)))
    _check(d, grads_from_gamma(gamma_from_x_dy(x, dy, L), L), name)


@pytest.mark.parametrize("name", golden_names())
def test_dequant_backward_oracle_matches_torch_port_autograd(name):
    import torch_port as tp
    L, _, _ = load_golden(name)
    d = _port_layer(L)
    gamma = np.random.default_rng(5).standard_normal((L.out_features, L.in_features))
    tp.dequant(d).backward(torch.from_numpy(gamma).float())
    _check(d, grads_from_gamma(gamma.astype(np.float32), L), name)


# ---------------------------------------------------------------- C interface
def _grad_header_symbols():
    src = open(os.path.join(ROOT, "include", "vptq_b200_grad.h")).read()
    return sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", src)))


def test_grad_header_symbols_are_exported_and_the_inference_abi_is_unchanged():
    from vptq_b200 import native
    L = native.lib()
    syms = _grad_header_symbols()
    assert syms == sorted(native.GRAD_EXPORTS) and len(syms) == 4
    for s in syms:
        assert hasattr(L, s), s
    assert L.vptq_b200_grad_version() == native.GRAD_VERSION == 1
    main = open(os.path.join(ROOT, "include", "vptq_b200.h")).read()
    main_syms = sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", main)))
    assert len(main_syms) == 15 and sorted(native.EXPORTS) == main_syms and not set(syms) & set(main_syms)
    assert L.vptq_b200_abi_version() == native.ABI_VERSION == 7
    assert "#define VPTQ_B200_ABI_VERSION 7" in main
    assert "vptq_b200_grad.h" in main   # the inference header points to the gradients' header


def test_linear_grads_layout_matches_header():
    from vptq_b200 import native
    src = open(os.path.join(ROOT, "include", "vptq_b200_grad.h")).read()
    body = re.search(r"typedef struct vptq_linear_grads \{(.*?)\} vptq_linear_grads;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"(\w+)\s*;", body)
    assert fields == [f for f, _ in native.LinearGrads._fields_]
    assert ctypes.sizeof(native.LinearGrads) == 8 + 5 * 8
    assert native.GRAD_FIELDS == tuple(f for f, _ in native.LinearGrads._fields_[2:])


def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    base = dict(dtype=0, in_features=4096, out_features=14336, vector_len=8, num_centroids=65536,
                num_res_centroids=256, num_codebooks=1, group_size=4096, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=0x10000, index_stride_codebook=1792 * 3072, index_stride_row=3072,
                centroids=0x20000, centroid_stride=65536 * 8, res_centroids=0x30000, res_centroid_stride=2048,
                weight_scale=0x60000, weight_bias=0x70000)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


ZERO = 65536 * 4 + 65536 * 64   # the zero-at-rest head every op leaves untouched


def _a(n, a):
    return (n + a - 1) // a * a


def test_grad_workspace_bytes_without_gpu():
    from vptq_b200 import native
    L = native.lib()
    ws = lambda d, t, op: L.vptq_b200_grad_workspace_bytes(ctypes.byref(d), t, op)
    I, O = 4096, 14336
    accs = 256 + _a(65536 * 8 * 8, 256) + 256 * 8 * 8 + 0 + 2 * I * 8
    for tokens in (1, 64, 65, 8192):
        tp = _a(tokens, 64)
        head = _a(ZERO + accs + 3 * _a(tokens * 8, 256), 1024)   # fp64 per-row bound sums
        staged = head + O * tp * 2 + I * tp * 2                    # dY^T, x'^T
        # v = 8, one group, no outliers: the fused route never stores G; the generic route adds fp32 G
        assert ws(_desc(), tokens, native.GRAD_OP_WGRAD) == staged, tokens
        assert ws(_desc(), tokens, native.GRAD_OP_WGRAD_GENERIC) == staged + O * I * 4, tokens
    # dequant backward: statistics per output row + the inverse permutation, no staging
    want = _a(ZERO + accs + 3 * _a(O * 8, 256) + _a(I * 2, 256), 1024)
    assert ws(_desc(), 1, native.GRAD_OP_DEQUANT_BACKWARD) == want
    # v = 2 (generic route only), odd in_features: x'^T gets an even row count, G an aligned pitch
    odd = _desc(in_features=1001, out_features=250, vector_len=2, num_centroids=256, num_res_centroids=-1,
                res_centroids=None, group_size=1001, index_stride_row=251, index_stride_codebook=125 * 251,
                centroid_stride=512)
    accs = 256 + _a(256 * 2 * 8, 256) + 0 + 0 + 2 * _a(1001 * 8, 256)
    want = _a(ZERO + accs + 3 * 256, 1024) + _a(250 * 64 * 2, 1024) + _a(1002 * 64 * 2, 1024) + \
        _a(250 * 1004 * 4, 1024)
    assert ws(odd, 5, native.GRAD_OP_WGRAD) == want == ws(odd, 5, native.GRAD_OP_WGRAD_GENERIC)
    # unknown op codes are refused; the inference workspace query still refuses op 5
    assert ws(_desc(), 1, 3) == 0 and "unknown op" in native.last_error()
    assert L.vptq_b200_workspace_bytes(ctypes.byref(_desc()), 1, 5) == 0
    assert "unknown op" in native.last_error()


def _grads(**ptrs):
    from vptq_b200 import native
    g = native.LinearGrads()
    g.struct_size = ctypes.sizeof(native.LinearGrads)
    for k, v in ptrs.items():
        setattr(g, k, v)
    return g


def test_wgrad_validates_arguments():
    from vptq_b200 import native
    L = native.lib()
    wg, db = L.vptq_b200_quant_gemm_wgrad, L.vptq_b200_dequant_backward
    d, g = _desc(), _grads(centroids=0x80000)
    # x = [tokens][>= 4096], dy = [tokens][>= 14336]
    for xs, ys in ((4095, 14336), (4096, 14335), (14336, 4096)):
        assert wg(ctypes.byref(d), 0x1000, xs, 0x2000, ys, 8, ctypes.byref(g), None, 0, 0, None) == -1
        assert "stride" in native.last_error()
    assert wg(ctypes.byref(d), None, 4096, 0x2000, 14336, 8, ctypes.byref(g), None, 0, 0, None) == -1
    assert wg(ctypes.byref(d), 0x1000, 4096, None, 14336, 8, ctypes.byref(g), None, 0, 0, None) == -1
    assert wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 0, ctypes.byref(g), None, 0, 0, None) == -1
    assert wg(ctypes.byref(d), 0x1001, 4096, 0x2000, 14336, 8, ctypes.byref(g), None, 0, 0, None) == -1
    # the grads struct: NULL, wrong size, unknown flags, a gradient for a tensor the layer lacks, odd address
    assert wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, None, None, 0, 0, None) == -1
    bad = _grads(centroids=0x80000)
    bad.struct_size = 8
    assert wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(bad), None, 0, 0, None) == -1
    assert wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(g), None, 0, 2, None) == -1
    assert "flags" in native.last_error()
    assert db(ctypes.byref(d), 0x1000, 4096, ctypes.byref(g), None, 0, native.GRAD_FLAG_GENERIC, None) == -1
    assert "flags" in native.last_error()
    for over in (dict(outlier_centroids=0x80000), dict(centroids=0x80001)):
        gg = _grads(**over)
        assert wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(gg), None, 0, 0, None) == -1
    nonorm = _desc(weight_scale=None, weight_bias=None)
    gs = _grads(weight_scale=0x80000)
    assert wg(ctypes.byref(nonorm), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(gs), None, 0, 0, None) == -1
    assert "does not have" in native.last_error()
    # dequant backward: dw [14336][>= 4096]
    assert db(ctypes.byref(d), 0x1000, 4095, ctypes.byref(g), None, 0, 0, None) == -1
    assert db(ctypes.byref(d), None, 4096, ctypes.byref(g), None, 0, 0, None) == -1
    # decode-only descriptor (lists only, no packed words): refused before anything is launched
    dec = _desc(indices=None, lists_stream=0x40000, lists_tab=0x50000, lists_tile_cols=4096)
    assert wg(ctypes.byref(dec), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(g), None, 0, 0, None) == -2
    assert "decode-only" in native.last_error()
    assert db(ctypes.byref(dec), 0x1000, 4096, ctypes.byref(g), None, 0, 0, None) == -2
    assert "decode-only" in native.last_error()
    if not torch.cuda.is_available():
        # well-formed arguments (either route) reach the device check, which fails on a host without an H100
        for flags in (0, native.GRAD_FLAG_GENERIC):
            rc = wg(ctypes.byref(d), 0x1000, 4096, 0x2000, 14336, 8, ctypes.byref(g), None, 0, flags, None)
            assert rc < 0 and "flags" not in native.last_error()


def test_python_binding_checks_before_the_library():
    from vptq_b200 import native
    with pytest.raises(RuntimeError, match="unknown gradient outputs"):
        native.make_grads({"bias": torch.zeros(2)})
    with pytest.raises(RuntimeError, match="CUDA"):
        native.make_grads({"centroids": torch.zeros(2)})


def test_set_quant_grad_without_gpu():
    import torch.nn as nn
    import vptq_b200
    from vptq_b200 import VQuantLinear
    mk = lambda: VQuantLinear(64, 32, vector_lens=[-1, 8], num_centroids=[-1, 256], num_res_centroids=[-1, -1],
                              group_num=1, group_size=64, outlier_size=0, indices_as_float=False, enable_norm=True,
                              enable_perm=True, is_indice_packed=True, dtype=torch.float16, enable_proxy_error=False)
    model = nn.Sequential(mk(), nn.ReLU(), mk())
    assert not model[0]._quant_grad
    assert vptq_b200.set_quant_grad(model, True) == 2 and model[0]._quant_grad and model[2]._quant_grad
    assert vptq_b200.set_quant_grad(model, False) == 2 and not model[2]._quant_grad
    m = model[2]
    m._drop_packed = True
    m.indices.data = torch.empty(0, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="decode-only"):
        m.set_quant_grad(True)
    # model level: all or nothing -- the first layer is not left opted in when the second refuses
    with pytest.raises(RuntimeError, match="decode-only"):
        vptq_b200.set_quant_grad(model, True)
    assert not model[0]._quant_grad and not model[2]._quant_grad
    m.set_quant_grad(False)
    # an opted-in module refuses to become decode-only
    model[0].set_quant_grad(True)
    with pytest.raises(RuntimeError, match="set_quant_grad"):
        model[0].prepare(drop_packed=True)
