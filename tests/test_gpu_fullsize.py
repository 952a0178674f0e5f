"""Dense random inputs at full Llama-3-8B layer sizes against an fp64 reference computed on the GPU
(y* = x.double() @ W64^T + bias, W64 = the oracle's dequant in float64), at the project's bar
max|y - y*| / max|y*| <= 1e-3 (fp16), 4e-3 (bf16).  Covers every route at the size where the persistent tile walk
runs many tiles per CTA and the list kernel cuts its rows over all SMs."""
import pytest
import torch

import vptq_oracle as vo
from _probe import fp64_bias, fp64_weight, launched_kernels, ran
from _util import TOL

pytestmark = pytest.mark.gpu

LLAMA = {"4096x4096": (4096, 4096), "4096x14336": (4096, 14336), "14336x4096": (14336, 4096)}


def _layer(i, o, dtype="fp16", seed=4242, bias=False):
    L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      dtype=dtype, seed=seed, bias=bias)
    L.meta = {}
    return L


def _module(L, lists=True):
    from _gpu import make_module
    m = make_module(L)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("VPTQ_B200_LISTS", "1" if lists else "0")
        m.prepare()
    return m


def _err(y, ref):
    return float((y.double() - ref).abs().max() / ref.abs().max())


def _x(tokens, i, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(tokens, i, device="cuda", generator=g).to(dt)


@pytest.mark.parametrize("shape", list(LLAMA))
def test_decode_full_size_vs_fp64(shape):
    i, o = LLAMA[shape]
    L = _layer(i, o, bias=True)
    m = _module(L)
    W, b = fp64_weight(L), fp64_bias(L)
    x = _x(2, i, torch.float16, 1)
    names = launched_kernels(lambda: m(x[:1]))
    assert ran(names, "gemv_lists_kernel"), names
    assert ran(launched_kernels(lambda: m(x)), "gemv_kernel")
    for tokens in (1, 2):
        ref = x[:tokens].double() @ W.T + b
        assert _err(m(x[:tokens]), ref) <= TOL["fp16"], (shape, tokens)


@pytest.mark.parametrize("group", ["qkv", "gate_up"])
def test_fused_decode_full_size_vs_fp64(group):
    from vptq_b200 import native
    shapes = [(4096, 4096), (4096, 1024), (4096, 1024)] if group == "qkv" else [(4096, 14336), (4096, 14336)]
    Ls = [_layer(i, o, seed=300 + k) for k, (i, o) in enumerate(shapes)]
    ms = [_module(L) for L in Ls]
    x = _x(1, 4096, torch.float16, 2)
    ys = [torch.full((1, L.out_features), float("nan"), dtype=torch.float16, device="cuda") for L in Ls]
    fused = native.FusedGemv([m._desc_cache[0] for m in ms], ys)
    names = launched_kernels(lambda: fused(x))
    assert not fused.separate and sum(ran([n], "gemv_lists_kernel") for n in names) == 1, names
    for L, y in zip(Ls, ys):
        assert _err(y, x.double() @ fp64_weight(L).T) <= TOL["fp16"], (group, L.out_features)


@pytest.mark.parametrize("route", ["direct", "prep"])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", list(LLAMA))
def test_prefill_8192_tokens_vs_fp64(shape, dtype, route, monkeypatch):
    i, o = LLAMA[shape]
    L = _layer(i, o, dtype=dtype, bias=True)
    m = _module(L, lists=False)
    if route == "prep":
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    x = _x(8192, i, m.centroids.weight.dtype, 3)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "gemm_tn_wgmma") and ran(names, "prefill_prep_x") == (route == "prep"), names
    y = m(x)
    ref = x.double() @ fp64_weight(L).T + fp64_bias(L)
    assert _err(y, ref) <= TOL[dtype]


@pytest.mark.parametrize("shape", list(LLAMA))
def test_dgrad_2048_tokens_vs_fp64(shape):
    from vptq_b200 import native
    i, o = LLAMA[shape]
    L = _layer(i, o)
    m = _module(L, lists=False)
    dy = _x(2048, o, torch.float16, 4)
    dx = torch.empty(2048, i, dtype=torch.float16, device="cuda")
    native.quant_gemm_dgrad(m._desc_cache[0], dy, dx)
    assert _err(dx, dy.double() @ fp64_weight(L)) <= TOL["fp16"]
