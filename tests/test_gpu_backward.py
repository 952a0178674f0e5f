"""GPU checks of the layer's backward: dX = dY W through the transposed dequant + wgmma GEMM
(vptq_b200_quant_gemm with VPTQ_FLAG_TRANSPOSE), reached through VQuantLinear / vptq.ops.quant_gemm autograd.

Bars: the forward's, max|dX - dX*| / max|dX*| <= 1e-3 (fp16), 4e-3 (bf16), dX* = dY @ W in fp64 on the identical
16-bit tensors (tests/_dgrad.py).  With dY = identity the GEMM returns W itself, which checks the transposed
dequant bit for bit against `dequant()`.
"""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _dgrad import quant_gemm_dgrad
from _util import TOL, golden_names, load_golden, parity_error

pytestmark = pytest.mark.gpu


def _input_grad(m, x, dy):
    x = x.detach().clone().requires_grad_()
    y = m(x)
    y.backward(dy)
    torch.cuda.synchronize()
    return x.grad


def _identity_grad(m, L):
    """dX for dY = identity (tokens = out_features): the weight W[o][f] itself."""
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    x = torch.zeros(L.out_features, L.in_features, dtype=dt, device="cuda")
    return _input_grad(m, x, torch.eye(L.out_features, dtype=dt, device="cuda"))


# ---------------------------------------------------------------- exact transpose
FAST = {
    "k65536_r256_4096_fp16": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256),
    "k65536_r256_4096_bf16": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256,
                                  dtype="bf16"),
    "ragged_1000x1004": dict(in_features=1000, out_features=1004, num_centroids=4096, num_res_centroids=32),
}


@pytest.mark.parametrize("name", sorted(FAST))
def test_identity_dy_returns_the_dequantised_weight_fast_path(name):
    from _gpu import make_module
    L = vo.make_layer(vector_len=8, seed=21, **FAST[name])
    m = make_module(L)
    gx = _identity_grad(m, L)
    W = m.dequant()
    assert torch.isfinite(gx).all()
    assert torch.equal(gx, W), name   # every value identical (+0 and -0 count as equal)


@pytest.mark.parametrize("name", golden_names())
def test_identity_dy_returns_the_dequantised_weight_golden_configs(name):
    """v4 no-norm no-perm, v6 with padding rows, v12, v16, outlier columns, 2 groups, bf16: the generic path."""
    from _gpu import make_module
    L, _, _ = load_golden(name)
    m = make_module(L)
    gx = _identity_grad(m, L)
    assert torch.isfinite(gx).all()
    assert torch.equal(gx, m.dequant()), name


# ---------------------------------------------------------------- accuracy against the oracle
ACC = {
    "k65536_r256": dict(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256),
    "k65536_r256_bf16": dict(in_features=1024, out_features=512, vector_len=8, num_centroids=65536,
                             num_res_centroids=256, dtype="bf16"),
    "ragged_1000x1004": dict(in_features=1000, out_features=1004, vector_len=8, num_centroids=4096, num_res_centroids=32),
    "wide_9000x72": dict(in_features=9000, out_features=72, vector_len=8, num_centroids=65536, num_res_centroids=256),
    "outliers_bias": dict(in_features=1024 + 128, out_features=512, vector_len=8, num_centroids=4096,
                          num_res_centroids=256, outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096,
                          bias=True),
    "v6_pad": dict(in_features=512, out_features=250, vector_len=6, num_centroids=4096),
}


@pytest.mark.parametrize("tokens", [1, 2, 3, 64, 300, 2048])
@pytest.mark.parametrize("name", sorted(ACC))
def test_dgrad_vs_oracle(name, tokens):
    from _gpu import from_t, make_module, x_to_t
    L = vo.make_layer(seed=23, **ACC[name])
    m = make_module(L)
    x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=1), L)
    dy_np = vo.make_x(tokens, L.out_features, L.dtype, seed=2)
    gx = from_t(_input_grad(m, x, x_to_t(dy_np, L)))
    assert np.isfinite(gx).all()
    err = parity_error(gx, quant_gemm_dgrad(dy_np, L))
    assert err <= TOL[L.dtype], f"{name} tokens={tokens}: {err:.3e}"


# ---------------------------------------------------------------- module level
@pytest.mark.parametrize("shape", [(5,), (2, 150)])
@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_module_backward_matches_dense_autograd(shape, dtype):
    """2-D and 3-D inputs; y.sum() hands the backward a zero-stride dY."""
    from _gpu import make_module, x_to_t
    L = vo.make_layer(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      bias=True, dtype=dtype, seed=25)
    m = make_module(L)
    tokens = int(np.prod(shape))
    x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=4), L).reshape(*shape, L.in_features).requires_grad_()
    m(x).sum().backward()
    torch.cuda.synchronize()
    xr = x.detach().float().requires_grad_()
    br = m.bias.detach().float().requires_grad_()
    torch.nn.functional.linear(xr, m.dequant().float(), br).sum().backward()
    assert x.grad.shape == x.shape and x.grad.dtype == x.dtype
    assert parity_error(x.grad.float().cpu().numpy(), xr.grad.cpu().numpy()) <= TOL[dtype]
    assert m.bias.grad is not None and m.bias.grad.dtype == m.bias.dtype
    assert parity_error(m.bias.grad.float().cpu().numpy(), br.grad.cpu().numpy()) <= TOL[dtype]
    # no gradient for the quantised weight's own tensors
    assert m.centroids.weight.grad is None and m.weight_scale.grad is None


def test_lora_style_chain_gets_the_base_layers_share_of_the_gradient():
    """y = base(x) + B(A(x)) on two stacked layers: every adapter gradient needs dL/dx of the layer above it."""
    from _gpu import make_module, x_to_t
    L1 = vo.make_layer(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                       seed=27)
    L2 = vo.make_layer(in_features=512, out_features=768, vector_len=8, num_centroids=4096, num_res_centroids=256,
                       seed=28)
    m1, m2 = make_module(L1), make_module(L2)
    g = torch.Generator(device="cuda").manual_seed(3)
    r = 8
    A1 = (torch.randn(r, 1024, device="cuda", generator=g) / 32).half()
    B1 = (torch.randn(512, r, device="cuda", generator=g) / 4).half()
    A2 = (torch.randn(r, 512, device="cuda", generator=g) / 24).half()
    B2 = (torch.randn(768, r, device="cuda", generator=g) / 4).half()
    x = x_to_t(vo.make_x(300, 1024, "fp16", seed=6), L1)
    w_out = torch.randn(300, 768, device="cuda", generator=g)

    def run(base1, base2, params, xx):
        a1, b1, a2, b2 = params
        h = base1(xx) + (xx @ a1.t()) @ b1.t()
        y = base2(h) + (h @ a2.t()) @ b2.t()
        (y.float() * w_out).sum().backward()
        return [p.grad.float() for p in params]

    ours = run(m1, m2, [p.clone().requires_grad_() for p in (A1, B1, A2, B2)], x)
    W1, W2 = m1.dequant().float(), m2.dequant().float()
    ref = run(lambda t: t @ W1.t(), lambda t: t @ W2.t(), [p.float().requires_grad_() for p in (A1, B1, A2, B2)],
              x.float())
    for name, a, b in zip(("A1", "B1", "A2", "B2"), ours, ref):
        err = float((a - b).abs().max() / b.abs().max())
        assert err <= 1e-2, f"{name}: {err:.3e}"   # fp16 activations in the chain vs fp32 throughout


# ---------------------------------------------------------------- forward unchanged
@pytest.mark.parametrize("tokens", [1, 2, 3, 300])
def test_forward_under_grad_mode_is_bit_identical(tokens):
    from _gpu import make_module, x_to_t
    L = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      bias=True, seed=29)
    m = make_module(L)
    m.prepare()
    x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=7), L)
    with torch.no_grad():
        y0 = m(x)
    y1 = m(x.clone().requires_grad_())
    assert y1.grad_fn is not None
    assert torch.equal(y0, y1.detach())


def test_fused_group_under_grad_mode_equals_unfused():
    import torch.nn as nn
    import vptq_b200
    from _gpu import make_module, x_to_t
    Ls = [vo.make_layer(in_features=1024, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                        seed=30 + k) for k, o in enumerate((1024, 256, 256))]
    parent = nn.Module()
    parent.q_proj, parent.k_proj, parent.v_proj = (make_module(L) for L in Ls)
    x = x_to_t(vo.make_x(1, 1024, "fp16", seed=8), Ls[0])
    with torch.no_grad():
        want = [parent.q_proj(x), parent.k_proj(x), parent.v_proj(x)]
    assert len(vptq_b200.fuse(parent)) == 1
    xg = x.clone().requires_grad_()
    got = [parent.q_proj(xg), parent.k_proj(xg), parent.v_proj(xg)]
    for a, b in zip(got, want):
        assert a.grad_fn is not None and torch.equal(a.detach(), b)
    sum(t.float().sum() for t in got).backward()
    assert xg.grad is not None and torch.isfinite(xg.grad).all()
    with torch.no_grad():   # inference on the fused model is unchanged
        for mod, b in zip((parent.q_proj, parent.k_proj, parent.v_proj), want):
            assert torch.equal(mod(x), b)


# ---------------------------------------------------------------- workspace sharing, CUDA graphs, decode-only
def test_transpose_calls_leave_the_list_gemv_workspace_clean():
    from _gpu import make_module, x_to_t
    from vptq_b200 import native
    L = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      seed=32)
    m = make_module(L)
    m.prepare()
    desc = m._desc_cache[0]
    assert desc.lists_stream                      # single-token calls run the list kernel
    x = x_to_t(vo.make_x(1, 2048, "fp16", seed=9), L)
    with torch.no_grad():
        y0 = m(x).clone()
    dy = x_to_t(vo.make_x(200, 1024, "fp16", seed=10), L)
    dx = torch.empty(200, 2048, dtype=torch.float16, device="cuda")
    for _ in range(5):
        native.quant_gemm_dgrad(desc, dy, dx)
        with torch.no_grad():
            assert torch.equal(m(x), y0)
    torch.cuda.synchronize()
    assert parity_error(dx.float().cpu().numpy(), quant_gemm_dgrad(vo.make_x(200, 1024, "fp16", seed=10), L)) <= 1e-3


def test_transposed_call_replays_bit_identically_in_a_cuda_graph():
    from _gpu import make_module, x_to_t
    from vptq_b200 import native
    L = vo.make_layer(in_features=1024, out_features=1000, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      seed=33)
    m = make_module(L)
    m.prepare()
    desc = m._desc_cache[0]
    dy = x_to_t(vo.make_x(130, 1000, "fp16", seed=11), L)   # 1000 % 64 != 0: the staged-dY route
    dx = torch.empty(130, 1024, dtype=torch.float16, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        native.quant_gemm_dgrad(desc, dy, dx)    # warm-up outside capture (workspace allocation)
        torch.cuda.synchronize()
        first = dx.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            native.quant_gemm_dgrad(desc, dy, dx)
    for _ in range(3):
        dx.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(dx, first)
    assert parity_error(first.float().cpu().numpy(), quant_gemm_dgrad(vo.make_x(130, 1000, "fp16", seed=11), L)) <= 1e-3


def test_decode_only_module_forward_works_backward_raises():
    from _gpu import make_module, x_to_t
    L = vo.make_layer(in_features=2048, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      seed=34)
    m = make_module(L)
    x = x_to_t(vo.make_x(1, 2048, "fp16", seed=12), L)
    with torch.no_grad():
        y0 = m(x)
    m.prepare(drop_packed=True)
    xg = x.clone().requires_grad_()
    y = m(xg)
    assert torch.equal(y.detach(), y0)
    with pytest.raises(RuntimeError, match="decode-only"):
        y.sum().backward()


def test_in_place_weight_update_between_forward_and_backward_is_refused():
    from _gpu import make_module, x_to_t
    L = vo.make_layer(in_features=512, out_features=256, vector_len=8, num_centroids=4096, seed=35)
    m = make_module(L)
    y = m(x_to_t(vo.make_x(4, 512, "fp16", seed=13), L).requires_grad_())
    with torch.no_grad():
        m.centroids.weight.mul_(2)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()
