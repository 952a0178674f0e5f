"""GPU checks of the weight gradients (include/vptq_b200_grad.h): codebooks, weight_scale and weight_bias of
VQuantLinear after `set_quant_grad(True)`, through `forward` (vptq_b200_quant_gemm_wgrad: G = dY^T x by the wgmma
GEMM, reduced in 64-bit fixed point) and through `dequant()` (vptq_b200_dequant_backward).

Bars: exact values for one-hot probes; otherwise parity_error <= TOL[dtype] per gradient against the fp64 oracle
(tests/_wgrad.py, or the same formulas in fp64 on the GPU for the Llama shapes).  Every test asserts which kernels
ran.
"""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _probe import launched_kernels, ran
from _util import TOL, golden_names, load_golden, parity_error
from _wgrad import grads_from_gamma, quant_gemm_wgrad

pytestmark = pytest.mark.gpu

WGRAD_KERNELS = ("wg_row_stats", "wg_transpose", "gemm_tn_wgmma", "wg_units", "wg_finish")
DQB_KERNELS = ("wg_row_stats", "wg_units", "wg_scatter", "wg_finish")


def _fused(L):
    """The fused route (GEMM epilogue, no scatter kernel) covers v = 8, one group, no outliers, Kr <= 256."""
    return L.vector_len == 8 and L.num_codebooks == 1 and not L.enable_outlier and L.num_res_centroids <= 256


def _generic_grads(m, x, dy):
    """The same gradients through the generic route (G in the workspace + scatter kernel), forced by the flag."""
    from vptq_b200 import native
    desc = m._desc_cache[0]
    outs = {n: torch.empty_like(t) for n, t in _params(m).items()}
    native.quant_gemm_wgrad(desc, x, dy, outs, flags=native.GRAD_FLAG_GENERIC)
    torch.cuda.synchronize()
    return outs


def _params(m):
    p = {"centroids": m.centroids.weight}
    if m.res_centroids is not None:
        p["res_centroids"] = m.res_centroids.weight
    if m.enable_outlier:
        p["outlier_centroids"] = m.outlier_centroids.weight
    if m.weight_scale is not None:
        p["weight_scale"], p["weight_bias"] = m.weight_scale, m.weight_bias
    return p


def _module(L):
    from _gpu import make_module
    m = make_module(L)
    m.set_quant_grad(True)
    for t in _params(m).values():
        t.requires_grad_(True)
    return m


def _grads(m):
    return {n: (None if t.grad is None else t.grad.detach().clone()) for n, t in _params(m).items()}


def _run_wgrad(m, x, dy):
    m.zero_grad(set_to_none=True)
    m(x).backward(dy)
    torch.cuda.synchronize()
    return _grads(m)


def _run_dequant_backward(m, gamma):
    m.zero_grad(set_to_none=True)
    m.dequant().backward(gamma)
    torch.cuda.synchronize()
    return _grads(m)


def _np(g):
    return g.detach().float().cpu().numpy()


def _check_parity(got, want, tol, what):
    assert sorted(k for k, v in got.items() if v is not None) == sorted(want), what
    for n, w in want.items():
        g = got[n]
        assert torch.isfinite(g).all(), f"{what} {n}"
        err = parity_error(_np(g).reshape(w.shape), w)
        assert err <= tol, f"{what} {n}: {err:.3e}"


# ---------------------------------------------------------------- exact probes
PROBE = {
    "v8_pad_perm_norm": dict(in_features=1024, out_features=516, vector_len=8, num_centroids=4096,
                             num_res_centroids=256),
    "v8_bf16": dict(in_features=512, out_features=256, vector_len=8, num_centroids=65536, num_res_centroids=256,
                    dtype="bf16"),
    "v6_pad_nonorm_noperm": dict(in_features=512, out_features=250, vector_len=6, num_centroids=4096,
                                 enable_norm=False, enable_perm=False),
    "outliers": dict(in_features=1024 + 128, out_features=510, vector_len=8, num_centroids=4096,
                     num_res_centroids=256, outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096),
    "two_groups_v4": dict(in_features=1024, out_features=258, vector_len=4, num_centroids=4096, num_res_centroids=16,
                          num_codebooks=2),
}


def _probe_points(L):
    """(o, f) pairs: first / last index rows, next to the padding rows, both sides of a group boundary, outlier
    columns, permuted features."""
    O, I, v = L.out_features, L.in_features, L.vector_len
    S = L.outlier_size if L.enable_outlier else 0
    cols = [0, I - 1, S, S + L.group_size - 1, min(S + L.group_size, I - 1)] + ([S - 1, S // 2] if S else [])
    rows = [0, O - 1, (O // v) * v - 1, O // 2, v, 1, O - 2]
    perm = None if L.perm is None else np.asarray(L.perm).astype(np.int64)
    return [(rows[i % len(rows)], int(perm[c]) if perm is not None else c) for i, c in enumerate(cols)]


def _expected_probe(L, o, f):
    gamma = np.zeros((L.out_features, L.in_features))
    gamma[o, f] = 1.0
    return {n: vo.round_to(w.astype(np.float32), L.dtype) for n, w in grads_from_gamma(gamma, L).items()}


def _assert_exact(got, want, what):
    assert sorted(k for k, v in got.items() if v is not None) == sorted(want), what
    for n, w in want.items():
        g = _np(got[n]).reshape(w.shape)
        bad = np.argwhere(g != w)
        assert bad.size == 0, f"{what} {n}: {len(bad)} elements differ, first {bad[:3].tolist()}"
        assert np.count_nonzero(g) <= 1, f"{what} {n}"   # one vector element (or one feature), the rest exactly 0


@pytest.mark.parametrize("name", sorted(PROBE))
def test_one_hot_probes_are_exact_on_both_entries(name):
    L = vo.make_layer(seed=41, **PROBE[name])
    m = _module(L)
    dt = m.centroids.weight.dtype
    for k, (o, f) in enumerate(_probe_points(L)):
        want = _expected_probe(L, o, f)
        # dequant() backward with G = one-hot at (o, f)
        gamma = torch.zeros(L.out_features, L.in_features, dtype=dt, device="cuda")
        gamma[o, f] = 1
        _assert_exact(_run_dequant_backward(m, gamma), want, f"{name} dequant (o={o}, f={f})")
        # quant_gemm with x = e_f, dY = e_o, one token (x does not require grad)
        x = torch.zeros(1, L.in_features, dtype=dt, device="cuda")
        x[0, f] = 1
        dy = torch.zeros(1, L.out_features, dtype=dt, device="cuda")
        dy[0, o] = 1
        if k == 0:
            names = launched_kernels(lambda: _run_wgrad(m, x, dy))
            assert all(ran(names, kn) for kn in WGRAD_KERNELS), names
            assert ran(names, "wg_scatter") != _fused(L), names    # the fused route has no scatter kernel
            names = launched_kernels(lambda: _run_dequant_backward(m, gamma))
            assert all(ran(names, kn) for kn in DQB_KERNELS) and not ran(names, "gemm_tn_wgmma"), names
        _assert_exact(_run_wgrad(m, x, dy), want, f"{name} wgrad (o={o}, f={f})")
        if _fused(L):
            if k == 0:
                names = launched_kernels(lambda: _generic_grads(m, x, dy))
                assert ran(names, "wg_scatter") and ran(names, "gemm_tn_wgmma"), names
            _assert_exact(_generic_grads(m, x, dy), want, f"{name} wgrad, generic route (o={o}, f={f})")


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
def test_wgrad_vs_oracle(name, tokens):
    from _gpu import x_to_t
    L = vo.make_layer(seed=43, **ACC[name])
    m = _module(L)
    x_np = vo.make_x(tokens, L.in_features, L.dtype, seed=1)
    dy_np = vo.make_x(tokens, L.out_features, L.dtype, seed=2)
    got = _run_wgrad(m, x_to_t(x_np, L), x_to_t(dy_np, L))
    for n, g in got.items():
        assert g.dtype == _params(m)[n].dtype and g.shape == _params(m)[n].shape
    _check_parity(got, quant_gemm_wgrad(x_np, dy_np, L), TOL[L.dtype], f"{name} tokens={tokens}")


@pytest.mark.parametrize("name", golden_names())
def test_golden_configs_both_entries(name):
    from _gpu import x_to_t
    L, x_np, _ = load_golden(name)
    m = _module(L)
    dy_np = vo.make_x(x_np.shape[0], L.out_features, L.dtype, seed=3)
    _check_parity(_run_wgrad(m, x_to_t(x_np, L), x_to_t(dy_np, L)), quant_gemm_wgrad(x_np, dy_np, L),
                  TOL[L.dtype], f"{name} wgrad")
    gamma_np = vo.make_x(L.out_features, L.in_features, L.dtype, seed=4)
    _check_parity(_run_dequant_backward(m, x_to_t(gamma_np, L)), grads_from_gamma(vo.to_f32(gamma_np, L.dtype), L),
                  TOL[L.dtype], f"{name} dequant backward")


@pytest.mark.parametrize("name", ["k65536_r256", "k65536_r256_bf16", "outliers_bias", "v6_pad"])
def test_dequant_backward_random_gamma(name):
    from _gpu import x_to_t
    L = vo.make_layer(seed=44, **ACC[name])
    m = _module(L)
    gamma_np = vo.make_x(L.out_features, L.in_features, L.dtype, seed=5)
    _check_parity(_run_dequant_backward(m, x_to_t(gamma_np, L)), grads_from_gamma(vo.to_f32(gamma_np, L.dtype), L),
                  TOL[L.dtype], name)


def _gpu_reference(L, m, x, dy):
    """The oracle's formulas in fp64 on the GPU (one codebook group, no outliers): full Llama shapes."""
    O, I, v, K, Kr = L.out_features, L.in_features, L.vector_len, L.num_centroids, L.num_res_centroids
    G = dy.double().t() @ x.double()                                       # [O, I]
    perm = torch.from_numpy(np.asarray(L.perm).astype(np.int64)).cuda()
    s = m.weight_scale.detach().double()
    idx = torch.from_numpy(L.meta["idx"][0]).cuda()                        # [Ro, I] quantised order
    ridx = torch.from_numpy(L.meta["ridx"][0]).cuda()
    Ro = idx.shape[0]
    sg = torch.zeros(Ro * v, I, dtype=torch.float64, device="cuda")
    sg[:O] = G[:, perm] * s[perm]
    t = sg.view(Ro, v, I).permute(0, 2, 1).reshape(-1, v)
    dC = torch.zeros(K, v, dtype=torch.float64, device="cuda").index_add_(0, idx.reshape(-1), t)
    dR = torch.zeros(Kr, v, dtype=torch.float64, device="cuda").index_add_(0, ridx.reshape(-1), t)
    del t, sg
    C = m.centroids.weight.detach().double().view(K, v)
    R = m.res_centroids.weight.detach().double().view(Kr, v)
    wq = (C[idx] + R[ridx]).float().double().permute(0, 2, 1).reshape(Ro * v, I)[:O]   # fp32 sum, quantised order
    wq_orig = torch.empty_like(wq)
    wq_orig[:, perm] = wq
    return {"centroids": dC.reshape(1, -1), "res_centroids": dR.reshape(1, -1),
            "weight_scale": (G * wq_orig).sum(0), "weight_bias": G.sum(0)}


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336), (14336, 4096)])
def test_llama_shapes_2048_tokens_vs_fp64_on_gpu(shape, dtype):
    from _gpu import x_to_t
    I, O = shape
    L = vo.make_layer(in_features=I, out_features=O, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      dtype=dtype, seed=45)
    m = _module(L)
    x = x_to_t(vo.make_x(2048, I, dtype, seed=6), L)
    dy = x_to_t(vo.make_x(2048, O, dtype, seed=7), L)
    got = _run_wgrad(m, x, dy)
    # the fused route (GEMM epilogue) and the generic route (G in the workspace + scatter) agree bit for bit
    gen = _generic_grads(m, x, dy)
    for n in got:
        assert torch.equal(got[n], gen[n]), f"{shape} {dtype} {n}: fused != generic"
    want = _gpu_reference(L, m, x, dy)
    for n, w in want.items():
        g = got[n].double().reshape(w.shape)
        assert torch.isfinite(g).all()
        err = float((g - w).abs().max() / w.abs().max())
        assert err <= TOL[dtype], f"{shape} {dtype} {n}: {err:.3e}"


# ---------------------------------------------------------------- determinism
DET = dict(in_features=4096, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256)


def test_two_eager_calls_are_bit_identical():
    from _gpu import x_to_t
    L = vo.make_layer(seed=46, **DET)
    m = _module(L)
    x = x_to_t(vo.make_x(777, L.in_features, "fp16", seed=8), L)
    dy = x_to_t(vo.make_x(777, L.out_features, "fp16", seed=9), L)
    a = _run_wgrad(m, x, dy)
    b = _run_wgrad(m, x, dy)
    gamma = x_to_t(vo.make_x(L.out_features, L.in_features, "fp16", seed=10), L)
    c, d = _run_dequant_backward(m, gamma), _run_dequant_backward(m, gamma)
    for n in a:
        assert torch.equal(a[n], b[n]) and torch.equal(c[n], d[n]), n


def test_cuda_graph_replays_bit_identically():
    from _gpu import make_module, x_to_t
    from vptq_b200 import native
    L = vo.make_layer(seed=47, **DET)
    m = make_module(L)
    m.prepare()
    desc = m._desc_cache[0]
    x = x_to_t(vo.make_x(300, L.in_features, "fp16", seed=11), L)
    dy = x_to_t(vo.make_x(300, L.out_features, "fp16", seed=12), L)
    outs = {n: torch.empty_like(t) for n, t in _params(m).items()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        native.quant_gemm_wgrad(desc, x, dy, outs)      # warm-up outside capture (workspace allocation)
        torch.cuda.synchronize()
        first = {n: t.clone() for n, t in outs.items()}
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            native.quant_gemm_wgrad(desc, x, dy, outs)
    for _ in range(3):
        for t in outs.values():
            t.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        for n in outs:
            assert torch.equal(outs[n], first[n]), n
    _check_parity(first, quant_gemm_wgrad(vo.make_x(300, L.in_features, "fp16", seed=11),
                                          vo.make_x(300, L.out_features, "fp16", seed=12), L), TOL["fp16"], "graph")


def test_wgrad_calls_leave_the_list_gemv_workspace_clean():
    from _gpu import make_module, x_to_t
    from vptq_b200 import native
    L = vo.make_layer(seed=48, **DET)
    m = make_module(L)
    m.prepare()
    desc = m._desc_cache[0]
    assert desc.lists_stream                      # single-token calls run the list kernel
    x1 = x_to_t(vo.make_x(1, L.in_features, "fp16", seed=13), L)
    with torch.no_grad():
        y0 = m(x1).clone()
    x = x_to_t(vo.make_x(200, L.in_features, "fp16", seed=14), L)
    dy = x_to_t(vo.make_x(200, L.out_features, "fp16", seed=15), L)
    outs = {n: torch.empty_like(t) for n, t in _params(m).items()}
    for _ in range(3):
        native.quant_gemm_wgrad(desc, x, dy, outs)
        native.dequant_backward(desc, dy.new_ones(L.out_features, L.in_features), outs)
        with torch.no_grad():
            assert torch.equal(m(x1), y0)


# ---------------------------------------------------------------- module level
MOD = dict(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256, bias=True)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_module_fills_requested_grads_without_x_grad(dtype):
    from _gpu import x_to_t
    L = vo.make_layer(seed=49, dtype=dtype, **MOD)
    m = _module(L)
    x = x_to_t(vo.make_x(5, 1024, dtype, seed=16), L)
    dy = x_to_t(vo.make_x(5, 512, dtype, seed=17), L)
    y = m(x)
    assert not x.requires_grad and y.grad_fn is not None
    y.backward(dy)
    for n, t in _params(m).items():
        assert t.grad is not None and t.grad.dtype == t.dtype and t.grad.shape == t.shape, n
    assert m.bias.grad is not None and x.grad is None
    _check_parity(_grads(m), quant_gemm_wgrad(vo.make_x(5, 1024, dtype, seed=16), vo.make_x(5, 512, dtype, seed=17), L),
                  TOL[dtype], dtype)


def test_tensors_without_requires_grad_get_nothing():
    from _gpu import x_to_t
    L = vo.make_layer(seed=50, **MOD)
    m = _module(L)
    for t in (m.res_centroids.weight, m.weight_scale, m.weight_bias):
        t.requires_grad_(False)
    x = x_to_t(vo.make_x(8, 1024, "fp16", seed=18), L)
    dy = x_to_t(vo.make_x(8, 512, "fp16", seed=19), L)
    got = _run_wgrad(m, x, dy)
    assert got["centroids"] is not None
    assert got["res_centroids"] is None and got["weight_scale"] is None and got["weight_bias"] is None
    # the absolute-maximum pass exists only for d weight_scale
    names = launched_kernels(lambda: _run_wgrad(m, x, dy))
    assert ran(names, "gemm_tn_wgmma") and ran(names, "wg_finish") and not ran(names, "wg_absmax"), names
    # nothing needs a gradient: no autograd node, no weight-gradient kernel
    m.centroids.weight.requires_grad_(False)
    m.bias.requires_grad_(False)
    names = launched_kernels(lambda: m(x))
    assert m(x).grad_fn is None and not any(ran(names, k) for k in WGRAD_KERNELS[:2] + WGRAD_KERNELS[3:]), names


def test_without_the_opt_in_nothing_changes():
    from _gpu import make_module, x_to_t
    L = vo.make_layer(seed=51, **MOD)
    m = make_module(L)
    assert m.centroids.weight.requires_grad and m.weight_scale.requires_grad
    x = x_to_t(vo.make_x(4, 1024, "fp16", seed=20), L)
    assert m(x).grad_fn is None                       # x does not require grad: no graph, as before
    xg = x.clone().requires_grad_()
    m(xg).sum().backward()
    assert xg.grad is not None and m.centroids.weight.grad is None and m.weight_scale.grad is None
    w = m.dequant()
    assert w.grad_fn is None


@pytest.mark.parametrize("tokens", [1, 2, 300])
def test_forward_values_are_bit_identical_under_the_opt_in(tokens):
    from _gpu import make_module, x_to_t
    L = vo.make_layer(seed=52, **MOD)
    ref = make_module(L)
    m = _module(L)
    x = x_to_t(vo.make_x(tokens, 1024, "fp16", seed=21), L)
    with torch.no_grad():
        y0 = ref(x)
        y1 = m(x)
        w0 = ref.dequant()
    y2 = m(x)
    w1 = m.dequant()
    assert y2.grad_fn is not None and w1.grad_fn is not None
    assert torch.equal(y0, y1) and torch.equal(y0, y2.detach()) and torch.equal(w0, w1.detach())


def test_proxy_error_forward_backpropagates_into_the_codebooks():
    from _gpu import x_to_t
    L = vo.make_layer(seed=53, in_features=512, out_features=256, vector_len=8, num_centroids=4096,
                      num_res_centroids=256)
    m = _module(L)
    W = (m.dequant().detach().float() + 0.01 * torch.randn(256, 512, device="cuda")).half()
    H = torch.rand(512, 512, device="cuda").half() / 512
    m.proxy_error_forward(W, H).float().sum().backward()
    # the same loss through a dense leaf W_: its gradient is G, fed to the oracle
    Wl = m.dequant().detach().requires_grad_()
    diff = Wl.to(W.dtype) - W
    (diff.T @ diff * H).float().sum().backward()
    _check_parity(_grads(m), grads_from_gamma(Wl.grad.double().cpu().numpy(), L), TOL["fp16"], "proxy")


def test_fused_qkv_under_the_opt_in_equals_unfused():
    import torch.nn as nn
    import vptq_b200
    from _gpu import make_module, x_to_t
    Ls = [vo.make_layer(in_features=1024, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                        seed=60 + k) for k, o in enumerate((1024, 256, 256))]
    x = x_to_t(vo.make_x(1, 1024, "fp16", seed=22), Ls[0])
    g = torch.Generator(device="cuda").manual_seed(4)
    ws = [torch.randn(1, o, device="cuda", generator=g) for o in (1024, 256, 256)]

    def run(fused):
        parent = nn.Module()
        parent.q_proj, parent.k_proj, parent.v_proj = (make_module(L) for L in Ls)
        mods = [parent.q_proj, parent.k_proj, parent.v_proj]
        if fused:
            assert len(vptq_b200.fuse(parent)) == 1
        assert vptq_b200.set_quant_grad(parent, True) == 3
        ys = [parent.q_proj(x), parent.k_proj(x), parent.v_proj(x)]
        sum((y.float() * w).sum() for y, w in zip(ys, ws)).backward()
        return [y.detach() for y in ys], [_grads(mm) for mm in mods]

    ya, ga = run(False)
    yb, gb = run(True)
    for a, b in zip(ya, yb):
        assert torch.equal(a, b)
    for a, b in zip(ga, gb):
        for n in a:
            assert a[n] is not None and torch.equal(a[n], b[n]), n


def test_decode_only_module_refuses_the_opt_in():
    from _gpu import make_module
    L = vo.make_layer(seed=54, in_features=2048, out_features=512, vector_len=8, num_centroids=65536,
                      num_res_centroids=256)
    m = make_module(L)
    m.prepare(drop_packed=True)
    with pytest.raises(RuntimeError, match="decode-only"):
        m.set_quant_grad(True)


def test_in_place_update_between_forward_and_backward_is_refused():
    from _gpu import x_to_t
    L = vo.make_layer(seed=55, in_features=512, out_features=256, vector_len=8, num_centroids=4096)
    m = _module(L)
    y = m(x_to_t(vo.make_x(4, 512, "fp16", seed=23), L))
    with torch.no_grad():
        m.centroids.weight.mul_(2)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


# ---------------------------------------------------------------- non-finite inputs
@pytest.mark.parametrize("where", ["dy", "x", "gamma"])
def test_one_inf_makes_every_requested_gradient_nan(where):
    from _gpu import x_to_t
    L = vo.make_layer(seed=56, **MOD)
    m = _module(L)
    x = x_to_t(vo.make_x(6, 1024, "fp16", seed=24), L)
    dy = x_to_t(vo.make_x(6, 512, "fp16", seed=25), L)
    if where == "gamma":
        gamma = x_to_t(vo.make_x(512, 1024, "fp16", seed=26), L)
        gamma[100, 7] = float("inf")
        got = _run_dequant_backward(m, gamma)
    else:
        (dy if where == "dy" else x)[3, 5] = float("inf")
        got = _run_wgrad(m, x, dy)
    for n, g in got.items():
        assert g is not None and torch.isnan(g).all(), n


# ---------------------------------------------------------------- training loop
def test_adam_steps_reduce_the_loss_and_keep_the_descriptor():
    import torch.nn as nn
    import vptq_b200
    from _gpu import make_module, x_to_t
    L1 = vo.make_layer(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                       seed=57)
    L2 = vo.make_layer(in_features=512, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256,
                       seed=58)
    model = nn.Sequential(make_module(L1), nn.ReLU(), make_module(L2))
    vptq_b200.set_quant_grad(model, True)
    for mm in (model[0], model[2]):
        mm.prepare()
        mm.weight_bias.requires_grad_(False)
    params = [p for mm in (model[0], model[2]) for p in (mm.centroids.weight, mm.res_centroids.weight, mm.weight_scale)]
    opt = torch.optim.Adam(params, lr=1e-4, eps=1e-4)
    x = x_to_t(vo.make_x(256, 1024, "fp16", seed=27), L1)
    target = torch.randn(256, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 0.1
    descs = [mm._desc_cache[0] for mm in (model[0], model[2])]
    streams = [d.lists_stream for d in descs]
    assert all(streams)
    x1 = x[:1].clone()
    x300 = x_to_t(vo.make_x(300, 1024, "fp16", seed=28), L1)
    losses = []
    for step in range(5):
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(model(x).float(), target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
        for k, (mm, L) in enumerate(((model[0], L1), (model[2], L2))):
            inp1, inp300 = (x1, x300) if k == 0 else (x1.new_zeros(1, 512).normal_(), x300.new_zeros(300, 512).normal_())
            fresh = make_module(L)
            fresh.load_state_dict(mm.state_dict())
            with torch.no_grad():
                assert torch.equal(mm(inp1), fresh(inp1)), (step, k)
                assert torch.equal(mm(inp300), fresh(inp300)), (step, k)
            assert mm._desc_cache[0] is descs[k], (step, k)                  # descriptor and lists were kept
            assert mm._desc_cache[0].lists_stream == streams[k], (step, k)
    assert losses[-1] < losses[0], losses


def test_large_finite_bf16_inputs_are_not_reported_as_non_finite():
    """|x| near the top of the bf16 range: the per-row bound sums exceed fp32 but are kept in fp64, and G itself is
    small, so every gradient is finite and accurate."""
    from _gpu import x_to_t
    L = vo.make_layer(seed=59, dtype="bf16", **MOD)
    m = _module(L)
    x_np = vo.f32_to_bf16_bits(np.full((2, 1024), 1e36, np.float32) * np.sign(np.random.default_rng(1).standard_normal((2, 1024))).astype(np.float32))
    dy_np = vo.f32_to_bf16_bits((1e-33 * np.random.default_rng(2).standard_normal((2, 512))).astype(np.float32))
    got = _run_wgrad(m, x_to_t(x_np, L), x_to_t(dy_np, L))
    _check_parity(got, quant_gemm_wgrad(x_np, dy_np, L), TOL["bf16"], "large bf16")
