"""GPU tests of the batched list kernel (csrc/gemv_lists_batch.cu, include/vptq_b200_batch.h): 1..8 tokens per launch
from the index lists.

Bars, per token t: |y - y*| <= TOL max|y*_t| + Q 2^-31 against the fp64 evaluation of the kernel's arithmetic
(x' = x * scale rounded to the layer type, c + r rounded to fp16 for fp16 layers), twice that against the exact
product.  One-hot probes are exact (tests/_probe.py, route "lists").  A token's outputs are bit-identical whatever
else is in its batch.  Every test asserts which kernel ran."""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _util import TOL

pytestmark = pytest.mark.gpu

from _batch import BATCH, ZERO_HEAD, assert_close, batch as _batch, desc_of as _desc, head_zero as _head_zero, q_of
from _batch import kernel_star as _kernel_star

CASES = {
    "4096x4096_r256": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256),
    "1024x4096_r256_bf16": dict(in_features=4096, out_features=1024, num_centroids=65536, num_res_centroids=256,
                                dtype="bf16"),
    "14336x4096_r256": dict(in_features=4096, out_features=14336, num_centroids=65536, num_res_centroids=256),
    "4096x14336_r256_bf16": dict(in_features=14336, out_features=4096, num_centroids=65536, num_res_centroids=256,
                                 dtype="bf16"),
    "k8192_r2_noperm": dict(in_features=2048, out_features=1024, num_centroids=8192, num_res_centroids=2,
                            enable_perm=False),
    "k65536_plain_bias_bf16": dict(in_features=2048, out_features=512, num_centroids=65536, enable_perm=False,
                                   enable_norm=False, bias=True, dtype="bf16"),
    "ragged_r16_bias": dict(in_features=1004, out_features=100, num_centroids=65536, num_res_centroids=16, bias=True),
}
SMALL = ("4096x4096_r256", "k8192_r2_noperm", "k65536_plain_bias_bf16", "ragged_r16_bias")

_layers = {}


def _layer(name):
    if name not in _layers:
        _layers[name] = vo.make_layer(vector_len=8, seed=71 + len(name), **CASES[name])
    return _layers[name]


def _q(L):
    return q_of(L.in_features, L.num_centroids)


def _x(L, tokens, seed):
    from _gpu import x_to_t
    return x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)


def _assert_close(y, ystar, L, factor=1.0):
    assert_close(y, ystar, L.dtype, _q(L), factor)


# ---------------------------------------------------------------- probes
@pytest.mark.parametrize("name", SMALL)
def test_probes_are_exact(name):
    from _probe import launched_kernels, probe_expect, ran
    L = _layer(name)
    d = _desc(L)
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)
    _batch(d, torch.zeros(1, L.in_features, dtype=dt, device="cuda"))   # (allocates the stream's workspace)
    rng = np.random.default_rng(5)
    for tokens in range(1, 9):
        f = rng.choice(L.in_features, size=tokens, replace=False)
        x = torch.zeros(tokens, L.in_features, dtype=dt, device="cuda")
        x[torch.arange(tokens), torch.from_numpy(f).cuda()] = 1.0
        y = torch.full((tokens, L.out_features), float("nan"), dtype=dt, device="cuda")
        names = launched_kernels(lambda: _batch(d, x, [y]))
        assert names and all(ran([nm], BATCH) for nm in names), names
        torch.cuda.synchronize()
        assert torch.equal(y.view(torch.int16), expect[torch.from_numpy(f).cuda()].view(torch.int16)), (name, tokens)
    _head_zero()


# ---------------------------------------------------------------- random x against fp64
@pytest.mark.parametrize("name", sorted(CASES))
def test_random_x_against_fp64(name):
    from _probe import fp64_bias, fp64_weight, launched_kernels, ran
    L = _layer(name)
    d = _desc(L)
    x = _x(L, 8, seed=3)
    y8 = _batch(d, x)
    names = launched_kernels(lambda: _batch(d, x, [y8]))
    assert ran(names, BATCH) and len(names) == 1, names
    exact = x.double() @ fp64_weight(L).t()
    if L.bias is not None:
        exact = exact + fp64_bias(L)
    kstar = _kernel_star(L, x)
    for tokens in (1, 2, 3, 4, 5, 8):
        y = _batch(d, x[:tokens])
        torch.cuda.synchronize()
        assert torch.isfinite(y).all()
        _assert_close(y, kstar[:tokens], L)
        _assert_close(y, exact[:tokens], L, factor=2.0)
    _head_zero()


# ---------------------------------------------------------------- token invariance
@pytest.mark.parametrize("name", ("4096x4096_r256", "1024x4096_r256_bf16", "ragged_r16_bias"))
def test_token_invariance(name):
    L = _layer(name)
    d = _desc(L)
    x = _x(L, 8, seed=11)
    y8 = _batch(d, x).clone()
    for tokens in range(1, 9):
        assert torch.equal(_batch(d, x[:tokens]), y8[:tokens]), tokens
    for seed in range(3):
        p = torch.from_numpy(np.random.default_rng(seed).permutation(8)).cuda()
        assert torch.equal(_batch(d, x[p]), y8[p])
    for tokens in (2, 5, 8):
        other = _x(L, tokens, seed=100 + tokens)
        other[tokens // 2] = x[0]
        assert torch.equal(_batch(d, other)[tokens // 2], y8[0])
    for _ in range(20):
        assert torch.equal(_batch(d, x), y8)
    torch.cuda.synchronize()
    _head_zero()


# ---------------------------------------------------------------- fused launches, graphs, PDL, strides
@pytest.mark.parametrize("n", (1, 2, 3, 4))
def test_fused_layers(n):
    from _probe import launched_kernels, ran
    from vptq_b200 import native
    outs = [4096, 1024, 1024, 520][:n]
    Ls = [vo.make_layer(in_features=4096, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                        seed=200 + k, bias=k == 1) for k, o in enumerate(outs)]
    ds = [_desc(L) for L in Ls]
    assert native.batch_max_tokens(ds) == 8
    x = _x(Ls[0], 6, seed=21)
    ys = _batch(ds, x)
    names = launched_kernels(lambda: _batch(ds, x, ys))
    assert [ran([nm], BATCH) for nm in names] == [True], names
    for L, y, d in zip(Ls, ys, ds):
        kstar = _kernel_star(L, x)
        _assert_close(y, kstar, L)
        _assert_close(_batch(d, x), kstar, L)
    # strided x and y: x rows 4100 elements apart (8-byte aligned rows), outputs into column slices of one buffer
    xs = torch.zeros(6, 4100, dtype=x.dtype, device="cuda")[:, :4096]
    xs.copy_(x)
    big = torch.full((6, sum(outs) + 8), float("nan"), dtype=x.dtype, device="cuda")
    offs = np.cumsum([0] + outs)
    views = [big[:, a:b] for a, b in zip(offs[:-1], offs[1:])]
    _batch(ds, xs, views)
    for y, v in zip(ys, views):
        assert torch.equal(y, v)
    # PDL and CUDA-graph capture / replay give the eager bits
    yp = _batch(ds, x, flags=native.FLAG_PDL)
    for y, v in zip(ys, yp):
        assert torch.equal(y, v)
    gy = [torch.empty_like(y) for y in ys]
    fb = native.FusedGemvBatch(ds, gy)
    fb(x, native.FLAG_PDL)                        # (workspace allocated outside the capture)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        fb(x, native.FLAG_PDL)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            fb(x, native.FLAG_PDL)
    for v in gy:
        v.fill_(float("nan"))
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    for y, v in zip(ys, gy):
        assert torch.equal(y, v)
    _head_zero()


def test_refusals_launch_nothing():
    from _probe import launched_kernels
    from vptq_b200 import native
    L = _layer("4096x4096_r256")
    d = _desc(L)
    x = _x(L, 9, seed=1)
    with pytest.raises(RuntimeError, match="9 tokens"):
        _batch(d, x)
    y9 = [torch.empty(9, L.out_features, dtype=x.dtype, device="cuda")]
    assert launched_kernels(lambda: pytest.raises(RuntimeError, _batch, d, x, y9)) == []
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        _batch(d, torch.zeros(2 * 4096 + 1, dtype=x.dtype, device="cuda")[1:].view(2, 4096))
    ys = [torch.empty(2, L.out_features, dtype=x.dtype, device="cuda")]
    fb = native.FusedGemvBatch([d], ys)
    rc = native.lib().vptq_b200_quant_gemv_batch(1, fb.desc_arr, x.data_ptr(), 4096, fb.y_arr, fb.stride_arr, 2,
                                                  native.workspace(x.device, ZERO_HEAD).data_ptr(), 1024, 0,
                                                  torch.cuda.current_stream().cuda_stream)
    assert rc == -3 and "workspace" in native.last_error()        # VPTQ_ERR_WORKSPACE
    d_nolists = native.make_desc(**{**_desc_kwargs(L), "lists": False})
    assert native.batch_max_tokens(d_nolists) == 0


def _desc_kwargs(L):
    from _gpu import tdtype, to_t
    return dict(dtype=tdtype(L), in_features=L.in_features, out_features=L.out_features, vector_len=8,
                num_centroids=L.num_centroids, num_res_centroids=L.num_res_centroids, num_codebooks=1,
                group_size=L.group_size, outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1,
                outlier_indices=None, outlier_centroids=None, indices=to_t(L.indices, L, "i32"),
                centroids=to_t(L.centroids, L), res_centroids=to_t(L.res_centroids, L), perm=to_t(L.perm, L, "u16"),
                weight_scale=to_t(L.weight_scale, L), weight_bias=to_t(L.weight_bias, L), bias=None)


# ---------------------------------------------------------------- skewed lists
@pytest.mark.parametrize("kind", ("zipf_hot0", "row_slice", "constant", "ramp", "col_slice"))
def test_skewed_lists(kind):
    import _envelope as en
    L = en.layer_with(kind, in_features=4096, out_features=1024, vector_len=8, num_centroids=65536,
                      num_res_centroids=256, seed=31)
    d = _desc(L)
    x = _x(L, 8, seed=4)
    y8 = _batch(d, x)
    _assert_close(y8, _kernel_star(L, x), L)
    assert torch.equal(_batch(d, x[3:6]), y8[3:6])
    _head_zero()


# ---------------------------------------------------------------- non-finite values
@pytest.mark.parametrize("value", ("nan", "+inf", "-inf"))
@pytest.mark.parametrize("dtype", ("fp16", "bf16"))
def test_nonfinite_x_stays_in_its_token(value, dtype):
    import _extreme as ex
    L = vo.make_layer(in_features=2048, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      seed=41, dtype=dtype)
    d = _desc(L)
    x = _x(L, 5, seed=6)
    clean = _batch(d, x).clone()
    xb = x.clone()
    xb[2, 77] = ex.VALUES[value]
    y = _batch(d, xb)
    others = [0, 1, 3, 4]
    assert torch.equal(y[others], clean[others])
    assert torch.equal(ex.classify(y[2]), ex.classify(_kernel_star(L, xb)[2]))
    assert not torch.isfinite(y[2]).any()
    _head_zero()


@pytest.mark.parametrize("site", ("C", "R", "scale", "wbias", "bias"))
@pytest.mark.parametrize("value", ("nan", "+inf", "-inf"))
def test_nonfinite_layer_values(site, value):
    import _extreme as ex
    L = vo.make_layer(in_features=2048, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      seed=43, bias=True)
    k = int(L.meta["ridx" if site == "R" else "idx"][0, 3, 10])     # an entry index row 3 uses
    L = ex.inject(L, site, ex.VALUES[value], k=k, e=2, f=ex.feature_of(L, 10), o=21)
    d = _desc(L)
    x = _x(L, 4, seed=8)
    y = _batch(d, x)
    ystar = _kernel_star(L, x)
    cls = ex.classify(ystar)
    assert torch.equal(ex.classify(y), cls)
    assert (cls != 0).any()
    fin = cls == 0            # (none where scale or wbias of a feature is not finite: every output reads it)
    if fin.any():
        bar = TOL["fp16"] * float(ystar[fin].abs().max()) + _q(L) * 2.0 ** -31
        assert float((y[fin].double() - ystar[fin]).abs().max()) <= bar
    _head_zero()


def test_fp16_overflow_becomes_inf():
    L = vo.make_layer(in_features=4096, out_features=512, vector_len=8, num_centroids=65536, seed=45,
                      enable_norm=False)
    L.centroids = (np.abs(L.centroids.astype(np.float32)) * 300).astype(np.float16)
    d = _desc(L)
    x = _x(L, 3, seed=9).abs()
    x[0] *= 8                                     # token 0: outputs past 65504; tokens 1, 2: ordinary values
    y = _batch(d, x)
    ystar = _kernel_star(L, x)
    big, small = ystar.abs() > 70000, ystar.abs() < 60000
    assert big.any() and small.any()
    assert torch.equal(y[big].double(), torch.sign(ystar[big]) * float("inf"))
    assert torch.isfinite(y[small]).all()
    _head_zero()


# ---------------------------------------------------------------- module level
def _module(name="4096x4096_r256"):
    from _gpu import make_module
    return make_module(_layer(name))


def test_module_opt_in_routing():
    from _probe import launched_kernels, ran
    m, fresh = _module(), _module()
    L = _layer("4096x4096_r256")
    x = _x(L, 9, seed=12)
    with torch.no_grad():
        m.set_batched_decode(True)
        for tokens in range(1, 10):
            names = launched_kernels(lambda: m(x[:tokens]))
            assert ran(names, BATCH) == (2 <= tokens <= 8), (tokens, names)
            if tokens == 1:
                assert ran(names, "gemv_lists_kernel")
        yb = m(x[:8])
        _assert_close(yb, _kernel_star(L, x[:8]), L)
        m.set_batched_decode(False)
        for tokens in range(1, 10):
            names = launched_kernels(lambda: m(x[:tokens]))
            assert not ran(names, BATCH)
            assert torch.equal(m(x[:tokens]), fresh(x[:tokens])), tokens


def test_module_grad_mode_same_values_and_backward():
    m, ref = _module(), _module()
    m.set_batched_decode(True)
    L = _layer("4096x4096_r256")
    x = _x(L, 4, seed=13)
    with torch.no_grad():
        y0 = m(x)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    assert torch.equal(y.detach(), y0)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.clone().requires_grad_(True)
    ref(xr).backward(dy)
    assert torch.equal(xg.grad, xr.grad)          # backward unchanged: the same dX kernel


def test_decode_only_module_serves_2_to_8_tokens():
    from _probe import launched_kernels, ran
    full, m = _module(), _module()
    full.set_batched_decode(True)
    m.set_batched_decode(True)
    m.prepare(drop_packed=True)
    L = _layer("4096x4096_r256")
    x = _x(L, 9, seed=14)
    with torch.no_grad():
        for tokens in range(2, 9):
            assert ran(launched_kernels(lambda: m(x[:tokens])), BATCH)
            assert torch.equal(m(x[:tokens]), full(x[:tokens]))
        with pytest.raises(RuntimeError, match="decode-only"):
            m(x)
    with pytest.raises(RuntimeError, match="decode-only"):
        m.dequant()


def test_fuse_opt_in_launches_each_group_once():
    import vptq_b200
    from _gpu import make_module
    from _probe import launched_kernels, ran
    Ls = {n: vo.make_layer(in_features=4096, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                           seed=300 + k) for k, (n, o) in enumerate((("q_proj", 4096), ("k_proj", 1024),
                                                                     ("v_proj", 1024)))}

    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for n, L in Ls.items():
                setattr(self, n, make_module(L))

        def forward(self, x):
            return self.q_proj(x), self.k_proj(x), self.v_proj(x)

    model, plain = Attn(), Attn()
    groups = vptq_b200.fuse(model)
    assert len(groups) == 1
    assert vptq_b200.set_batched_decode(model) == 3
    for n in Ls:
        getattr(plain, n).set_batched_decode(True)
    x = _x(Ls["q_proj"], 8, seed=15)
    with torch.no_grad():
        for tokens in (2, 5, 8):
            model(x[:tokens])                       # (allocates the group's output and workspace)
            names = launched_kernels(lambda: model(x[:tokens]))
            assert sum(ran([nm], BATCH) for nm in names) == 1 and len(names) == 1, names
            for n, y in zip(Ls, model(x[:tokens])):
                _assert_close(y, _kernel_star(Ls[n], x[:tokens]), Ls[n])
                _assert_close(getattr(plain, n)(x[:tokens]), _kernel_star(Ls[n], x[:tokens]), Ls[n])
        assert vptq_b200.set_batched_decode(model, False) == 3
        names = launched_kernels(lambda: model(x[:5]))
        assert not any(ran([nm], BATCH) for nm in names)
    _head_zero()
