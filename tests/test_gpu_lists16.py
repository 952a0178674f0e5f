"""GPU tests of the vector-length-16 list kernel (csrc/gemv_lists16.cu, include/vptq_b200_lists16.h): 1..4 tokens per
launch of v = 16 layers from index lists with rows of 16 outputs.

Bars, per token t: |y - y*| <= TOL max|y*_t| + Q 2^-31 against the fp64 evaluation of the kernel's arithmetic
(x' = x * scale rounded to the layer type, c + r rounded to fp16 for fp16 layers), twice that against the exact
product.  One-hot probes are exact (tests/_probe.py, route "lists": the same arithmetic for any vector length).  A
token's outputs are bit-identical whatever else is in its launch.  Every test asserts which kernel ran."""
import numpy as np
import pytest
import torch

import vptq_oracle as vo

pytestmark = pytest.mark.gpu

from _batch import ZERO_HEAD, assert_close, head_zero, kernel_star, q_of, rand_x
from _lists16 import KERNEL, GpuLayer16, desc_t as _desc_t

CASES = {
    "k65536_r256_fp16": dict(in_features=4096, out_features=1024, num_centroids=65536, num_res_centroids=256),
    "k65536_r256_bf16": dict(in_features=4096, out_features=1024, num_centroids=65536, num_res_centroids=256,
                             dtype="bf16"),
    "k8192_r2_noperm": dict(in_features=2048, out_features=512, num_centroids=8192, num_res_centroids=2,
                            enable_perm=False),
    "k16384_r64_bf16": dict(in_features=1024, out_features=256, num_centroids=16384, num_res_centroids=64,
                            dtype="bf16"),
    "k65536_plain_bias_bf16": dict(in_features=2048, out_features=512, num_centroids=65536, enable_perm=False,
                                   enable_norm=False, bias=True, dtype="bf16"),
    "ragged_4100_r256_bias": dict(in_features=4100, out_features=264, num_centroids=65536, num_res_centroids=256,
                                  bias=True),
    "ragged_9004_nores": dict(in_features=9004, out_features=200, num_centroids=65536),
    "k32768_r256_nonorm": dict(in_features=3000, out_features=520, num_centroids=32768, num_res_centroids=256,
                               enable_norm=False),
}
SMALL = ("k65536_r256_fp16", "k8192_r2_noperm", "k65536_plain_bias_bf16", "ragged_4100_r256_bias")

_layers = {}


def _layer(name):
    if name not in _layers:
        _layers[name] = vo.make_layer(vector_len=16, seed=91 + len(name), **CASES[name])
    return _layers[name]


def _tensors(L):
    from _gpu import to_t
    return dict(indices=to_t(L.indices, L, "i32"), centroids=to_t(L.centroids, L),
                res_centroids=to_t(L.res_centroids, L) if L.res_bits else None,
                perm=to_t(L.perm, L, "u16") if L.perm is not None else None,
                weight_scale=to_t(L.weight_scale, L) if L.weight_scale is not None else None,
                weight_bias=to_t(L.weight_bias, L) if L.weight_bias is not None else None,
                bias=to_t(L.bias, L) if L.bias is not None else None)


def _desc(L, lists16=True):
    d = _desc_t(_tensors(L), L.dtype, L.in_features, L.out_features, L.num_centroids, L.num_res_centroids, lists16)
    assert bool(d.lists_stream) == lists16
    return d


def _run(descs, x, ys=None, flags=0):
    """one vptq_b200_quant_gemv_lists16 launch; outputs NaN-filled unless given"""
    from vptq_b200 import native
    single = not isinstance(descs, (list, tuple))
    descs = [descs] if single else list(descs)
    if ys is None:
        ys = [torch.full((x.shape[0], d.out_features), float("nan"), dtype=x.dtype, device=x.device) for d in descs]
    native.FusedGemvLists16(descs, ys)(x, flags)
    return ys[0] if single else ys


def _x(L, tokens, seed):
    from _gpu import x_to_t
    return x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)


def _close(y, ystar, L, factor=1.0):
    assert_close(y, ystar, L.dtype, q_of(L.in_features, L.num_centroids), factor)


def _only_kernel(fn):
    from _probe import launched_kernels, ran
    names = launched_kernels(fn)
    assert names and all(ran([n], KERNEL) for n in names), names


# ---------------------------------------------------------------- probes
@pytest.mark.parametrize("name", SMALL)
def test_probes_are_exact_on_both_halves(name):
    from _probe import probe_expect
    L = _layer(name)
    d = _desc(L)
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)
    _run(d, torch.zeros(1, L.in_features, dtype=dt, device="cuda"))
    rng = np.random.default_rng(5)
    for rep in range(3):
        for tokens in range(1, 5):
            f = rng.choice(L.in_features, size=tokens, replace=False)
            x = torch.zeros(tokens, L.in_features, dtype=dt, device="cuda")
            x[torch.arange(tokens), torch.from_numpy(f).cuda()] = 1.0
            y = torch.full((tokens, L.out_features), float("nan"), dtype=dt, device="cuda")
            _only_kernel(lambda: _run(d, x, [y]))
            torch.cuda.synchronize()
            want = expect[torch.from_numpy(f).cuda()]
            for half in (slice(0, 8), slice(8, 16)):       # outputs 16 r + 0..7 (lo plane), 16 r + 8..15 (hi plane)
                cols = torch.arange(L.out_features, device="cuda")
                cols = cols[(cols % 16 >= half.start) & (cols % 16 < half.stop)]
                assert torch.equal(y[:, cols].view(torch.int16), want[:, cols].view(torch.int16)), (name, tokens)
    head_zero()


# ---------------------------------------------------------------- random x against fp64
@pytest.mark.parametrize("name", sorted(CASES))
def test_random_x_against_fp64(name):
    from _probe import fp64_bias, fp64_weight
    from vptq_b200 import native
    L = _layer(name)
    d = _desc(L)
    assert native.lists16_max_tokens(d) == 4
    x = _x(L, 4, seed=3)
    exact = x.double() @ fp64_weight(L).t()
    if L.bias is not None:
        exact = exact + fp64_bias(L)
    kstar = kernel_star(L, x)
    for tokens in (1, 2, 3, 4):
        y = _run(d, x[:tokens])
        if tokens == 4:
            _only_kernel(lambda: _run(d, x[:tokens], [y]))
        torch.cuda.synchronize()
        assert torch.isfinite(y).all()
        _close(y, kstar[:tokens], L)
        _close(y, exact[:tokens], L, factor=2.0)
    head_zero()


# ---------------------------------------------------------------- full-size layers, checked on sampled rows
FULL = {   # (in_features, [out_features of the fused members]): Llama-3-70B / Nemotron-70B and Llama-3.1-405B
    "70b_qkv": (8192, [8192, 1024, 1024]), "70b_o": (8192, [8192]), "70b_gate_up": (8192, [28672, 28672]),
    "70b_down": (28672, [8192]), "405b_q": (16384, [16384]), "405b_o": (16384, [16384]),
    "405b_gate_up": (16384, [53248, 53248]),
}


@pytest.mark.parametrize("name", sorted(FULL))
def test_full_size_shapes_against_fp64(name):
    from vptq_b200 import native
    I, outs = FULL[name]
    Ls = [GpuLayer16(I, o, seed=500 + k) for k, o in enumerate(outs)]
    ds = [G.desc for G in Ls]
    assert native.lists16_max_tokens(ds) == 4
    x = rand_x(4, I, "fp16", seed=7)
    ys = _run(ds, x)
    _only_kernel(lambda: _run(ds, x, ys))
    for G, y in zip(Ls, ys):
        G.check(x, y)
    y1 = _run(ds, x[2:3])
    for a, b in zip(ys, y1):
        assert torch.equal(a[2:3], b)
    del Ls, ds, ys
    torch.cuda.empty_cache()
    head_zero()


# ---------------------------------------------------------------- token invariance, fused launches, graphs, PDL
@pytest.mark.parametrize("name", ("k65536_r256_fp16", "k65536_r256_bf16", "ragged_4100_r256_bias"))
def test_token_invariance(name):
    L = _layer(name)
    d = _desc(L)
    x = _x(L, 4, seed=11)
    y4 = _run(d, x).clone()
    for tokens in range(1, 5):
        for start in range(0, 5 - tokens):
            xs = x[start:start + tokens].clone()          # (rows of 4100 features: a fresh, aligned copy)
            assert torch.equal(_run(d, xs), y4[start:start + tokens]), (tokens, start)
    for seed in range(3):
        p = torch.from_numpy(np.random.default_rng(seed).permutation(4)).cuda()
        assert torch.equal(_run(d, x[p]), y4[p])
    for tokens in (2, 3, 4):
        for pos in range(tokens):
            other = _x(L, tokens, seed=100 + 7 * tokens + pos)
            other[pos] = x[0]
            assert torch.equal(_run(d, other)[pos], y4[0]), (tokens, pos)
    for _ in range(10):
        assert torch.equal(_run(d, x), y4)
    torch.cuda.synchronize()
    head_zero()


@pytest.mark.parametrize("n", (1, 2, 3, 4))
def test_fused_layers_graphs_pdl_strides(n):
    from vptq_b200 import native
    outs = [4096, 1024, 1024, 520][:n]
    Ls = [vo.make_layer(in_features=4096, out_features=o, vector_len=16, num_centroids=65536, num_res_centroids=256,
                        seed=200 + k, bias=k == 1) for k, o in enumerate(outs)]
    ds = [_desc(L) for L in Ls]
    assert native.lists16_max_tokens(ds) == 4
    x = _x(Ls[0], 3, seed=21)
    ys = _run(ds, x)
    _only_kernel(lambda: _run(ds, x, ys))
    fresh = _run([_desc(L) for L in Ls], x)             # a fresh fused group: the same bits
    for L, y, d, f in zip(Ls, ys, ds, fresh):
        assert torch.equal(y, f)
        _close(y, kernel_star(L, x), L)
        if n == 1:
            assert torch.equal(_run(d, x), y)
        else:                                            # alone: another partition of the same sums
            _close(_run(d, x), kernel_star(L, x), L)
    xs = torch.zeros(3, 4104, dtype=x.dtype, device="cuda")[:, :4096]
    xs.copy_(x)
    big = torch.full((3, sum(outs) + 8), float("nan"), dtype=x.dtype, device="cuda")
    offs = np.cumsum([0] + outs)
    views = [big[:, a:b] for a, b in zip(offs[:-1], offs[1:])]
    _run(ds, xs, views)
    for y, v in zip(ys, views):
        assert torch.equal(y, v)
    for y, v in zip(ys, _run(ds, x, flags=native.FLAG_PDL)):
        assert torch.equal(y, v)
    gy = [torch.empty_like(y) for y in ys]
    fb = native.FusedGemvLists16(ds, gy)
    fb(x, native.FLAG_PDL)
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
    head_zero()


def test_refusals_launch_nothing():
    from _probe import launched_kernels
    from vptq_b200 import native
    L = _layer("k65536_r256_fp16")
    d = _desc(L)
    x = _x(L, 5, seed=1)
    with pytest.raises(RuntimeError, match="5 tokens"):
        _run(d, x)
    y5 = [torch.empty(5, L.out_features, dtype=x.dtype, device="cuda")]
    assert launched_kernels(lambda: pytest.raises(RuntimeError, _run, d, x, y5)) == []
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        _run(d, torch.zeros(2 * 4096 + 1, dtype=x.dtype, device="cuda")[1:].view(2, 4096))
    ys = [torch.empty(2, L.out_features, dtype=x.dtype, device="cuda")]
    fb = native.FusedGemvLists16([d], ys)
    ws = native.workspace(x.device, ZERO_HEAD)
    st = torch.cuda.current_stream().cuda_stream
    assert native.lib().vptq_b200_quant_gemv_lists16(1, fb.desc_arr, x.data_ptr(), 4096, fb.y_arr, fb.stride_arr, 2,
                                                     ws.data_ptr(), 1024, 0, st) == -3
    assert "workspace" in native.last_error()
    assert native.lib().vptq_b200_quant_gemv_lists16(1, fb.desc_arr, x.data_ptr(), 4096, fb.y_arr, fb.stride_arr, 2,
                                                     ws.data_ptr(), ws.numel(), 4, st) == -1
    assert native.lists16_max_tokens(_desc(L, lists16=False)) == 0
    # a v = 8 descriptor with v = 8 lists is not this kernel's
    L8 = vo.make_layer(in_features=4096, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                       seed=3)
    from _batch import desc_of
    d8 = desc_of(L8)
    assert native.lib().vptq_b200_quant_gemv_lists16_max_tokens(1, native._desc_array([d8])) == 0
    assert "vector-length-16" in native.last_error()
    assert launched_kernels(lambda: pytest.raises(RuntimeError, native.FusedGemvLists16([d8], y5[:1]), x[:2])) == []
    head_zero()


# ---------------------------------------------------------------- skewed lists
@pytest.mark.parametrize("kind", ("zipf_hot0", "row_slice", "constant"))
def test_skewed_lists(kind):
    import _envelope as en
    L = en.layer_with(kind, in_features=4096, out_features=1024, vector_len=16, num_centroids=65536,
                      num_res_centroids=256, seed=31)
    d = _desc(L)
    x = _x(L, 4, seed=4)
    y4 = _run(d, x)
    _close(y4, kernel_star(L, x), L)
    assert torch.equal(_run(d, x[1:3]), y4[1:3])
    head_zero()


# ---------------------------------------------------------------- non-finite values
@pytest.mark.parametrize("value", ("nan", "+inf", "-inf"))
@pytest.mark.parametrize("dtype", ("fp16", "bf16"))
def test_nonfinite_x_stays_in_its_token(value, dtype):
    import _extreme as ex
    L = vo.make_layer(in_features=2048, out_features=512, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      seed=41, dtype=dtype)
    d = _desc(L)
    x = _x(L, 4, seed=6)
    clean = _run(d, x).clone()
    xb = x.clone()
    xb[2, 77] = ex.VALUES[value]
    y = _run(d, xb)
    assert torch.equal(y[[0, 1, 3]], clean[[0, 1, 3]])
    assert torch.equal(ex.classify(y[2]), ex.classify(kernel_star(L, xb)[2]))
    assert not torch.isfinite(y[2]).any()
    head_zero()


@pytest.mark.parametrize("site,e", (("C", 2), ("C", 13), ("R", 5), ("R", 10), ("scale", 0), ("wbias", 0),
                                    ("bias", 0)))
@pytest.mark.parametrize("value", ("nan", "+inf", "-inf"))
def test_nonfinite_layer_values(site, e, value):
    import _extreme as ex
    L0 = vo.make_layer(in_features=2048, out_features=512, vector_len=16, num_centroids=65536, num_res_centroids=256,
                       seed=43, bias=True)
    k = int(L0.meta["ridx" if site == "R" else "idx"][0, 3, 10])     # an entry index row 3 uses
    L = ex.inject(L0, site, ex.VALUES[value], k=k, e=e, f=ex.feature_of(L0, 10), o=21)
    x = _x(L, 4, seed=8)
    clean = _run(_desc(L0), x).clone()
    y = _run(_desc(L), x)
    ystar = kernel_star(L, x)
    cls = ex.classify(ystar)
    assert torch.equal(ex.classify(y), cls)
    assert (cls != 0).any()
    fin = cls == 0
    assert torch.equal(y[fin], clean[fin])                    # every other output unchanged, bit for bit
    head_zero()


def test_nan_entry_0_of_every_slice_plane_reaches_no_other_output():
    """Padding lanes read entry 0 of the slice (and residual entry 0): with no field using those entries, NaN in both
    planes of all of them changes no output."""
    import _extreme as ex
    L0 = vo.make_layer(in_features=4100, out_features=272, vector_len=16, num_centroids=65536, num_res_centroids=256,
                       seed=47)
    idx, ridx = vo.unpack_index(L0.indices, L0.index_bits, L0.group_size, L0.res_bits)
    idx = np.where(idx % 4096 == 0, idx + 1, idx)
    ridx = np.where(ridx == 0, 1, ridx)
    L0 = ex.copy_layer(L0)
    L0.indices = vo.pack_index(idx, L0.index_bits, ridx, L0.res_bits)
    L = L0
    for s in range(16):
        for e in range(16):
            L = ex.inject(L, "C", float("nan"), k=s * 4096, e=e)
    for e in range(16):
        L = ex.inject(L, "R", float("nan"), k=0, e=e)
    x = _x(L, 4, seed=9)
    d = _desc(L)
    assert native_tab_has_padding(d)
    clean = _run(_desc(L0), x).clone()
    y = _run(d, x)
    assert torch.isfinite(y).all() and (ex.classify(kernel_star(L, x)) == 0).all()
    assert torch.equal(y, clean)
    head_zero()


def native_tab_has_padding(d):
    """some list of the descriptor ends in a partial step (its padding lanes read entry 0)"""
    tab = d._keep[3] if len(d._keep) > 3 else d._keep[1]
    t = tab.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return bool(((t[:-1] >> 26) < 32).any())


# ---------------------------------------------------------------- existing entry points ignore the v = 16 lists
@pytest.mark.parametrize("dtype", ("fp16", "bf16"))
def test_existing_entry_points_treat_v16_lists_as_absent(dtype):
    from _probe import launched_kernels, ran
    from vptq_b200 import native
    L = vo.make_layer(in_features=4096, out_features=512, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      seed=51, dtype=dtype, bias=True)
    t = _tensors(L)
    with_l = _desc_t(t, L.dtype, 4096, 512, 65536, 256, True)
    without = _desc_t(t, L.dtype, 4096, 512, 65536, 256, False)
    assert with_l.lists_stream and not without.lists_stream
    dt = t["centroids"].dtype
    for tokens in (1, 2, 3, 16):
        assert native.workspace_bytes(with_l, tokens, native.OP_GEMV) == native.workspace_bytes(without, tokens,
                                                                                                native.OP_GEMV)
    for tokens in (1, 2):                                       # the generic GEMV
        x = _x(L, tokens, seed=tokens)
        a, b = (torch.empty(tokens, 512, dtype=dt, device="cuda") for _ in range(2))
        names = launched_kernels(lambda: native.quant_gemv(with_l, x, a))
        assert not ran(names, KERNEL) and not ran(names, "gemv_lists_kernel"), names
        native.quant_gemv(without, x, b)
        assert torch.equal(a, b)
        fa, fb = (torch.empty(tokens, 512, dtype=dt, device="cuda") for _ in range(2))
        native.FusedGemv([with_l], [fa])(x)
        native.FusedGemv([without], [fb])(x)
        assert torch.equal(fa, fb)
    x = _x(L, 16, seed=5)                                       # prefill
    a, b = (torch.empty(16, 512, dtype=dt, device="cuda") for _ in range(2))
    native.quant_gemm(with_l, x, a)
    native.quant_gemm(without, x, b)
    assert torch.equal(a, b)
    wa, wb = (torch.empty(512, 4096, dtype=dt, device="cuda") for _ in range(2))
    native.dequant(with_l, wa)
    native.dequant(without, wb)
    assert torch.equal(wa, wb)
    dy = rand_x(16, 512, dtype, seed=6)
    da, db = (torch.empty(16, 4096, dtype=dt, device="cuda") for _ in range(2))
    native.quant_gemm_dgrad(with_l, dy, da)
    native.quant_gemm_dgrad(without, dy, db)
    assert torch.equal(da, db)
    ga = {"centroids": torch.empty_like(t["centroids"]), "weight_scale": torch.empty_like(t["weight_scale"])}
    gb = {k: torch.empty_like(v) for k, v in ga.items()}
    native.quant_gemm_wgrad(with_l, x, dy, ga)
    native.quant_gemm_wgrad(without, x, dy, gb)
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k
    gb2 = {k: torch.empty_like(v) for k, v in ga.items()}
    native.dequant_backward(with_l, wa, ga)
    native.dequant_backward(without, wa, gb2)
    for k in ga:
        assert torch.equal(ga[k], gb2[k]), k


# ---------------------------------------------------------------- module level
def _module(L):
    from _gpu import make_module
    return make_module(L)


def test_module_opt_in_routing_and_refusals():
    from _probe import launched_kernels, ran
    L = _layer("k65536_r256_fp16")
    m, fresh = _module(L), _module(L)
    x = _x(L, 6, seed=12)
    with torch.no_grad():
        fresh(x[:1])
        m(x[:1])                                              # a descriptor without lists exists: opt-in rebuilds it
        assert m.set_list_decode(True) is m
        for tokens in range(1, 7):
            names = launched_kernels(lambda: m(x[:tokens]))
            assert ran(names, KERNEL) == (tokens <= 4), (tokens, names)
            if tokens > 4:
                assert torch.equal(m(x[:tokens]), fresh(x[:tokens]))
        _close(m(x[:4]), kernel_star(L, x[:4]), L)
        assert torch.equal(m(x[:4]), _run(_desc(L), x[:4]))
        m.set_list_decode(False)
        for tokens in range(1, 7):
            assert not ran(launched_kernels(lambda: m(x[:tokens])), KERNEL)
            assert torch.equal(m(x[:tokens]), fresh(x[:tokens])), tokens
    with pytest.raises(RuntimeError, match="vector_len 8 only"):
        m.set_list_decode(True).prepare(drop_packed=True)
    assert m.indices.numel() > 0
    head_zero()


def _v16_layer_kwargs():
    return dict(in_features=4096, out_features=512, vector_len=16, num_centroids=65536, num_res_centroids=256)


@pytest.mark.parametrize("kind", ("groups", "outliers", "kr512", "k4096", "v8"))
def test_ineligible_layers_opted_in_run_todays_kernels(kind):
    from _probe import launched_kernels, ran
    from vptq_b200 import native
    kw = _v16_layer_kwargs()
    if kind == "groups":
        kw.update(num_codebooks=2)
    elif kind == "outliers":
        kw.update(outlier_size=128, outlier_vector_len=4, num_outlier_centroids=256)
    elif kind == "kr512":
        kw.update(num_res_centroids=512)
    elif kind == "k4096":
        kw.update(num_centroids=4096)
    else:
        kw.update(vector_len=8)
    L = vo.make_layer(seed=61, **kw)
    m, fresh = _module(L), _module(L)
    m.set_list_decode(True)
    x = _x(L, 4, seed=13)
    with torch.no_grad():
        for tokens in (1, 2, 4):
            names = launched_kernels(lambda: m(x[:tokens]))
            assert not ran(names, KERNEL), names
            assert torch.equal(m(x[:tokens]), fresh(x[:tokens]))
    d = m._desc_cache[0]
    assert native.lists16_max_tokens(d) == 0
    if kind != "v8":
        assert not d.lists_stream


def test_405b_down_is_left_to_todays_route():
    """I = 53248: 16 slices x 13 column tiles > 132 SMs: no lists are built, the query returns 0, the module keeps its
    route"""
    from _probe import launched_kernels, ran
    from vptq_b200 import VQuantLinear, native
    G = GpuLayer16(53248, 2048, seed=9)
    assert not G.desc.lists_stream and native.lists16_max_tokens(G.desc) == 0
    m = VQuantLinear(53248, 2048, vector_lens=[-1, 16], num_centroids=[-1, 65536], num_res_centroids=[-1, 256],
                     group_num=1, group_size=53248, outlier_size=0, indices_as_float=False, enable_norm=True,
                     enable_perm=True, is_indice_packed=True, device="cuda", dtype=torch.float16,
                     enable_proxy_error=False)
    with torch.no_grad():
        for k in ("indices", "perm", "weight_scale", "weight_bias"):
            getattr(m, k).data = G.t[k]
        m.centroids.weight.data = G.t["centroids"].reshape(1, -1)
        m.res_centroids.weight.data = G.t["res_centroids"].reshape(1, -1)
        x = rand_x(2, 53248, "fp16", seed=3)
        y0 = m(x)
        m.set_list_decode(True)
        names = launched_kernels(lambda: m(x))
        assert not ran(names, KERNEL) and torch.equal(m(x), y0)


def test_module_grad_mode_same_values_and_backward():
    L = _layer("k65536_r256_bf16")
    m, ref = _module(L), _module(L)
    m.set_list_decode(True)
    x = _x(L, 3, seed=13)
    with torch.no_grad():
        y0 = m(x)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    assert torch.equal(y.detach(), y0)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.clone().requires_grad_(True)
    ref(xr).backward(dy)
    assert torch.equal(xg.grad, xr.grad)


def test_fuse_opt_in_launches_each_group_once():
    import vptq_b200
    from _probe import launched_kernels, ran
    Ls = {n: vo.make_layer(in_features=4096, out_features=o, vector_len=16, num_centroids=65536,
                           num_res_centroids=256, seed=300 + k)
          for k, (n, o) in enumerate((("q_proj", 4096), ("k_proj", 1024), ("v_proj", 1024)))}

    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for n, L in Ls.items():
                setattr(self, n, _module(L))

        def forward(self, x):
            return self.q_proj(x), self.k_proj(x), self.v_proj(x)

    model, plain = Attn(), Attn()
    assert len(vptq_b200.fuse(model)) == 1
    x = _x(Ls["q_proj"], 6, seed=15)
    with torch.no_grad():
        for tokens in (1, 2):                                  # not opted in: each member's own forward, today's bits
            for a, b in zip(model(x[:tokens]), plain(x[:tokens])):
                assert torch.equal(a, b)
            assert not any(ran([nm], KERNEL) for nm in launched_kernels(lambda: model(x[:tokens])))
        assert vptq_b200.set_list_decode(model) == 3
        descs = [_desc(L) for L in Ls.values()]
        for tokens in (1, 2, 3, 4):
            model(x[:tokens])
            names = launched_kernels(lambda: model(x[:tokens]))
            assert len(names) == 1 and ran(names, KERNEL), names
            for y, f in zip(model(x[:tokens]), _run(descs, x[:tokens])):   # = a fresh fused group, bit for bit
                assert torch.equal(y, f)
        names = launched_kernels(lambda: model(x[:5]))
        assert not any(ran([nm], KERNEL) for nm in names)
        assert vptq_b200.set_list_decode(model, False) == 3
        assert not any(ran([nm], KERNEL) for nm in launched_kernels(lambda: model(x[:2])))
    head_zero()


# ---------------------------------------------------------------- lifecycle
def test_graph_replay_across_workspace_growth():
    from vptq_b200 import native
    L = _layer("k65536_r256_fp16")
    m = _module(L).set_list_decode(True)
    m.prepare()
    x = _x(L, 2, seed=17)
    with torch.no_grad():
        want = m(x).clone()
        native.release_workspaces()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                out = m(x)
        native.workspace(x.device, 64 << 20)                  # the stream's workspace grows after the capture
        big = torch.randn(64, 4096, dtype=x.dtype, device="cuda")
        for _ in range(2):
            out.fill_(float("nan"))
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, want)
            assert torch.equal(m(x), want)                    # eager calls on the grown buffer
            m(big)                                            # (other routes share it)
    head_zero()


def test_adam_steps_then_prepare_state_dict_and_inference_mode():
    from _probe import launched_kernels, ran
    L = _layer("k65536_r256_fp16")
    m = _module(L).set_list_decode(True)
    m.prepare()
    x = _x(L, 3, seed=19)
    for p in (m.centroids.weight, m.res_centroids.weight, m.weight_scale, m.weight_bias):
        p.requires_grad_(True)
    opt = torch.optim.Adam([m.centroids.weight, m.res_centroids.weight, m.weight_scale, m.weight_bias], lr=1e-4,
                           eps=1e-3)                          # (fp16 parameters and state: eps must not flush to 0)
    m.set_quant_grad(True)
    for _ in range(2):
        opt.zero_grad()
        m(x).float().square().sum().backward()
        opt.step()
    m.set_quant_grad(False)
    m.prepare()
    with torch.no_grad():
        y = m(x)
        assert torch.isfinite(y).all() and not torch.equal(y, _run(_desc(L), x))     # (the step changed something)
        assert ran(launched_kernels(lambda: m(x)), KERNEL)
        f = _module(L).set_list_decode(True)
        f.load_state_dict(m.state_dict())
        assert torch.equal(f(x), y)                           # a fresh module with the updated tensors
    sd = {k: v.clone() for k, v in _module(L).state_dict().items()}
    m.load_state_dict(sd)
    with torch.no_grad():
        assert torch.equal(m(x), _run(_desc(L), x))           # reloaded: the original layer's bits again
    with torch.inference_mode():
        mi = _module(L).set_list_decode(True)
        yi = mi(x)
        assert ran(launched_kernels(lambda: mi(x)), KERNEL)
        assert torch.equal(yi, _run(_desc(L), x))
        mi.prepare(rebuild=True)
        assert torch.equal(mi(x), yi)
    head_zero()
