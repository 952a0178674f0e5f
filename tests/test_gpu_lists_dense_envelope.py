"""The dense weight from the index lists (lists_dense_kernel<T, TR, V> in csrc/lists_dense.cu and its GEMM glue
lists_gemm_launch in csrc/gemm_wgmma.cu) at the index data, shapes, layouts and values where a writer like it goes
wrong.  What tests/test_gpu_lists_dense.py and test_gpu_lists16_dense.py check on uniform indices is not repeated.

Bars:
* bit bar (shapes, index data): W from vptq_b200_lists_dequant is bit-identical to vptq_b200_dequant of the same
  descriptor, Wt to its transpose, both in sentinel-filled buffers whose padding columns must be zero and whose tail
  must be untouched; the input-gradient GEMM on the lists with dY = I is bit-identical to the packed one
  (`_lists_dense.check_weight`);
* exact bar (probes): x = e_f and dY = e_o give probe_expect(L, "direct") to the last bit (W has scale folded in, as on
  the prep-free prefill route; tests/test_lists_dense_envelope_host.py shows that this is the writer's arithmetic);
* fp64 bar (GEMM glue): |y - y*| <= TOL max|y*| against y* / dX* in fp64, plus bit identity with the packed prefill
  where the full descriptor takes its prep-free route and with the packed input gradient always;
* extremes: non-finite exactly where y* rounded to the layer type is, NaN as NaN, inf with the sign of y*, every
  other output bit-identical to the clean call (the contract of tests/test_gpu_extremes.py);
* anchor: lists_dequant against the reference CUDA kernels' recorded dequant samples, with the packed dequant's bound.

Every test asserts the kernels that ran (lists_dense_kernel, gemm_tn_wgmma where a GEMM is called, no dequant*) and
that the workspace head is zero afterwards.  fp16 and bf16 throughout unless a test says otherwise.
"""
import numpy as np
import pytest
import torch

import _extreme as ex
import _envelope as env
import vptq_oracle as vo
from _batch import head_zero
from _lists_dense import (DENSE, GEMM, SENTINEL, SM_COUNT, STAGE, DenseLayer, _bits, assert_route, check_weight,
                          deal_stats, dt_of)
from _probe import aligned_rows, launched_kernels, probe_expect, ran
from _util import TOL, parity_error
from vptq_b200 import lists

pytestmark = pytest.mark.gpu

DTYPES = ("fp16", "bf16")
WIDTHS = (4096, 4100, 9004, 65528, 65535)
NS_I = [(ns, I) for ns in (2, 4, 8, 16) for I in WIDTHS if ns * lists.geometry(I, 4096 * ns)[1] <= SM_COUNT]
OUTS = {8: (1, 3, 8, 9, 1003, 1004), 16: (8, 9, 15, 16, 17, 1000)}
SKEWED = ("ones", "row_slice", "constant", "ramp")


def _desc_of(L):
    from _batch import desc_of as desc8
    from _lists16 import desc_of as desc16
    return desc8(L) if L.vector_len == 8 else desc16(L)


# ---------------------------------------------------------------- 2. shapes (first: the cheapest cover of every path)
@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("ns,I", NS_I)
def test_shapes_slices_and_widths(ns, I, v):
    """NS slices x in_features up to 65535 (16 tiles, a last tile of 4095 columns), pitches min, +8, +16"""
    G = DenseLayer(v, I, 24 if v == 8 else 40, K=4096 * ns, seed=ns + I)
    for dtype in DTYPES:
        check_weight(G.desc(dtype), dt_of(dtype))
    head_zero()


@pytest.mark.parametrize("v,O", [(v, o) for v in OUTS for o in OUTS[v]])
def test_shapes_out_features(v, O):
    """out_features down to 1 and a partial last index row (at v = 16 a hi plane partly or wholly padding), with a
    ragged last tile (in_features 4100); every value is accepted by the layer and the descriptor"""
    from vptq_b200 import VQuantLinear
    VQuantLinear(4100, O, vector_lens=[-1, v], num_centroids=[-1, 65536], num_res_centroids=[-1, 256], group_num=1,
                 group_size=4100, outlier_size=0, indices_as_float=False, is_indice_packed=True, device="cuda",
                 dtype=torch.float16, enable_proxy_error=False)
    G = DenseLayer(v, 4100, O, seed=O)
    for dtype in DTYPES:
        check_weight(G.desc(dtype), dt_of(dtype))
    head_zero()


@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("perm,norm,bias", [(True, True, False), (False, True, True), (True, False, False),
                                            (False, False, True), (True, False, True)])
def test_shapes_perm_and_norm(perm, norm, bias, v):
    """perm and norm on and off (norm off with a bias): the weight, and the prefill against fp64 and, where the full
    descriptor takes its prep-free route (v = 8, in_features % 64 == 0), bit for bit"""
    from _gpu import x_to_t
    from vptq_b200 import native
    for dtype in DTYPES:
        L = vo.make_layer(in_features=2048, out_features=1000 if v == 16 else 1003, vector_len=v,
                          num_centroids=32768, num_res_centroids=64, enable_perm=perm, enable_norm=norm, bias=bias,
                          dtype=dtype, seed=70 + v)
        d = _desc_of(L)
        check_weight(d, dt_of(dtype))
        x = x_to_t(vo.make_x(200, L.in_features, dtype, seed=5), L)
        y = torch.empty(200, L.out_features, dtype=x.dtype, device="cuda")
        assert_route(launched_kernels(lambda: native.lists_quant_gemm(d, x, y)))
        # W itself is rounded to the layer type before the GEMM: in bf16 that rounding (2^-9 relative per weight) sits
        # beside the output's own, so the bar there is twice TOL; the bits are held by the packed route (v = 8) and
        # check_weight
        bar = TOL[dtype] * (2 if dtype == "bf16" else 1)
        assert parity_error(y.double().cpu().numpy(), ex.y_star(L, x).cpu().numpy()) <= bar
        if v == 8:
            y_p = torch.empty_like(y)
            assert not ran(launched_kernels(lambda: native.quant_gemm(d, x, y_p)), "prefill_prep_x")
            assert torch.equal(_bits(y), _bits(y_p))
    head_zero()


# ---------------------------------------------------------------- 1. index data
IDX_CASES = [(kind, res, Kr) for kind in env.PATTERNS for Kr in (0, 2, 256)
             for res in (("uniform", "ones") if Kr else ("uniform",))]


@pytest.mark.parametrize("K", [8192, 65536])
@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("kind,res,Kr", IDX_CASES)
def test_index_data(kind, res, Kr, v, K):
    """every index pattern of _envelope.PATTERNS with a uniform and an all-ones residual, Kr none, 2 and 256"""
    O = 4096 if v == 8 else 1024
    G = DenseLayer(v, 4096, O, K=K, Kr=Kr, kind=kind, res_kind=res, seed=K + Kr + v)
    for dtype in DTYPES:
        check_weight(G.desc(dtype), dt_of(dtype), lds=(8,))
    ns, nt, _ = lists.geometry(4096, K)
    st = deal_stats(G.lists()[1], ns, nt, G.Ro)
    print(f"lists {kind}/{res} Kr={Kr} v={v} K={K}: {st}")
    if kind in SKEWED:    # a unit of a whole tile's steps next to 1-step empty units
        assert st["longest"] >= 64 and st["empty"] > 0, st
    head_zero()


# ---------------------------------------------------------------- 3. probes
PROBE = {8: dict(in_features=1024, out_features=264), 16: dict(in_features=1024, out_features=272)}


def _no_neg_zero(t):
    """the GEMM's fp32 accumulator starts at +0: a -0 weight comes out as +0"""
    return torch.where(t == 0, torch.zeros_like(t), t)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["uniform", "zipf_hot0"])
@pytest.mark.parametrize("v", [8, 16])
def test_probes(v, kind, dtype):
    """x = e_f for every feature f (one call of in_features tokens) and dY = e_o for every output o, bit for bit"""
    from vptq_b200 import native
    L = env.layer_with(kind, vector_len=v, num_centroids=65536, num_res_centroids=256, bias=True, dtype=dtype,
                       seed=300 + v, **PROBE[v])
    P = ex.copy_layer(L)
    P.bias = None
    d = _desc_of(L)
    dt = dt_of(dtype)
    I, O = L.in_features, L.out_features
    want = torch.from_numpy(probe_expect(L, "direct")).cuda().to(dt)                   # [I, O]
    want_t = _no_neg_zero(torch.from_numpy(probe_expect(P, "direct")).cuda().to(dt).t().contiguous())   # [O, I]
    x, dy = torch.eye(I, dtype=dt, device="cuda"), torch.eye(O, dtype=dt, device="cuda")
    y, dx = torch.empty(I, O, dtype=dt, device="cuda"), torch.empty(O, I, dtype=dt, device="cuda")

    def calls():
        native.lists_quant_gemm(d, x, y)
        native.lists_quant_gemm(d, dy, dx, native.FLAG_TRANSPOSE)
    assert_route(launched_kernels(calls))
    for got, exp in ((y, want), (dx, want_t)):
        bad = (_bits(got) != _bits(exp)).nonzero()
        assert bad.numel() == 0, (bad.shape[0], bad[:8].tolist())
    head_zero()


# ---------------------------------------------------------------- 4. GEMM glue
GLUE_SHAPES = {"aligned": (1024, 1024), "ragged": (1000, 1004)}    # ragged: in_features, out_features % 64 != 0
LAYOUTS = [("aligned", "aligned"), ("odd", "aligned"), ("off2", "aligned"), ("aligned", "odd"), ("aligned", "off2"),
           ("aligned", "guard")]
TOKENS = (1, 2, 3, 127, 128, 129, 300, 4400)    # 4400 tokens: 35 x 4 = 140 tiles of 128 x 256 > 132 SMs


def _rows(n, cols, dt, layout, fill=None):
    """[n, cols] view: aligned (pitch cols rounded up to 8), odd pitch, base 2 bytes off, or inside a sentinel buffer
    with a guard row on either side.  Returns (view, buffer, guard check)."""
    pitch = (cols + 7) // 8 * 8
    if layout == "odd":
        pitch = cols + 1 if cols % 2 == 0 else cols
    if layout == "guard":
        buf = torch.full(((n + 2) * pitch,), SENTINEL, dtype=torch.int16, device="cuda")
        view = buf.view(dt).as_strided((n, cols), (pitch, 1), pitch)

        def guard():
            b = buf.view(n + 2, pitch)
            assert bool((b[0] == SENTINEL).all() and (b[-1] == SENTINEL).all() and (b[1:-1, cols:] == SENTINEL).all())
        return view, guard
    view = aligned_rows(n, cols, dt, pitch=pitch, offset=1 if layout == "off2" else 0)
    if fill is not None:
        view.copy_(fill)
    return view, lambda: None


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("xl,yl", LAYOUTS)
@pytest.mark.parametrize("shape", sorted(GLUE_SHAPES))
@pytest.mark.parametrize("v", [8, 16])
def test_gemm_glue(v, shape, xl, yl, dtype):
    from vptq_b200 import native
    I, O = GLUE_SHAPES[shape]
    L = vo.make_layer(in_features=I, out_features=O, vector_len=v, num_centroids=65536, num_res_centroids=256,
                      bias=True, dtype=dtype, seed=90 + v)
    d = _desc_of(L)
    dt = dt_of(dtype)
    W64 = torch.from_numpy(ex.dense64(L)).cuda()
    for tokens in TOKENS:
        g = torch.Generator(device="cuda").manual_seed(tokens)
        xv = torch.randn(tokens, I, device="cuda", generator=g).to(dt)
        dyv = torch.randn(tokens, O, device="cuda", generator=g).to(dt)
        for tr, a_val, n_in, n_out in ((0, xv, I, O), (native.FLAG_TRANSPOSE, dyv, O, I)):
            a, _ = _rows(tokens, n_in, dt, xl, fill=a_val)
            out, guard = _rows(tokens, n_out, dt, yl)
            names = launched_kernels(lambda: native.lists_quant_gemm(d, a, out, tr))
            assert_route(names)
            pitch = native.row_pitch(a)
            assert ran(names, STAGE) == bool(n_in % 64 or a.data_ptr() % 16 or pitch % 8), (names, tokens, tr)
            guard()
            star = ex.dgrad_star(L, a_val, W64) if tr else ex.y_star(L, a_val, W64)
            assert parity_error(out.double().cpu().numpy(), star.cpu().numpy()) <= TOL[dtype], (tokens, tr)
            ref = torch.empty(tokens, n_out, dtype=dt, device="cuda")
            if tr:                                  # the input gradient: the same Wt and GEMM as the packed route
                native.quant_gemm_dgrad(d, a, ref)
                assert torch.equal(_bits(out), _bits(ref)), tokens
            elif v == 8 and I % 64 == 0 and a.data_ptr() % 16 == 0 and pitch % 8 == 0:
                # the full descriptor's prep-free prefill: the same W, the same GEMM
                assert not ran(launched_kernels(lambda: native.quant_gemm(d, a, ref)), "prefill_prep_x")
                assert torch.equal(_bits(out), _bits(ref)), tokens
    head_zero()


# ---------------------------------------------------------------- 5. extremes
EXT = {8: dict(in_features=1024, out_features=264), 16: dict(in_features=1024, out_features=272)}


def _ext_layer(v, dtype):
    return vo.make_layer(vector_len=v, num_centroids=65536, num_res_centroids=256, bias=True, dtype=dtype,
                         seed=500 + v, **EXT[v])


def _both(L, x, dy):
    """(y, dX) from the lists for x and dY, with the kernels that ran asserted"""
    from vptq_b200 import native
    d = _desc_of(L)
    y = torch.empty(x.shape[0], L.out_features, dtype=x.dtype, device="cuda")
    dx = torch.empty(dy.shape[0], L.in_features, dtype=x.dtype, device="cuda")

    def calls():
        native.lists_quant_gemm(d, x, y)
        native.lists_quant_gemm(d, dy, dx, native.FLAG_TRANSPOSE)
    assert_route(launched_kernels(calls))
    return y, dx


def _contract(got, clean, star, dt):
    """non-finite exactly where y* rounded to dt is, NaN as NaN, inf with the sign of y*; the rest as the clean call"""
    want = ex.classify(star.to(dt))
    assert torch.equal(ex.classify(got), want), int((ex.classify(got) != want).sum())
    fin = want == ex.FINITE
    assert torch.equal(_bits(got)[fin], _bits(clean)[fin])
    return int((~fin).sum())


def _inputs(L, tokens=16):
    from _gpu import x_to_t
    return (x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=1), L),
            x_to_t(vo.make_x(tokens, L.out_features, L.dtype, seed=2), L))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("value", sorted(ex.VALUES))
@pytest.mark.parametrize("v,plane", [(8, "lo"), (16, "lo"), (16, "hi")])
def test_extremes_in_the_residual_codebook(v, plane, value, dtype):
    """inf / NaN in one element of a residual entry each listed index row uses once (v = 16: lo and hi plane)"""
    L = ex.isolate(_ext_layer(v, dtype), res={7: [1, 5, 9]})
    x, dy = _inputs(L)
    clean = _both(L, x, dy)
    e = 3 if plane == "lo" else 11
    B = ex.inject(L, "R", ex.VALUES[value], k=7, e=e)
    got = _both(B, x, dy)
    W64 = torch.from_numpy(ex.dense64(B)).cuda()
    n = _contract(got[0], clean[0], ex.y_star(B, x, W64), dt_of(dtype))
    n += _contract(got[1], clean[1], ex.dgrad_star(B, dy, W64), dt_of(dtype))
    assert n >= 3 * 16 * 2
    head_zero()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("value", sorted(ex.VALUES))
@pytest.mark.parametrize("site", ["dY", "scale_last", "wbias_last", "bias_last"])
@pytest.mark.parametrize("v", [8, 16])
def test_extremes_in_dy_and_the_last_entries(v, site, value, dtype):
    """inf / NaN in dY (input gradient), in weight_scale / weight_bias of the last feature (the last tile's ragged end
    at in_features 1004) and in the bias of the last output"""
    L = vo.make_layer(vector_len=v, num_centroids=65536, num_res_centroids=256, bias=True, dtype=dtype, seed=600 + v,
                      in_features=1004, out_features=264 if v == 8 else 272)
    x, dy = _inputs(L)
    clean = _both(L, x, dy)
    B, dyb = L, dy.clone()
    if site == "dY":
        dyb[3, 17] = ex.VALUES[value]
        dyb[9, L.out_features - 1] = ex.VALUES[value]
    else:
        kind = site.split("_")[0]
        B = ex.inject(L, kind, ex.VALUES[value], f=L.in_features - 1, o=L.out_features - 1)
    got = _both(B, x, dyb)
    W64 = torch.from_numpy(ex.dense64(B)).cuda()
    n = _contract(got[0], clean[0], ex.y_star(B, x, W64), dt_of(dtype))
    n += _contract(got[1], clean[1], ex.dgrad_star(B, dyb, W64), dt_of(dtype))
    assert n > 0
    head_zero()


@pytest.mark.parametrize("v", [8, 16])
def test_fp16_outputs_past_65504(v):
    """fp16 only, no bias, weight_scale times 8: one token of x (of dY) scaled by 2^13 takes outputs past 65504.
    Those are inf with the sign of y*; the token's finite outputs are the clean ones times 2^13 (forward bit for bit,
    the input gradient within 1 ulp: the tensor cores' fp32 accumulation moves a few cancelling sums, as on the
    packed route, tests/test_gpu_extremes.py); the other tokens keep their bits"""
    from _probe import ulp_diff
    L = vo.make_layer(vector_len=v, num_centroids=65536, num_res_centroids=256, dtype="fp16", seed=500 + v, **EXT[v])
    L.weight_scale = (L.weight_scale.astype(np.float32) * 8).astype(np.float16)
    x, dy = _inputs(L)
    clean = _both(L, x, dy)
    xs, dys = x.clone(), dy.clone()
    xs[5] *= 8192
    dys[5] *= 8192
    assert bool(torch.isfinite(xs).all() and torch.isfinite(dys).all())
    got = _both(L, xs, dys)
    W64 = torch.from_numpy(ex.dense64(L)).cuda()
    for g, c, star, ulps in ((got[0], clean[0], ex.y_star(L, xs, W64), 0),
                             (got[1], clean[1], ex.dgrad_star(L, dys, W64), 1)):
        s = star[5]
        near = (s.abs() > 65504 * 0.99) & (s.abs() < 65520 * 1.01)     # where fp32 rounding may fall either side
        want = ex.classify(s.half())
        assert bool((want != ex.FINITE).any()) and bool((want == ex.FINITE).any())
        got5 = ex.classify(g[5])
        assert torch.equal(got5[~near], want[~near])
        assert bool((g[5][near].float().abs() >= 64000).all()) and torch.equal(g[5][near].sign(), s[near].sign().half())
        fin = (got5 == ex.FINITE) & (c[5].float().abs() >= 2.0 ** -14)     # normal values scale exactly
        assert int(ulp_diff(g[5][fin], (c[5][fin].float() * 8192).half()).max()) <= ulps
        rest = torch.ones(g.shape[0], dtype=torch.bool, device="cuda")
        rest[5] = False
        assert torch.equal(_bits(g[rest]), _bits(c[rest]))
    head_zero()


# ---------------------------------------------------------------- 6. anchor against the reference CUDA kernels
ANCHOR = [("outputs.npz", "llama3_k65536_r256"), ("outputs.npz", "bf16"), ("v16.npz", "v16_k65536_r256"),
          ("v16.npz", "v16_k65536_r256_bf16")]


@pytest.mark.parametrize("fixture,name", ANCHOR)
def test_lists_dequant_matches_reference_cuda(fixture, name):
    """the list-eligible dequant cases of test_gpu_vs_ref_cuda.py with the bound the packed dequant meets there"""
    import os
    from _util import GOLDEN_DIR
    from test_gpu_vs_ref_cuda import CASES, DEQUANT_SEED, V16_CASES, from_bits, sample_positions
    from vptq_b200 import native
    ref = np.load(os.path.join(GOLDEN_DIR, "ref_cuda", fixture), allow_pickle=False)
    L = vo.make_layer(seed=DEQUANT_SEED, **dict(CASES, **V16_CASES)[name])
    d = _desc_of(L)
    w = torch.empty(L.out_features, L.in_features, dtype=dt_of(L.dtype), device="cuda")
    assert_route(launched_kernels(lambda: native.lists_dequant(d, w, L.in_features)), gemm=False)
    W = w.float().cpu().numpy()
    assert W.shape == tuple(ref[f"dequant__{name}__shape"])
    W = W.reshape(-1)[sample_positions(W.size)]
    W_ref = from_bits(ref[f"dequant__{name}__values"], L.dtype)
    ulp = 2.0 ** -10 if L.dtype == "fp16" else 2.0 ** -7
    bound = 2 * ulp * (np.abs(W_ref) + np.abs(vo.to_f32(L.weight_bias, L.dtype)).max()) + 1e-7
    bad = np.abs(W - W_ref) > bound
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} sampled elements beyond the double-rounding bound"
    head_zero()


# ---------------------------------------------------------------- 7. lifecycle
def _ops(L, d, dec):
    """name -> (callable writing into its own output, output): the list routes and every other op on one layer"""
    from vptq_b200 import native
    from _gpu import x_to_t
    dt = dt_of(L.dtype)
    I, O = L.in_features, L.out_features
    x = x_to_t(vo.make_x(300, I, L.dtype, seed=1), L)
    dy = x_to_t(vo.make_x(300, O, L.dtype, seed=2), L)
    x1 = x[:1].clone()
    out = {}

    def add(name, shape, fn):
        buf = torch.empty(shape, dtype=dt, device="cuda")
        out[name] = (lambda: fn(buf), buf)
    add("lists_gemm", (300, O), lambda y: native.lists_quant_gemm(dec, x, y))
    add("lists_gemm_t", (300, I), lambda y: native.lists_quant_gemm(dec, dy, y, native.FLAG_TRANSPOSE))
    add("lists_dequant", (O, I), lambda w: native.lists_dequant(dec, w, I))
    add("lists_dequant_t", (I, O), lambda w: native.lists_dequant(dec, w, O, native.FLAG_TRANSPOSE))
    add("gemm", (300, O), lambda y: native.quant_gemm(d, x, y))
    add("dgrad", (300, I), lambda y: native.quant_gemm_dgrad(d, dy, y))
    add("dequant", (O, I), lambda w: native.dequant(d, w))
    if L.vector_len == 8:
        add("list_decode", (1, O), lambda y: native.quant_gemv(dec, x1, y))
        add("batch_decode", (4, O), lambda y: native.quant_gemv_batch(dec, x[:4], y))
        add("wgrad", (1, L.centroids.size), lambda g: native.quant_gemm_wgrad(d, x, dy, {"centroids": g}))
    else:
        add("list_decode", (1, O), lambda y: native.quant_gemv_lists16(dec, x1, y))
    return out


def _decode_only(L):
    """decode-only descriptor (packed words forgotten) of oracle layer L, its tensors kept on it"""
    from _lists16 import tensors_of
    from vptq_b200 import native
    t = tensors_of(L)
    d = native.make_desc(dtype=dt_of(L.dtype), in_features=L.in_features, out_features=L.out_features,
                         vector_len=L.vector_len, num_centroids=L.num_centroids,
                         num_res_centroids=L.num_res_centroids, num_codebooks=1, group_size=L.in_features,
                         outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1, outlier_indices=None,
                         outlier_centroids=None, lists=True, lists16=True, lists_prefill=True, drop_packed=True, **t)
    d._tensors = t
    assert not d.indices and d.lists_stream
    return d


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("v", [8, 16])
def test_lifecycle_interleaved_and_graph(v, dtype):
    """the list routes interleaved with every other op on one stream's workspace, then a graph of a decode-only
    prefill (both GEMMs and the dequant) captured on torch's capture stream after eager workspace growth: each output
    bit-identical to the op run alone on a fresh stream"""
    from _gpu import x_to_t
    from vptq_b200 import native
    L = vo.make_layer(in_features=1024, out_features=1000, vector_len=v, num_centroids=65536, num_res_centroids=256,
                      bias=True, dtype=dtype, seed=800 + v)
    d, dec = _desc_of(L), _decode_only(L)
    alone = {}
    torch.cuda.synchronize()
    for name, (fn, buf) in _ops(L, d, dec).items():
        with torch.cuda.stream(torch.cuda.Stream()):
            buf.fill_(float("nan"))
            fn()
        torch.cuda.synchronize()
        alone[name] = buf.clone()
    ops = _ops(L, d, dec)
    order = list(ops) + list(reversed(ops))
    names = launched_kernels(lambda: [ops[n][0]() for n in order])
    assert ran(names, DENSE) and ran(names, GEMM)
    for name, (_, buf) in ops.items():
        assert torch.equal(_bits(buf), _bits(alone[name])), name
    head_zero()
    # the graph: eager growth first, then capture, then replay into zeroed outputs
    native.lists_quant_gemm(dec, x_to_t(vo.make_x(2048, L.in_features, dtype, seed=3), L),
                            torch.empty(2048, L.out_features, dtype=dt_of(dtype), device="cuda"))
    graph_ops = {n: ops[n] for n in ("lists_gemm", "lists_gemm_t", "lists_dequant")}
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for fn, _ in graph_ops.values():
            fn()
    for _, buf in graph_ops.values():
        buf.zero_()
    g.replay()
    torch.cuda.synchronize()
    for name, (_, buf) in graph_ops.items():
        assert torch.equal(_bits(buf), _bits(alone[name])), name
    head_zero()
