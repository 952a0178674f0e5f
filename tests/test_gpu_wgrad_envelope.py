"""The weight gradients (vptq_b200_quant_gemm_wgrad on the fused and the generic route, vptq_b200_dequant_backward) bit
for bit against the exact mirror of their fixed-point reduction (tests/_wgrad_exact.py), at the shapes, index data,
values and layouts where a reduction like it goes wrong.  tests/test_gpu_wgrad.py (probes, fp64 parity) is not
repeated.

Bar: every element of every requested gradient equals the mirror's bits.  G is exact where the mirror is used:
dequant() backward takes the caller's 16-bit gradient, and quant_gemm backward gets integer x and dY with |.| <= 4, so
every partial sum of dY^T x is an integer below 2^24 and the fp32 GEMM forms it exactly.  Power-of-two scaling
(random non-integer inputs) is checked against the unscaled call instead.

Every test asserts the kernels that ran, runs quant_gemm backward on the fused route and with GRAD_FLAG_GENERIC (same
bits required), and leaves the workspace head zero.  fp16 and bf16 unless a test says otherwise.
"""
import numpy as np
import pytest
import torch

import _envelope as env
import _wgrad_exact as wx
import vptq_oracle as vo
from _batch import head_zero
from _probe import aligned_rows, launched_kernels, ran

pytestmark = pytest.mark.gpu

DTYPES = ("fp16", "bf16")
WGRAD_KERNELS = ("wg_row_stats", "wg_transpose", "gemm_tn_wgmma", "wg_units", "wg_finish")
DQB_KERNELS = ("wg_row_stats", "wg_units", "wg_scatter", "wg_finish")


# ---------------------------------------------------------------- helpers
def _tdt(dtype):
    return torch.float16 if dtype == "fp16" else torch.bfloat16


def _fused(L):
    return L.vector_len == 8 and L.num_codebooks == 1 and not L.enable_outlier and L.num_res_centroids <= 256


def _desc(L, scale_q=True):
    """the module's descriptor (its tensors stay alive with the module); scale_q=False drops the quantised-order copy
    of weight_scale, so the fused epilogue gathers the scale through perm"""
    from _gpu import make_module
    m = make_module(L)
    m.prepare()
    d = m._desc_cache[0]
    if not scale_q:
        assert d.weight_scale_q
        d.weight_scale_q = None
    d._module = m
    return d


def _outs(L, names=None):
    I, G = L.in_features, L.num_codebooks
    shapes = {"centroids": (G, L.num_centroids * L.vector_len)}
    if L.res_bits:
        shapes["res_centroids"] = (G, L.num_res_centroids * L.vector_len)
    if L.enable_outlier:
        shapes["outlier_centroids"] = (1, L.num_outlier_centroids * L.outlier_vector_len)
    if L.weight_scale is not None:
        shapes["weight_scale"] = shapes["weight_bias"] = (I,)
    return {n: torch.full(s, float("nan"), dtype=_tdt(L.dtype), device="cuda") for n, s in shapes.items()
            if names is None or n in names}


def _bits(t):
    return t.detach().contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def wgrad(d, L, x, dy, generic=False, names=None, check_route=False):
    from vptq_b200 import native
    outs = _outs(L, names)
    fn = lambda: native.quant_gemm_wgrad(d, x, dy, outs, flags=native.GRAD_FLAG_GENERIC if generic else 0)
    if check_route:
        k = launched_kernels(fn)
        assert all(ran(k, n) for n in WGRAD_KERNELS), k
        assert ran(k, "wg_scatter") == (generic or not _fused(L)), k
    else:
        fn()
    torch.cuda.synchronize()
    return {n: _bits(t) for n, t in outs.items()}


def dqb(d, L, gamma, names=None, check_route=False):
    from vptq_b200 import native
    outs = _outs(L, names)
    fn = lambda: native.dequant_backward(d, gamma, outs)
    if check_route:
        k = launched_kernels(fn)
        assert all(ran(k, n) for n in DQB_KERNELS) and not ran(k, "gemm_tn_wgmma"), k
    else:
        fn()
    torch.cuda.synchronize()
    return {n: _bits(t) for n, t in outs.items()}


def assert_bits(got, want, what):
    assert sorted(got) == sorted(want), what
    for n, w in want.items():
        g = got[n].reshape(w.shape)
        bad = np.argwhere(g != w)
        assert bad.size == 0, (f"{what} {n}: {len(bad)} of {g.size} elements differ, first at {bad[0].tolist()}: "
                               f"{int(g[tuple(bad[0])]):#06x} != {int(w[tuple(bad[0])]):#06x}")


def ints(T, n, dtype, seed, lo=-4, hi=4):
    """integer inputs (exact in both 16-bit types), as a cuda tensor"""
    a = np.random.default_rng(seed).integers(lo, hi + 1, size=(T, n)).astype(np.float32)
    return torch.from_numpy(a).to("cuda", _tdt(dtype))


def f64(t):
    return t.double().cpu().numpy()


def both_routes(d, L, x, dy, what, backend="numpy", names=None, route=True):
    """quant_gemm backward on the fused route and with GRAD_FLAG_GENERIC: the same bits, equal to the mirror"""
    want = (wx.quant_gemm_wgrad(f64(x), f64(dy), L, backend="numpy", want=names or wx.NAMES)[0] if backend == "numpy"
            else wx.quant_gemm_wgrad(x, dy, L, backend="torch", want=names or wx.NAMES)[0])
    a = wgrad(d, L, x, dy, names=names, check_route=route)
    assert_bits(a, want, what + " (fused)" if _fused(L) else what)
    if _fused(L):
        b = wgrad(d, L, x, dy, generic=True, names=names, check_route=route)
        assert_bits(b, want, what + " (generic)")
    return a


def random16(shape, dtype, seed, lo=-20, hi=6):
    """random 16-bit values of any magnitude: sign * mantissa * 2^uniform(lo, hi), rounded to the type"""
    rng = np.random.default_rng(seed)
    a = (rng.choice([-1.0, 1.0], shape) * rng.uniform(1, 2, shape) * 2.0 ** rng.integers(lo, hi, shape))
    a[rng.random(shape) < 0.05] = 0.0
    t = torch.from_numpy(a.astype(np.float32)).to("cuda", _tdt(dtype))
    return t


# ---------------------------------------------------------------- tiles and tokens (fused route, v = 8)
# (O, I, tokens, perm, norm, Kr): 128-row tiles over O, 256-column tiles over I, K = tokens rounded up to 64; the
# last four have more than 132 tiles, so each persistent CTA works several before its single dR flush
TILES = [(8, 64, 1, True, True, 256), (120, 256, 63, False, True, 2), (128, 264, 64, True, False, -1),
         (136, 4100, 65, False, False, 256), (1004, 256, 128, True, True, 2), (1004, 4100, 129, True, True, 256),
         (128, 64, 2048, False, True, 256), (136, 14336, 1, True, True, -1), (4096, 264, 2048, True, True, 256),
         (4096, 4096, 65, True, True, 256), (14336, 4096, 64, False, True, 2), (4096, 14336, 129, True, False, 256)]


@pytest.mark.parametrize("O,I,T,perm,norm,Kr", TILES)
def test_tiles_and_tokens(O, I, T, perm, norm, Kr):
    for dtype in DTYPES:
        L = vo.make_layer(in_features=I, out_features=O, vector_len=8, num_centroids=4096, num_res_centroids=Kr,
                          enable_perm=perm, enable_norm=norm, dtype=dtype, seed=O + I + T)
        d = _desc(L)
        x, dy = ints(T, I, dtype, 1), ints(T, O, dtype, 2)
        both_routes(d, L, x, dy, f"{O}x{I} T={T} {dtype}", backend="torch", route=dtype == "fp16")
    head_zero()


def test_scale_gathered_through_perm_without_the_quantised_copy():
    """a descriptor without weight_scale_q: the fused epilogue reads weight_scale[perm[c]]"""
    for dtype in DTYPES:
        L = vo.make_layer(in_features=1024, out_features=264, vector_len=8, num_centroids=4096, num_res_centroids=256,
                          dtype=dtype, seed=8)
        d = _desc(L, scale_q=False)
        both_routes(d, L, ints(65, 1024, dtype, 3), ints(65, 264, dtype, 4), f"no scale_q {dtype}", backend="torch")
    head_zero()


# ---------------------------------------------------------------- scatter / dequant backward (generic route)
def _scatter_layer(v, I, O, groups=1, outl=False, Kr=16, dtype="fp16", seed=0):
    kw = dict(outlier_size=4 * groups if outl else 0, outlier_vector_len=4 if outl else -1,
              num_outlier_centroids=64 if outl else -1)
    S = kw["outlier_size"]
    return vo.make_layer(in_features=I + S, out_features=O, vector_len=v, num_centroids=256, num_res_centroids=Kr,
                         num_codebooks=groups, dtype=dtype, seed=seed, **kw)


SCATTER = ([(v, 256, 16 * v, 1, False) for v in (2, 4, 6, 8, 10, 12, 16)]
           + [(8, 255, 17 * 8, 1, False), (8, 257, 8, 1, False), (6, 4100, 17 * 6 - 2, 1, False),
              (4, 256, 16 * 4, 2, False), (12, 256, 12 * 17, 4, True), (16, 4100, 16, 2, True), (2, 256, 2, 4, True),
              (10, 257, 10 * 16 + 3, 1, True)])


@pytest.mark.parametrize("v,I,O,groups,outl", SCATTER)
def test_scatter_and_dequant_backward(v, I, O, groups, outl):
    """v = 2..16, 1 / 2 / 4 groups, outliers with vol = 4; ragged edges of the 256-column x 16-row CTA (I = 255, 256,
    257, 4100; Ro = 16, 17, 1); random 16-bit gamma of any magnitude"""
    for dtype in DTYPES:
        L = _scatter_layer(v, I, O, groups, outl, dtype=dtype, seed=v + I + O)
        d = _desc(L)
        gamma = random16((L.out_features, L.in_features), dtype, seed=v + groups)
        assert_bits(dqb(d, L, gamma, check_route=dtype == "fp16"), wx.dequant_backward(f64(gamma), L)[0],
                    f"dequant backward v={v} {I}x{O} G={groups} {dtype}")
        both_routes(d, L, ints(70, L.in_features, dtype, 5), ints(70, O, dtype, 6), f"wgrad v={v} {dtype}",
                    route=dtype == "fp16")
    head_zero()


# ---------------------------------------------------------------- cut-offs
@pytest.mark.parametrize("v,Kr,table", [(8, 256, "fused"), (8, 512, "shared"), (8, 1024, "global"),
                                        (16, 256, "shared"), (16, 512, "global")])
def test_cut_offs(v, Kr, table):
    """fused route up to Kr = 256 (a 16 KiB dR table), generic above; the scatter's shared dR table up to
    G Kr v 8 = 32 KiB, global atomics above"""
    for dtype in DTYPES:
        L = vo.make_layer(in_features=512, out_features=16 * v * 3, vector_len=v, num_centroids=4096,
                          num_res_centroids=Kr, dtype=dtype, seed=Kr + v)
        assert _fused(L) == (table == "fused")
        if table != "fused":
            assert (Kr * v * 8 <= 32 * 1024) == (table == "shared")
        d = _desc(L)
        gamma = random16((L.out_features, 512), dtype, seed=Kr)
        assert_bits(dqb(d, L, gamma, check_route=True), wx.dequant_backward(f64(gamma), L)[0], f"dqb Kr={Kr}")
        both_routes(d, L, ints(129, 512, dtype, 7), ints(129, L.out_features, dtype, 8), f"Kr={Kr} {dtype}")
    head_zero()


# ---------------------------------------------------------------- index data
IDX = [(kind, res) for kind in env.PATTERNS for res in ("uniform", "ones")]


@pytest.mark.parametrize("kind,res", IDX)
def test_index_patterns_fused(kind, res):
    """every skewed pattern of tests/_envelope.py with a uniform and an all-ones residual (K 65536, Kr 256)"""
    for dtype in DTYPES:
        L = env.layer_with(kind, res, in_features=4096, out_features=264, vector_len=8, num_centroids=65536,
                           num_res_centroids=256, dtype=dtype, seed=3)
        d = _desc(L)
        both_routes(d, L, ints(65, 4096, dtype, 9), ints(65, 264, dtype, 10), f"{kind}/{res} {dtype}",
                    backend="torch", route=dtype == "fp16")
        gamma = random16((264, 4096), dtype, seed=11)
        assert_bits(dqb(d, L, gamma), wx.dequant_backward(gamma.double(), L, backend="torch")[0], f"{kind} dqb")
    head_zero()


@pytest.mark.parametrize("b", [1, 8, 17, 24, 32])
def test_index_widths_generic(b):
    K, Kr = env._width_pair(b)
    for dtype in DTYPES:
        L = env.layer_with("uniform", in_features=256, out_features=48, vector_len=8, num_centroids=K,
                           num_res_centroids=Kr, dtype=dtype, seed=b)
        d = _desc(L)
        gamma = random16((48, 256), dtype, seed=b)
        assert_bits(dqb(d, L, gamma, check_route=True), wx.dequant_backward(f64(gamma), L)[0], f"b={b} dqb")
        x, dy = ints(33, 256, dtype, 12), ints(33, 48, dtype, 13)
        want = wx.quant_gemm_wgrad(f64(x), f64(dy), L)[0]
        assert_bits(wgrad(d, L, x, dy, generic=True, check_route=True), want, f"b={b} generic")
        if _fused(L):
            assert_bits(wgrad(d, L, x, dy), want, f"b={b} fused")
    head_zero()


def test_all_ones_indices_fill_one_entry_to_the_headroom():
    """every term positive on one dC entry: its sum is within a factor of two of B, i.e. between 2^60 and 2^61 units"""
    for dtype in DTYPES:
        L = env.layer_with("ones", in_features=4096, out_features=1024, vector_len=8, num_centroids=65536,
                           num_res_centroids=256, dtype=dtype, seed=4)
        L.weight_scale = np.abs(vo.to_f32(L.weight_scale, dtype)).astype(np.float16) if dtype == "fp16" else \
            L.weight_scale & np.uint16(0x7FFF)
        d = _desc(L)
        x = ints(129, 4096, dtype, 14, lo=1)
        dy = ints(129, 1024, dtype, 15, lo=1)
        dy[:, torch.arange(1024, device="cuda") % 8 != 0] = 0           # every output with e = 0
        bits, sums, es = wx.quant_gemm_wgrad(x, dy, L, backend="torch")
        top = int(sums["centroids"].max())
        assert 1 << 60 <= top < 1 << 61 and top == sums["centroids"][0, (65536 - 1) * 8], top
        got = both_routes(d, L, x, dy, f"all ones {dtype}", backend="torch")
        assert got["centroids"][0, (65536 - 1) * 8] == bits["centroids"][0, (65536 - 1) * 8]
    head_zero()


# ---------------------------------------------------------------- Llama shapes
LLAMA = [(4096, 4096), (14336, 4096), (4096, 14336)]        # (out_features, in_features)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("O,I", LLAMA)
def test_llama_shapes_bit_exact(O, I, dtype):
    L = vo.make_layer(in_features=I, out_features=O, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      dtype=dtype, seed=45)
    d = _desc(L)
    T = 8192 if (O, I, dtype) == (4096, 4096, "fp16") else 2048
    both_routes(d, L, ints(T, I, dtype, 16), ints(T, O, dtype, 17), f"llama {O}x{I} T={T} {dtype}", backend="torch")
    head_zero()


def _in_normal_range(f, dtype):
    p, emin, emax, _ = wx.FORMAT[dtype]
    top = (2 - 2.0 ** (1 - p)) * 2.0 ** emax
    return (f == 0) | ((f.abs() >= 2.0 ** emin) & (f.abs() <= top))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("O,I", LLAMA)
def test_power_of_two_scaling(O, I, dtype):
    """random non-integer inputs: dY 2^k and x 2^k (k = -8, +4) scale every gradient by 2^k bit for bit, except where
    a result leaves the type's normal range (the unit scales with the bound)"""
    from vptq_b200 import native
    L = vo.make_layer(in_features=I, out_features=O, vector_len=8, num_centroids=65536, num_res_centroids=256,
                      dtype=dtype, seed=46)
    d = _desc(L)
    gen = torch.Generator(device="cuda").manual_seed(O + I)

    def inputs(n):                     # |v| >= 2^-5: v 2^-8 stays a normal fp16 value, so the scaled input is exact
        t = torch.randn(2048, n, device="cuda", generator=gen)
        return torch.where(t.abs() < 2.0 ** -5, torch.full_like(t, 2.0 ** -5), t).to(_tdt(dtype))

    x, dy = inputs(I), inputs(O)

    def run(xx, yy, generic=False):
        outs = _outs(L)
        native.quant_gemm_wgrad(d, xx, yy, outs, flags=native.GRAD_FLAG_GENERIC if generic else 0)
        return outs

    base = run(x, dy)
    gen_base = run(x, dy, generic=True)
    for k in (-8, 4):
        for which in ("dy", "x"):
            xx, yy = (x, dy * 2.0 ** k) if which == "dy" else (x * 2.0 ** k, dy)
            assert torch.equal((yy if which == "dy" else xx).double(), (dy if which == "dy" else x).double() * 2.0 ** k)
            got = run(xx, yy)
            for n, g in got.items():
                b = base[n].double()
                ok = _in_normal_range(b, dtype) & _in_normal_range(b * 2.0 ** k, dtype)
                assert ok.any(), n
                gg = g.double()
                assert torch.equal(gg[ok], b[ok] * 2.0 ** k), f"{O}x{I} {dtype} {which}*2^{k} {n}"
    for n in base:
        assert torch.equal(_bits_t(base[n]), _bits_t(gen_base[n])), n
    head_zero()


def _bits_t(t):
    return t.contiguous().view(torch.int16)


# ---------------------------------------------------------------- layouts
@pytest.mark.parametrize("dtype", DTYPES)
def test_odd_pitch_and_misaligned_inputs(dtype):
    """x and dY with an odd row pitch and 2 bytes off alignment give the contiguous call's bits"""
    L = vo.make_layer(in_features=1000, out_features=264, vector_len=8, num_centroids=4096, num_res_centroids=256,
                      dtype=dtype, seed=47)
    d = _desc(L)
    x, dy = ints(77, 1000, dtype, 18), ints(77, 264, dtype, 19)
    want = wx.quant_gemm_wgrad(f64(x), f64(dy), L)[0]
    for pitch_x, pitch_y, off in ((1001, 265, 1), (1003, 267, 0), (1000, 264, 1)):
        xs = aligned_rows(77, 1000, x.dtype, pitch=pitch_x, offset=off)
        ys = aligned_rows(77, 264, x.dtype, pitch=pitch_y, offset=off)
        xs.copy_(x)
        ys.copy_(dy)
        assert xs.stride(0) == pitch_x and (xs.data_ptr() % 4 == 2) == (off == 1)
        for generic in (False, True):
            assert_bits(wgrad(d, L, xs, ys, generic=generic, check_route=off == 1), want,
                        f"pitch {pitch_x}/{pitch_y} offset {off} generic={generic}")
    head_zero()


# ---------------------------------------------------------------- rounding probes
@pytest.mark.parametrize("dtype", DTYPES)
def test_rounding_probes_are_rounded_once(dtype):
    """one dC / dR entry collects 1 + 2^-8 + 2^-60 (bf16) or 2^15 + 2^4 + 2^-38 (fp16): just above a tie of the
    type, below fp64's reach; the correctly rounded value is 1 + 2^-7 or 32800"""
    from _gpu import make_module
    L, gamma_np = wx.probe_layer(dtype)
    want, sums, _ = wx.dequant_backward(gamma_np, L)
    k, kr = int(L.meta["idx"][0, 0, 0]), int(L.meta["ridx"][0, 0, 0])
    for n, ent in (("centroids", k), ("res_centroids", kr)):
        assert wx.bits_to_float(want[n][0, ent * 8], dtype) == wx.PROBE_WANT[dtype]
    # dequant() backward through the module
    m = make_module(L)
    m.set_quant_grad(True)
    params = {"centroids": m.centroids.weight, "res_centroids": m.res_centroids.weight,
              "weight_scale": m.weight_scale, "weight_bias": m.weight_bias}
    for t in params.values():
        t.requires_grad_(True)
    gamma = torch.from_numpy(gamma_np.astype(np.float32)).to("cuda", _tdt(dtype))
    names = launched_kernels(lambda: m.dequant().backward(gamma))
    assert all(ran(names, kn) for kn in DQB_KERNELS), names
    m.zero_grad(set_to_none=True)          # the profiler may have run the call more than once: gradients accumulate
    m.dequant().backward(gamma)
    got = {n: _bits(t.grad) for n, t in params.items()}
    for n, ent in (("centroids", k), ("res_centroids", kr)):
        v = wx.bits_to_float(got[n].reshape(-1)[ent * 8], dtype)
        assert v == wx.PROBE_WANT[dtype], f"dequant() backward {n}: {v!r} != {wx.PROBE_WANT[dtype]!r}"
    assert_bits(got, want, f"dequant() backward {dtype}")
    # quant_gemm backward, one token per term
    x_np, dy_np = wx.probe_tokens(gamma_np)
    x = torch.from_numpy(x_np.astype(np.float32)).to("cuda", _tdt(dtype))
    dy = torch.from_numpy(dy_np.astype(np.float32)).to("cuda", _tdt(dtype))
    got = both_routes(_desc(L), L, x, dy, f"wgrad probe {dtype}")
    assert wx.bits_to_float(got["centroids"][0, k * 8], dtype) == wx.PROBE_WANT[dtype]
    head_zero()


# ---------------------------------------------------------------- extremes
EXT_FUSED = dict(in_features=512, out_features=264, vector_len=8, num_centroids=4096, num_res_centroids=256,
                 bias=True)
EXT_GEN = dict(in_features=512 + 8, out_features=260, vector_len=4, num_centroids=4096, num_res_centroids=16,
               outlier_size=8, outlier_vector_len=4, num_outlier_centroids=4096, num_codebooks=2, bias=True)


@pytest.mark.parametrize("cfg", ["fused", "generic"])
def test_terms_below_the_unit(cfg):
    """bf16: one term of 1.5 * 2^20 sets the unit near 2^-40; every other term lies between 2^-43 and 2^-36, around
    one unit, so each is rounded half-even on its own and every other entry is a sum of such roundings"""
    dtype = "bf16"
    L = vo.make_layer(dtype=dtype, seed=67, **(EXT_FUSED if cfg == "fused" else EXT_GEN))
    d = _desc(L)
    O, I = L.out_features, L.in_features
    gamma = random16((O, I), dtype, seed=68, lo=-43, hi=-37)
    gamma[0, 0] = 3.0 * 2.0 ** 19            # 1.5 * 2^20: the bounds keep clear of a power of two
    assert_bits(dqb(d, L, gamma, check_route=True), wx.dequant_backward(f64(gamma), L)[0], "dqb")
    # quant_gemm: token 0 carries the large term, token t one column of tiny values (one product per element of G)
    T = 48
    x = torch.zeros(T, I, dtype=_tdt(dtype), device="cuda")
    dy = random16((T, O), dtype, seed=69, lo=-43, hi=-37)
    dy[0] = 0.0
    x[0, 0], dy[0, 0] = 1.0, 3.0 * 2.0 ** 19
    t = torch.arange(1, T, device="cuda")
    x[t, t * 7 % I] = 1.0
    both_routes(d, L, x, dy, f"below the unit {cfg}")
    head_zero()


def _poison(d, where, value, used=True):
    """write `value` into one element of the descriptor's tensor `where` (through the module that owns it)"""
    m = d._module
    t = {"centroids": m.centroids.weight, "res_centroids": m.res_centroids.weight,
         "outlier_centroids": m.outlier_centroids.weight if m.enable_outlier else None,
         "weight_scale": m.weight_scale, "weight_bias": m.weight_bias, "bias": m.bias}[where]
    with torch.no_grad():
        flat = t.data.view(-1)
        if used:     # an entry an index refers to: the layer's first referenced main / residual / outlier entry
            L = d._layer
            v = L.vector_len
            if where == "centroids":
                i = int(L.meta["idx"][0, 0, 0]) * v
            elif where == "res_centroids":
                i = int(L.meta["ridx"][0, 0, 0]) * v
            elif where == "outlier_centroids":
                i = int(np.asarray(L.outlier_indices).reshape(-1)[0]) * L.outlier_vector_len
            else:
                i = t.numel() - 1
        else:        # an entry no index refers to
            L = d._layer
            n, used_idx, step = {"centroids": (L.num_centroids, L.meta["idx"][0], L.vector_len),
                                 "res_centroids": (L.num_res_centroids, L.meta["ridx"][0], L.vector_len),
                                 "outlier_centroids": (L.num_outlier_centroids, np.asarray(L.outlier_indices),
                                                       L.outlier_vector_len)}[where]
            unused = np.setdiff1d(np.arange(n), used_idx)     # group 0's codebook comes first in the tensor
            if not unused.size:
                return None
            i = int(unused[0]) * step
        old = flat[i].clone()
        flat[i] = value
    return lambda: flat.__setitem__(i, old)


def _ext_setup(cfg, dtype, seed):
    L = vo.make_layer(dtype=dtype, seed=seed, **cfg)
    d = _desc(L)
    d._layer = L
    x, dy = ints(40, L.in_features, dtype, seed), ints(40, L.out_features, dtype, seed + 1)
    gamma = random16((L.out_features, L.in_features), dtype, seed=seed)
    return L, d, x, dy, gamma


def _all_nan(got, what):
    for n, g in got.items():
        exp_all_ones = (g & 0x7C00) == 0x7C00 if what[1] == "fp16" else (g & 0x7F80) == 0x7F80
        mant = (g & 0x03FF) if what[1] == "fp16" else (g & 0x007F)
        assert (exp_all_ones & (mant != 0)).all(), f"{what} {n}: not NaN everywhere"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("cfg", ["fused", "generic"])
def test_non_finite_inputs_and_codebooks(cfg, dtype):
    """inf / NaN in x, dY, gamma, weight_scale, or a main / residual / outlier codebook entry (used or unused) with
    d weight_scale requested: NaN in every requested gradient.  A non-finite codebook entry without d weight_scale:
    the clean bits (codebook values are not read).  inf / NaN in weight_bias or bias: the clean bits."""
    L, d, x, dy, gamma = _ext_setup(EXT_FUSED if cfg == "fused" else EXT_GEN, dtype, 60)
    clean_w = both_routes(d, L, x, dy, "clean", route=True)
    clean_g = dqb(d, L, gamma, check_route=True)
    assert_bits(clean_g, wx.dequant_backward(f64(gamma), L)[0], "clean dqb")
    no_scale = [n for n in clean_w if n != "weight_scale"]
    books = ["centroids", "res_centroids"] + (["outlier_centroids"] if L.enable_outlier else [])
    for value in (float("inf"), float("-inf"), float("nan")):
        for where in ("x", "dy", "gamma"):
            xx, yy, gg = x.clone(), dy.clone(), gamma.clone()
            {"x": xx, "dy": yy, "gamma": gg}[where][3, 5] = value
            if where == "gamma":
                _all_nan(dqb(d, L, gg), (f"{where}={value}", dtype))
            else:
                for generic in (False, True):
                    _all_nan(wgrad(d, L, xx, yy, generic=generic), (f"{where}={value}", dtype))
        for where in books + ["weight_scale"]:
            for used in ((True, False) if where != "weight_scale" else (True,)):
                undo = _poison(d, where, value, used)
                if undo is None:                  # every residual entry is used
                    continue
                what = (f"{where}={value} used={used}", dtype)
                for generic in (False, True):
                    _all_nan(wgrad(d, L, x, dy, generic=generic), what)
                _all_nan(dqb(d, L, gamma), what)
                if where != "weight_scale":       # without d weight_scale the codebook values are never read
                    assert_bits(wgrad(d, L, x, dy, names=no_scale), {n: clean_w[n] for n in no_scale}, what[0])
                    assert_bits(wgrad(d, L, x, dy, generic=True, names=no_scale), {n: clean_w[n] for n in no_scale},
                                what[0])
                    assert_bits(dqb(d, L, gamma, names=no_scale), {n: clean_g[n] for n in no_scale}, what[0])
                undo()
        for where in ("weight_bias", "bias"):
            undo = _poison(d, where, value)
            for generic in (False, True):
                assert_bits(wgrad(d, L, x, dy, generic=generic), clean_w, f"{where}={value}")
            assert_bits(dqb(d, L, gamma), clean_g, f"{where}={value}")
            undo()
    assert_bits(wgrad(d, L, x, dy), clean_w, "clean again")
    head_zero()


@pytest.mark.parametrize("dtype", DTYPES)
def test_overflow_gives_signed_inf_exactly_where_the_exact_sum_rounds_past_the_maximum(dtype):
    """sums past the largest finite value: +-inf with the exact sum's sign on exactly those elements, the mirror's bits
    everywhere else"""
    L = env.layer_with("constant", "ones", in_features=512, out_features=264, vector_len=8, num_centroids=4096,
                       num_res_centroids=256, dtype=dtype, seed=61)
    d = _desc(L)
    big = 30000.0 if dtype == "fp16" else 2.0 ** 126
    gamma = random16((264, 512), dtype, seed=62, lo=0, hi=1) * big
    gamma[::2] = gamma[::2].abs()
    gamma[1::2] = -gamma[1::2].abs()
    want = wx.dequant_backward(f64(gamma), L)[0]
    inf = {n: np.isinf(wx.bits_to_float(w, dtype)) for n, w in want.items()}
    assert any(i.any() for i in inf.values()) and not all(i.all() for i in inf.values())
    assert_bits(dqb(d, L, gamma, check_route=True), want, f"overflow dqb {dtype}")
    if dtype == "fp16":          # integer inputs reach 65504 through the GEMM as well
        x, dy = ints(2048, 512, dtype, 63, lo=3), ints(2048, 264, dtype, 64, lo=3)
        dy[:, 1::2] = -dy[:, 1::2]
        w = both_routes(d, L, x, dy, "overflow wgrad", backend="torch")
        assert any(np.isinf(wx.bits_to_float(b, dtype)).any() for b in w.values())
    head_zero()


@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_dy_or_x_gives_plus_zero(dtype):
    L, d, x, dy, gamma = _ext_setup(EXT_FUSED, dtype, 65)
    for xx, yy in ((x, torch.zeros_like(dy)), (torch.zeros_like(x), dy)):
        for generic in (False, True):
            for n, g in wgrad(d, L, xx, yy, generic=generic, check_route=True).items():
                assert (g == 0).all(), n
    for n, g in dqb(d, L, torch.zeros_like(gamma)).items():
        assert (g == 0).all(), n
    head_zero()


# ---------------------------------------------------------------- graph
def test_graph_replay_clean_poisoned_clean():
    from vptq_b200 import native
    L = vo.make_layer(in_features=1024, out_features=520, vector_len=8, num_centroids=4096, num_res_centroids=256,
                      dtype="fp16", seed=66)
    d = _desc(L)
    x, dy = ints(200, 1024, "fp16", 20), ints(200, 520, "fp16", 21)
    eager = wgrad(d, L, x, dy, check_route=True)
    assert_bits(eager, wx.quant_gemm_wgrad(f64(x), f64(dy), L)[0], "eager")
    outs = _outs(L)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        native.quant_gemm_wgrad(d, x, dy, outs)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            native.quant_gemm_wgrad(d, x, dy, outs)
    clean = dy.clone()
    for step, poisoned in enumerate((False, True, False)):
        dy.copy_(clean)
        if poisoned:
            dy[7, 9] = float("nan")
        for t in outs.values():
            t.fill_(1.0)
        g.replay()
        torch.cuda.synchronize()
        got = {n: _bits(t) for n, t in outs.items()}
        if poisoned:
            _all_nan(got, ("graph poisoned", "fp16"))
        else:
            assert_bits(got, eager, f"graph replay {step}")
    head_zero()
