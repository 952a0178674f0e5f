"""CPU checks of tests/_wgrad_exact.py, the bit-exact mirror of the weight-gradient reduction, before the GPU file
(tests/test_gpu_wgrad_envelope.py) holds the kernels to it:
* its single rounding of sum * 2^e against fractions.Fraction, in fp16 and bf16, at ties +- one unit, subnormal
  results and results past the largest finite value;
* the crafted tie-plus-epsilon probes: the builders produce exactly the intended sums, and the old finish (fp64, then
  16 bit) rounds them the wrong way;
* the mirror against the fp64 oracle (tests/_wgrad.py) on every golden layer, within n_terms * u / 2 + 1/2 ulp;
* frexp semantics of the unit exponent, and the refusal near a power of two;
* the skewed index builders of tests/_envelope.py hit the entries they claim to.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import _envelope as env
import _wgrad_exact as wx
import vptq_oracle as vo
from _util import golden_names, load_golden
from _wgrad import grads_from_gamma, quant_gemm_wgrad

DTYPES = ("fp16", "bf16")


def _exact_bits(acc, e, dtype):
    return wx.fraction_to_bits(Fraction(int(acc)) * Fraction(2) ** e, dtype)


def _ulp(dtype, v):
    """one ulp of the 16-bit type at |v| (the subnormal spacing below the normal range)"""
    p, emin, _, _ = wx.FORMAT[dtype]
    a = abs(float(v))
    return 2.0 ** (max(math.frexp(a)[1] - 1, emin) - (p - 1)) if a else 2.0 ** (emin - (p - 1))


# ---------------------------------------------------------------- rounding
def _crafted(dtype):
    """(acc, e) pairs: ties of the 16-bit type +- one unit at several exponents, subnormals, overflow"""
    p, emin, emax, _ = wx.FORMAT[dtype]
    out = []
    for lead in (61, 60, 55, 54, 53, 40, 12):           # bit length of the sum
        for m in (1 << (p - 1), (1 << (p - 1)) + 1, (1 << p) - 1):   # even / odd significands, the largest one
            base = m << (lead - p)                        # exactly representable
            half = 1 << (lead - p - 1) if lead > p else 0
            for d in (0, 1, -1, half, half + 1, half - 1, -half, -half + 1, -half - 1):
                a = base + d
                if 0 < a < 1 << 62:
                    for e in (-lead + 1, -lead - 20, -lead + 10):
                        out += [(a, e), (-a, e)]
    for e in (emin - p - 60, emin - p - 62, emin - 62, emin - 70, emin - 55):     # subnormal and zero results
        for a in (1, 3, 1 << 40, (1 << 61) - 1, 1 << 60, (1 << 60) + 1, (3 << 59) + 12345):
            out += [(a, e), (-a, e)]
    for e in (emax - 60, emax - 61, emax - 50):           # at and past the largest finite value
        for a in ((1 << 61) - 1, 1 << 60, ((1 << p) - 1) << (61 - p), (((1 << p) - 1) << (61 - p)) + (1 << (60 - p))):
            out += [(a, e), (-a, e)]
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_round_fixed_matches_fractions_on_crafted_sums(dtype):
    cases = _crafted(dtype)
    acc = np.array([a for a, _ in cases], np.int64)
    for e in sorted({e for _, e in cases}):
        sel = [i for i, (_, ee) in enumerate(cases) if ee == e]
        got = wx.round_fixed(acc[sel], e, dtype)
        for i, g in zip(sel, got):
            assert int(g) == _exact_bits(acc[i], e, dtype), (dtype, int(acc[i]), e, hex(int(g)))
    bits = [wx.round_fixed(np.array([a]), e, dtype)[0] for a, e in cases]
    f = wx.bits_to_float(np.array(bits), dtype)
    assert np.isinf(f).any() and (np.abs(f[np.isfinite(f)]) < 2.0 ** wx.FORMAT[dtype][1]).any()


@pytest.mark.parametrize("dtype", DTYPES)
def test_round_fixed_matches_fractions_on_seeded_sums(dtype):
    rng = np.random.default_rng(11 if dtype == "fp16" else 12)
    _, emin, emax, _ = wx.FORMAT[dtype]
    for e in list(range(emin - 70, emax - 40, 7)) + [-60, -45, -61, 0]:
        lead = rng.integers(1, 62, size=64)
        acc = (rng.integers(0, 1 << 62, size=64, dtype=np.int64) >> (62 - lead)) * rng.choice([-1, 1], 64)
        got = wx.round_fixed(acc, e, dtype)
        for a, g in zip(acc, got):
            assert int(g) == _exact_bits(a, e, dtype), (dtype, int(a), e)


def test_round_fixed_zero_and_sign():
    for dtype in DTYPES:
        assert wx.round_fixed(np.array([0, -1]), -200, dtype).tolist() == [0, 0x8000]


# ---------------------------------------------------------------- the crafted tie-plus-epsilon probes
@pytest.mark.parametrize("dtype", DTYPES)
def test_probe_builders_give_the_intended_sums(dtype):
    L, gamma = wx.probe_layer(dtype)
    bits, sums, (e_cb, e_bias, e_scale) = wx.dequant_backward(gamma, L)
    terms = wx.PROBE_TERMS[dtype]
    B = sum(Fraction(g) * Fraction(s) for g, s in terms)
    assert Fraction(math.ldexp(1.0, e_cb)) == Fraction(2) ** (math.frexp(float(B))[1] - 61)
    k = int(L.meta["idx"][0, 0, 0])
    kr = int(L.meta["ridx"][0, 0, 0])
    for name, ent in (("centroids", k), ("res_centroids", kr)):
        acc = int(sums[name][0, ent * 8])
        assert Fraction(acc) * Fraction(2) ** e_cb == B, name                       # exact: no term was rounded
        assert wx.bits_to_float(bits[name][0, ent * 8], dtype) == wx.PROBE_WANT[dtype], name
        assert acc > 1 << 53 and acc & 0xFF                                           # fp64 cannot hold it
        old = wx.double_rounded(np.array([acc]), e_cb, dtype)
        assert int(old[0]) != int(bits[name][0, ent * 8]), name                       # the old finish is off by one
        assert wx.bits_to_float(old, dtype)[0] == (1.0 if dtype == "bf16" else 32768.0)
        assert np.count_nonzero(sums[name]) == 1
    assert np.count_nonzero(sums["weight_bias"]) == 3


@pytest.mark.parametrize("dtype", DTYPES)
def test_wgrad_probe_tokens_give_the_same_sums(dtype):
    """quant_gemm backward: one token per term (x = g e_f, dY = e_o), so B_cb has no cross terms and equals the
    dequant probe's bound"""
    L, gamma = wx.probe_layer(dtype)
    x, dy = wx.probe_tokens(gamma)
    a = wx.quant_gemm_wgrad(x, dy, L)
    b = wx.dequant_backward(gamma, L)
    assert a[2] == b[2]
    for n in a[0]:
        assert (a[1][n] == b[1][n]).all() and (a[0][n] == b[0][n]).all(), n


# ---------------------------------------------------------------- mirror vs the fp64 oracle
@pytest.mark.parametrize("name", golden_names())
def test_mirror_within_half_unit_per_term_of_fp64(name):
    L, x_np, _ = load_golden(name)
    gamma16 = vo.make_x(L.out_features, L.in_features, L.dtype, seed=4)
    gamma = vo.to_f32(gamma16, L.dtype).astype(np.float64)
    T = x_np.shape[0]
    dy16 = vo.make_x(T, L.out_features, L.dtype, seed=3)
    x = vo.to_f32(x_np, L.dtype).astype(np.float64)
    dy = vo.to_f32(dy16, L.dtype).astype(np.float64)
    for what, (bits, sums, es), want in (
            ("dequant", wx.dequant_backward(gamma, L), grads_from_gamma(gamma, L)),
            ("wgrad", wx.quant_gemm_wgrad(x, dy, L), quant_gemm_wgrad(x_np, dy16, L))):
        e_of = {"weight_scale": es[2], "weight_bias": es[1]}
        n_rows = L.out_features
        for n, w in want.items():
            e = e_of.get(n, es[0])
            fixed = sums[n].astype(np.float64).reshape(w.shape) * 2.0 ** e
            # terms per element: at most every (row, column) pair once
            n_terms = n_rows if n.startswith("weight_") else n_rows * L.in_features
            assert np.abs(fixed - w).max() <= n_terms * 2.0 ** e / 2 + 1e-300, (what, n)
            got = wx.bits_to_float(bits[n], L.dtype).reshape(w.shape)
            ulp = np.vectorize(lambda t: _ulp(L.dtype, t))(w)
            assert (np.abs(got - w) <= n_terms * 2.0 ** e / 2 + ulp / 2).all(), (what, n)


# ---------------------------------------------------------------- unit exponent
def test_unit_exponent_has_frexp_semantics():
    assert wx.unit_exponent(0.0) == 0
    for j in (-80, -1, 0, 1, 15, 60):
        p = 2.0 ** j
        assert wx.unit_exponent(p) == j + 1 - 61                 # B = 2^j: frexp gives m = 1/2, k = j + 1
        assert wx.unit_exponent(np.nextafter(p, 0)) == j - 61    # just below: m -> 1, k = j
        assert wx.unit_exponent(p * 1.5) == j + 1 - 61
        # every term |t| <= B is at most 2^61 units
        assert p <= 2.0 ** (wx.unit_exponent(p) + 61)


def test_bound_near_a_power_of_two_is_refused_unless_exact():
    L = vo.make_layer(in_features=64, out_features=16, vector_len=8, num_centroids=256, enable_norm=False, seed=3)
    g = np.zeros((16, 64))
    g[0, 0] = 1.0                                   # B = 1 exactly: a power of two the GPU also adds exactly
    assert wx.exponents_dequant(g, L)[0] == 1 - 61
    g[1, 0] = 2.0 ** -60                            # 1 + 2^-60 needs 61 bits: the GPU may round it to 1
    with pytest.raises(AssertionError, match="power of two"):
        wx.exponents_dequant(g, L)
    g[1, 0] = 2.0 ** -40                            # exact: 41 significant bits
    assert wx.exponents_dequant(g, L)[0] == 1 - 61
    with pytest.raises(AssertionError, match="power of two"):
        wx._exponent(2.0 - 2.0 ** -50, False, "B")
    assert wx._exponent(1.0 + 2.0 ** -40, False, "B") == 1 - 61


def test_lsb_and_exactness():
    assert wx._lsb(np.array([4.0, 0.5, 0.0])) == -1
    assert wx._lsb(np.array([3.0 * 2 ** -20])) == -20
    assert wx._lsb(np.zeros(3)) is None
    assert wx._exact(2.0 ** 52, 0) and not wx._exact(2.0 ** 53, 0)


# ---------------------------------------------------------------- skewed index builders
@pytest.mark.parametrize("kind", env.PATTERNS)
def test_index_builders_hit_the_entries_they_claim(kind):
    K = 65536
    L = env.layer_with(kind, in_features=4096, out_features=64, vector_len=8, num_centroids=K, num_res_centroids=256,
                       seed=9)
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    assert (idx == L.meta["idx"]).all() and (ridx == L.meta["ridx"]).all()
    i = idx[0]
    Ro = i.shape[0]
    if kind == "ones":
        assert (i == K - 1).all() and (ridx == 255).all()
    elif kind == "constant":
        assert (i == env.SLICE + 3).all()
    elif kind == "zipf_hot0":
        assert np.mean(i < 16) > 0.3
    elif kind == "zipf_spread":
        assert np.mean(i < 16) < 0.01 and np.bincount(i.ravel(), minlength=K).max() > 0.05 * i.size
    elif kind == "row_slice":
        assert ((i // env.SLICE) == (np.arange(Ro) % (K // env.SLICE))[:, None]).all()
    elif kind == "ramp":
        assert (i[-1] < env.SLICE).all() and np.mean(i[0] < env.SLICE) < 0.2
    elif kind == "col_slice":
        feat = np.asarray(L.perm).astype(np.int64)
        assert ((i // env.SLICE) == ((feat * (K // env.SLICE)) // 4096)[None, :]).all()
    else:
        assert len(np.unique(i)) > 0.9 * min(i.size, K) * (1 - np.exp(-i.size / K))
