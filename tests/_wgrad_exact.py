"""Bit-exact mirror of the weight-gradient reduction (csrc/wgrad.cu, the EPI_WGRAD epilogue of csrc/gemm_wgmma.cu).

Given G = dL/dW as an exact fp64 array [O, I] (original feature order), the kernels' arithmetic is exactly specified:
  * three bounds, B_cb = sum |s_f G| (>=), B_bias = sum |G| (>=), B_scale = B_bias max|Wq|, each giving the unit
    2^e with e = k - 61, where B = m 2^k, 1/2 <= m < 1 (frexp), and e = 0 for B = 0;
  * every term rounded half-even to its unit on its own: s_f G for dC, dR and dCol, G fp32(C + R) (or Col) for
    d weight_scale, G for d weight_bias;
  * integer sums (exact in any order);
  * one correct rounding of sum * 2^e to fp16 or bf16 (`round_fixed`, integer arithmetic only).
G is exact for dequant() backward (the caller's 16-bit gradient) and for quant_gemm backward when x and dY are
integers with |.| <= 4 (every partial sum of dY^T x is an integer below 2^24: the fp32 tensor-core GEMM is exact).

The GPU adds the bounds in fp64 in its own order.  Where every partial sum is exact (all terms multiples of one
power of two, the total below 2^53 of it) the bound is known exactly; otherwise a bound within 2^-45 (relative) of a
power of two could land on either side of it on the GPU, and the mirror refuses (AssertionError) instead of guessing.
The GPU's summation error is below 2^-46 relative for every shape here: per row at most ceil(n / 256) + 13 additions
in a chain, then ceil(rows / 256) + 9, each 2^-53 relative.

Two back ends accumulate the integer sums: numpy (np.add.at; any layer) and torch (index_add_ on int64; one codebook
group, no outlier columns; G may live on the GPU).  Both give the same integers.
"""
import math
from fractions import Fraction

import numpy as np

import _envelope as _env
import vptq_oracle as vo

FRAC_BITS = 61
MARGIN = 2.0 ** -45
# significant bits, least normal exponent, largest exponent, exponent bias
FORMAT = {"fp16": (11, -14, 15, 15), "bf16": (8, -126, 127, 127)}
NAMES = ("centroids", "res_centroids", "outlier_centroids", "weight_scale", "weight_bias")


# ---------------------------------------------------------------------------------------------------- rounding
def _bit_length(mag):
    """bit length of non-negative uint64 values (exact: a float64 estimate corrected by one shift)"""
    fl = np.frexp(mag.astype(np.float64))[1].astype(np.int64)
    over = (fl > 0) & ((mag >> np.maximum(fl - 1, 0).astype(np.uint64)) == 0)
    return np.where(over, fl - 1, fl)


def round_fixed(acc, e, dtype):
    """16-bit patterns (uint16) of acc * 2^e (acc int64, e an integer), rounded once to nearest even; +-inf past the
    largest finite value, -0 for a negative sum that rounds to zero."""
    p, emin, emax, bias = FORMAT[dtype]
    acc = np.asarray(acc, dtype=np.int64)
    neg = acc < 0
    mag = np.abs(acc).astype(np.uint64)                     # |acc| < 2^63: the fixed-point sums stay below 2^62
    E = _bit_length(mag) - 1 + e                            # exponent of the leading bit
    q = np.maximum(E - (p - 1), emin - (p - 1))             # exponent of the result's last bit
    shift = q - e
    rs = np.clip(shift, 0, 63).astype(np.uint64)            # shifts past 63 leave nothing: |acc| < 2^62 < half
    n = mag >> rs
    rem = mag - (n << rs)
    half = np.where(rs > 0, np.uint64(1) << np.maximum(rs, 1) - np.uint64(1), np.uint64(0))
    up = (rs > 0) & ((rem > half) | ((rem == half) & ((n & np.uint64(1)) == 1)))
    n = n + up.astype(np.uint64)
    n = np.where(shift < 0, mag << np.clip(-shift, 0, 63).astype(np.uint64), n)   # exact: no bits dropped
    carry = n == (np.uint64(1) << np.uint64(p))
    n = np.where(carry, n >> np.uint64(1), n)
    q = q + carry
    normal = n >= (np.uint64(1) << np.uint64(p - 1))
    expf = np.where(normal, q + (p - 1) + bias, 0).astype(np.int64)
    mant = np.where(normal, n - (np.uint64(1) << np.uint64(p - 1)), n).astype(np.int64)
    bits = (expf << (p - 1)) | mant
    bits = np.where(expf >= 2 * bias + 1, (2 * bias + 1) << (p - 1), bits)      # +-inf
    bits = np.where(mag == 0, 0, bits) | (neg.astype(np.int64) << 15)
    return bits.astype(np.uint16)


def double_rounded(acc, e, dtype):
    """The finish before round-to-odd: acc -> fp64 (rounds above 2^53), * 2^e, then fp64 -> 16 bit (rounds again)."""
    v = np.ldexp(np.asarray(acc, dtype=np.int64).astype(np.float64), e)
    if dtype == "fp16":
        return v.astype(np.float16).view(np.uint16)
    return _f64_to_bf16_bits(v)


def _f64_to_bf16_bits(v):
    """fp64 -> bf16 patterns, rounded once (through the exact Fraction of each value)"""
    out = np.empty(np.shape(v), np.uint16)
    for i, x in enumerate(np.ravel(v)):
        out.flat[i] = fraction_to_bits(Fraction(float(x)) if math.isfinite(x) else x, "bf16")
    return out


def bits_to_float(bits, dtype):
    bits = np.asarray(bits, dtype=np.uint16)
    return bits.view(np.float16).astype(np.float64) if dtype == "fp16" else vo.bf16_bits_to_f32(bits).astype(np.float64)


_TABLE = {}


def _positive_table(dtype):
    """(values as Fractions, bit patterns) of every positive finite value, then 2^(emax+1) standing for inf"""
    if dtype not in _TABLE:
        p, _, emax, bias = FORMAT[dtype]
        top = (2 * bias + 1) << (p - 1)
        bits = np.arange(1, top, dtype=np.uint16)
        vals = [Fraction(float(x)) for x in bits_to_float(bits, dtype)]
        _TABLE[dtype] = (vals + [Fraction(2) ** (emax + 1)], [int(b) for b in bits] + [top])
    return _TABLE[dtype]


def fraction_to_bits(v, dtype):
    """Independent rounding of an exact rational (or +-inf / nan float) to a 16-bit pattern by table search."""
    if isinstance(v, float):
        if math.isnan(v):
            return 0x7E00 if dtype == "fp16" else 0x7FC0
        return (0x7C00 if dtype == "fp16" else 0x7F80) | (0x8000 if v < 0 else 0)
    import bisect
    vals, bits = _positive_table(dtype)
    sign = 0x8000 if v < 0 else 0
    a = abs(v)
    if a == 0:
        return sign
    i = bisect.bisect_left(vals, a)
    if i < len(vals) and vals[i] == a:
        return sign | bits[i]
    if i == len(vals):                                  # past 2^(emax+1): inf
        return sign | bits[-1]
    lo_v, lo_b = (vals[i - 1], bits[i - 1]) if i > 0 else (Fraction(0), 0)
    hi_v, hi_b = vals[i], bits[i]
    d_lo, d_hi = a - lo_v, hi_v - a
    pick = lo_b if d_lo < d_hi or (d_lo == d_hi and lo_b % 2 == 0) else hi_b
    return sign | pick


# ---------------------------------------------------------------------------------------------------- bounds
def unit_exponent(B):
    """e of the unit 2^e for a bound B >= 0 (a float): frexp's k - 61, 0 for B = 0"""
    if not B > 0:
        return 0
    return math.frexp(B)[1] - FRAC_BITS


def _lsb(a):
    """least exponent j such that every finite value of a is a multiple of 2^j (None if all zero)"""
    a = np.abs(np.asarray(a, dtype=np.float64).ravel())
    a = a[a > 0]
    if a.size == 0:
        return None
    m, k = np.frexp(a)
    mi = (m * 2.0 ** 53).astype(np.int64)
    tz = np.log2((mi & -mi).astype(np.float64)).astype(np.int64)
    return int((k - 53 + tz).min())


def _exact(total, lsb):
    return lsb is None or total * 2.0 ** -lsb < 2.0 ** 53


def _exponent(B, exact, what):
    if exact or not B > 0:
        return unit_exponent(B)
    m = math.frexp(B)[0]
    assert 2 * (m - 0.5) >= MARGIN and 1 - m >= MARGIN, (
        f"{what} bound {B!r} lies within 2^-45 of a power of two: the GPU's fp64 sum could round it there")
    return unit_exponent(B)


def max_wq(L):
    """fmax(max|C| + max|R|, max|Col|) in fp64, as wg_units forms it"""
    f = lambda a: float(np.abs(vo.to_f32(a, L.dtype)).max()) if a is not None else 0.0
    return max(f(L.centroids) + (f(L.res_centroids) if L.res_bits else 0.0),
               f(L.outlier_centroids) if L.enable_outlier else 0.0)


def _scale(L):
    return (np.ones(L.in_features) if L.weight_scale is None
            else vo.to_f32(L.weight_scale, L.dtype).astype(np.float64))


def exponents_from_rows(a, b, c, lsb_a, lsb_b, lsb_c, mwq):
    """(e_cb, e_bias, e_scale) from the per-row sums a (None: all 1), b = sum |s v|, c = sum |v| (exact fp64 values,
    or accurate to a few ulps) and the least exponents of their terms."""
    a = np.ones_like(b) if a is None else a
    la = 0 if lsb_a is None else lsb_a
    rows_exact = all(_exact(float(np.max(t, initial=0.0)), l) for t, l in ((a, lsb_a), (b, lsb_b), (c, lsb_c)))
    bc, bb = float(np.sum(a * b)), float(np.sum(a * c))
    ex_c = rows_exact and _exact(bc, None if lsb_b is None else la + lsb_b)
    ex_b = rows_exact and _exact(bb, None if lsb_c is None else la + lsb_c)
    bs = bb * mwq
    ex_s = ex_b and Fraction(bb) * Fraction(mwq) == Fraction(bs)
    return _exponent(bc, ex_c, "B_cb"), _exponent(bb, ex_b, "B_bias"), _exponent(bs, ex_s, "B_scale")


def exponents_dequant(gamma, L):
    g = np.abs(np.asarray(gamma, dtype=np.float64))
    s = np.abs(_scale(L))
    sg = g * s[None, :]
    return exponents_from_rows(None, sg.sum(1), g.sum(1), None, _lsb(sg), _lsb(g), max_wq(L))


def exponents_wgrad(x, dy, L):
    """x [T, I], dy [T, O] as exact fp64 values"""
    x, dy = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(dy, np.float64))
    sx = x * np.abs(_scale(L))[None, :]
    return exponents_from_rows(dy.sum(1), sx.sum(1), x.sum(1), _lsb(dy), _lsb(sx), _lsb(x), max_wq(L))


# ---------------------------------------------------------------------------------------------------- sums
def _fixed(t, e):
    return np.rint(np.ldexp(t, -e)).astype(np.int64)


def _indices(L):
    if L.meta.get("idx") is not None:
        idx = np.asarray(L.meta["idx"], np.int64)
        ridx = None if L.res_bits == 0 else np.asarray(L.meta["ridx"], np.int64)
        return idx, ridx
    return vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)


def _perm(L):
    return np.arange(L.in_features) if L.perm is None else np.asarray(L.perm).astype(np.uint16).astype(np.int64)


def sums_numpy(gamma, L, es, want=NAMES):
    """integer sums {name: int64 array in the layer array's shape} for G = gamma [O, I] (exact fp64)"""
    e_cb, e_bias, e_scale = es
    gamma = np.asarray(gamma, dtype=np.float64)
    O, I, v, G, gs = L.out_features, L.in_features, L.vector_len, L.num_codebooks, L.group_size
    K, Kr = L.num_centroids, L.num_res_centroids
    S = L.outlier_size if L.enable_outlier else 0
    perm = _perm(L)
    s = _scale(L)
    idx, ridx = _indices(L)
    Ro = idx.shape[1]
    gq = np.zeros((Ro * v, I))
    gq[:O] = gamma[:, perm]                                  # quantised column order
    sgq = gq * s[perm][None, :]
    C = vo.to_f32(L.centroids, L.dtype).reshape(G, K, v)
    R = vo.to_f32(L.res_centroids, L.dtype).reshape(G, Kr, v) if L.res_bits else None
    out = {}
    dC = np.zeros((G, K, v), np.int64)
    dR = np.zeros((G, max(Kr, 1), v), np.int64)
    wq = np.zeros((Ro * v, I), np.float32)
    for g in range(G):
        cols = slice(S + g * gs, S + (g + 1) * gs)
        t = _fixed(sgq[:, cols], e_cb).reshape(Ro, v, gs).transpose(0, 2, 1)       # [Ro, gs, v]
        np.add.at(dC[g], idx[g], t)
        w = C[g][idx[g]]                                                           # [Ro, gs, v] fp32
        if R is not None:
            np.add.at(dR[g], ridx[g], t)
            w = w + R[g][ridx[g]]                                                  # fp32 add, as the kernels do
        wq[:, cols] = w.transpose(0, 2, 1).reshape(Ro * v, gs)
    if "centroids" in want:
        out["centroids"] = dC.reshape(G, K * v)
    if R is not None and "res_centroids" in want:
        out["res_centroids"] = dR.reshape(G, Kr * v)
    if S:
        vol, Kol = L.outlier_vector_len, L.num_outlier_centroids
        oidx = np.asarray(L.outlier_indices).astype(np.uint16).astype(np.int64).reshape(-1, S)   # [Rol, S]
        Rol = oidx.shape[0]
        po = np.zeros((Rol * vol, S))
        po[:O] = sgq[:O, :S]
        Col = vo.to_f32(L.outlier_centroids, L.dtype).reshape(Kol, vol)
        if "outlier_centroids" in want:
            dCol = np.zeros((Kol, vol), np.int64)
            np.add.at(dCol, oidx, _fixed(po, e_cb).reshape(Rol, vol, S).transpose(0, 2, 1))
            out["outlier_centroids"] = dCol.reshape(1, Kol * vol)
        n = min(Rol * vol, Ro * v)
        wq[:n, :S] = Col[oidx].transpose(0, 2, 1).reshape(Rol * vol, S)[:n]
    if L.weight_scale is not None:
        for name, t, e in (("weight_scale", gq[:O] * wq[:O].astype(np.float64), e_scale),
                           ("weight_bias", gq[:O], e_bias)):
            if name in want:
                r = np.zeros(I, np.int64)
                r[perm] = _fixed(t, e).sum(0)
                out[name] = r
    return out


def sums_torch(gamma, L, es, want=NAMES):
    """sums_numpy for one codebook group without outlier columns, in torch (gamma: fp64 tensor on any device)"""
    import torch
    assert L.num_codebooks == 1 and not L.enable_outlier
    e_cb, e_bias, e_scale = es
    dev = gamma.device
    O, I, v, K, Kr = L.out_features, L.in_features, L.vector_len, L.num_centroids, L.num_res_centroids
    perm = torch.from_numpy(_perm(L)).to(dev)
    s = torch.from_numpy(_scale(L)).to(dev)
    idx, ridx = _indices(L)
    idx = torch.from_numpy(idx[0]).to(dev)                                        # [Ro, I] quantised order
    ridx = torch.from_numpy(ridx[0]).to(dev) if L.res_bits else None
    Ro = idx.shape[0]

    def fixed(t, e):
        return torch.round(t * 2.0 ** -e).to(torch.int64)     # scaling by a power of two is exact

    gq = torch.zeros(Ro * v, I, dtype=torch.float64, device=dev)
    gq[:O] = gamma[:, perm]
    out = {}
    t = fixed(gq * s[perm][None, :], e_cb).view(Ro, v, I).permute(0, 2, 1).reshape(-1, v)
    if "centroids" in want:
        out["centroids"] = torch.zeros(K, v, dtype=torch.int64, device=dev).index_add_(0, idx.reshape(-1), t)
    if ridx is not None and "res_centroids" in want:
        out["res_centroids"] = torch.zeros(Kr, v, dtype=torch.int64, device=dev).index_add_(0, ridx.reshape(-1), t)
    del t
    if L.weight_scale is not None:
        C = torch.from_numpy(vo.to_f32(L.centroids, L.dtype).reshape(K, v)).to(dev)
        w = C[idx]
        if ridx is not None:
            w = w + torch.from_numpy(vo.to_f32(L.res_centroids, L.dtype).reshape(Kr, v)).to(dev)[ridx]
        wq = w.permute(0, 2, 1).reshape(Ro * v, I)[:O].double()
        del w
        for name, tt, e in (("weight_scale", lambda: gq[:O] * wq, e_scale), ("weight_bias", lambda: gq[:O], e_bias)):
            if name in want:
                r = torch.zeros(I, dtype=torch.int64, device=dev)
                r[perm] = fixed(tt(), e).sum(0)
                out[name] = r
    return {n: (a if n.startswith("weight_") else a.reshape(1, -1)).cpu().numpy() for n, a in out.items()}


# ---------------------------------------------------------------------------------------------------- results
def finish(sums, es, dtype):
    """{name: 16-bit patterns} from the integer sums"""
    e_cb, e_bias, e_scale = es
    e_of = {"weight_scale": e_scale, "weight_bias": e_bias}
    return {n: round_fixed(a, e_of.get(n, e_cb), dtype) for n, a in sums.items()}


def dequant_backward(gamma, L, want=NAMES, backend="numpy"):
    """(bits, sums, exponents) of vptq_b200_dequant_backward with G = gamma (exact fp64 [O, I], numpy, or a torch
    fp64 tensor for the torch back end)"""
    g_np = gamma if isinstance(gamma, np.ndarray) else gamma.double().cpu().numpy()
    es = exponents_dequant(g_np, L)
    sums = sums_numpy(g_np, L, es, want) if backend == "numpy" else sums_torch(gamma, L, es, want)
    return finish(sums, es, L.dtype), sums, es


def quant_gemm_wgrad(x, dy, L, want=NAMES, backend="numpy"):
    """(bits, sums, exponents) of vptq_b200_quant_gemm_wgrad; x [T, I], dy [T, O] exact fp64 (numpy, or torch
    tensors for the torch back end, where G = dY^T x is formed in fp64 on their device: exact for integer inputs)"""
    if backend == "numpy":
        x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
        es = exponents_wgrad(x, dy, L)
        sums = sums_numpy(dy.T @ x, L, es, want)
    else:
        es = exponents_wgrad(x.double().cpu().numpy(), dy.double().cpu().numpy(), L)
        sums = sums_torch(dy.double().t() @ x.double(), L, es, want)
    return finish(sums, es, L.dtype), sums, es


# ---------------------------------------------------------------------------------------------------- probes
# dequant() backward: three terms s_f G[o][f] land on one dC entry; each is one G entry times its feature's scale
PROBE_TERMS = {"bf16": [(1.0, 1.0), (2.0 ** -8, 1.0), (2.0 ** -30, 2.0 ** -30)],       # B = 1 + 2^-8 + 2^-60
               "fp16": [(2.0 ** 15, 1.0), (2.0 ** 4, 1.0), (2.0 ** -24, 2.0 ** -14)]}   # B = 2^15 + 2^4 + 2^-38
PROBE_WANT = {"bf16": 1.0 + 2.0 ** -7, "fp16": 32800.0}


def probe_layer(dtype, v=8, K=256, Kr=2, I=64, O=16):
    """constant main and residual indices, unit scales but for the probe's third feature; the three G entries sit at
    (0, f0), (0, f1), (v, f2): the same e = 0, so the same dC[k][0] and dR[kr][0]"""
    L = _env.layer_with("constant", "ones", in_features=I, out_features=O, vector_len=v, num_centroids=K,
                       num_res_centroids=Kr, dtype=dtype, seed=5)
    terms = PROBE_TERMS[dtype]
    feats = [3, 17, 40]
    s = np.ones(I, np.float32)
    s[feats[2]] = terms[2][1]
    cast = (lambda a: a.astype(np.float16)) if dtype == "fp16" else vo.f32_to_bf16_bits
    L.weight_scale = cast(s)
    gamma = np.zeros((O, I))
    for (g, _), o, f in zip(terms, (0, 0, v), feats):
        gamma[o, f] = g
    assert (vo.to_f32(cast(gamma.astype(np.float32)), dtype) == gamma).all()      # every G entry is 16 bit
    return L, gamma


def probe_tokens(gamma):
    O, I = gamma.shape
    nz = np.argwhere(gamma != 0)
    x, dy = np.zeros((len(nz), I)), np.zeros((len(nz), O))
    for t, (o, f) in enumerate(nz):
        x[t, f] = gamma[o, f]
        dy[t, o] = 1.0
    return x, dy
