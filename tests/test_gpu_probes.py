"""Basis probes: x = e_f makes every output one product, so each kernel route is checked column by column against
the exact simulation of its arithmetic (tests/_probe.py) -- every element within 1 output ulp, and bit-equal where
the order of operations is the simulation's.  A bookkeeping error (a wrong entry, tile column, perm slot or list,
a padding word let through) moves an output by tens to thousands of ulps in exactly one column, which the
aggregate metric max|y - y*| / max|y*| of the other tests can miss.

Also here: the GEMM tile-walk sweep (nkb below the ring depth, many tiles per CTA, ragged edges), x = 0 on every
route, and the input / output layouts that change the route (pitched and misaligned x, broadcast x, y with a pitch
and guard rows).  Every test asserts the kernel it means to run (torch.profiler kernel names)."""
import time

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _probe import aligned_rows, fp64_bias, fp64_weight, launched_kernels, probe_expect, ran, to_dev, ulp_diff
from _util import TOL, parity_error

pytestmark = pytest.mark.gpu

LLAMA = {"4096x4096": (4096, 4096), "4096x14336": (4096, 14336), "14336x4096": (14336, 4096)}
_LAYERS = {}


def layer(**kw):
    """seeded oracle layer (the small ones are built once per session)"""
    kw = {"vector_len": 8, "seed": 1009, "dtype": "fp16", **kw}
    key = tuple(sorted(kw.items()))
    L = _LAYERS.get(key)
    if L is None:
        L = vo.make_layer(**kw)
        L.meta = {}            # (the unpacked indices: up to 1 GB at full size; the probes unpack L.indices)
        if kw["in_features"] * kw["out_features"] <= 1 << 22:
            _LAYERS[key] = L
    return L


def module(L, lists=True, deal=True):
    """VQuantLinear holding L, descriptor prepared with / without the list format (and its bank dealing)"""
    from _gpu import make_module
    m = make_module(L)
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("VPTQ_B200_LISTS", "1" if lists else "0")
        mp.setenv("VPTQ_B200_LISTS_DEAL", "1" if deal else "0")
        m.prepare()
    return m, m._desc_cache[0]


def report(what, y, expect, max_ulps=1):
    d = ulp_diff(y, expect)
    worst, exact = int(d.max()), float((d == 0).double().mean())
    print(f"\n[probe] {what}: bit-equal {exact:.6f}, max {worst} ulp")
    assert worst <= max_ulps, f"{what}: {worst} ulps (bit-equal {exact:.6f}), first at {np.unravel_index(int(d.argmax()), d.shape)}"
    return exact


def probe_gemv(d, L, tokens=1, X=None):
    """Y [I, O]: row f = quant_gemv(e_f), `tokens` probes per launch; no synchronisation inside the loop"""
    from vptq_b200 import native
    I, O = L.in_features, L.out_features
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    if X is None:
        X = aligned_rows(I, I, dt)
        X[torch.arange(I), torch.arange(I)] = 1.0
    Y = torch.full((I, O), float("nan"), dtype=dt, device="cuda")
    for f in range(0, I, tokens):
        n = min(tokens, I - f)
        native.quant_gemv(d, X[f:f + n], Y[f:f + n])
    torch.cuda.synchronize()
    return Y


def route_of_gemv(d, L, tokens):
    from vptq_b200 import native
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    x = aligned_rows(tokens, L.in_features, dt)
    y = torch.empty(tokens, L.out_features, dtype=dt, device="cuda")
    return launched_kernels(lambda: native.quant_gemv(d, x, y))


# ----------------------------------------------------------------------------------------------------------------
# 1. list kernel, one token, every feature
# ----------------------------------------------------------------------------------------------------------------
LIST_CASES = {f"k{K}_r{max(Kr, 0)}": dict(in_features=1024, out_features=264, num_centroids=K, num_res_centroids=Kr)
              for K in (8192, 16384, 32768, 65536) for Kr in (-1, 16, 256)}
LIST_CASES.update({
    "noperm_nonorm": dict(in_features=1024, out_features=256, num_centroids=65536, num_res_centroids=256,
                          enable_perm=False, enable_norm=False),
    "bias": dict(in_features=1024, out_features=512, num_centroids=65536, num_res_centroids=256, bias=True),
    "bf16": dict(in_features=2048, out_features=512, num_centroids=65536, num_res_centroids=256, dtype="bf16"),
    "bf16_bias_wide": dict(in_features=1024, out_features=264, num_centroids=16384, num_res_centroids=16, dtype="bf16",
                           bias=True, llm_like=False),
    "ragged_i1004": dict(in_features=1004, out_features=1004, num_centroids=65536, num_res_centroids=256),
    "ragged_i9000_o24": dict(in_features=9000, out_features=24, num_centroids=65536, num_res_centroids=256),
    "o8": dict(in_features=4096, out_features=8, num_centroids=65536, num_res_centroids=256),
})
LIST_CASES.update({f"llama_{k}": dict(in_features=i, out_features=o, num_centroids=65536, num_res_centroids=256)
                   for k, (i, o) in LLAMA.items()})


@pytest.mark.parametrize("name", list(LIST_CASES))
def test_list_kernel_probes(name):
    L = layer(**LIST_CASES[name])
    m, d = module(L)
    names = route_of_gemv(d, L, 1)
    assert ran(names, "gemv_lists_kernel") and not ran(names, "gemv_kernel"), names
    t0 = time.perf_counter()
    Y = probe_gemv(d, L)
    dt = time.perf_counter() - t0
    report(f"lists {name} ({L.in_features} launches, {dt:.2f} s)", Y, to_dev(probe_expect(L, "lists"), L))


def _fused_probe(descs, L0, outs):
    """one fused launch per probe: rows f of every output in `outs`"""
    from vptq_b200 import native
    I = L0.in_features
    X = aligned_rows(I, I, torch.float16)
    X[torch.arange(I), torch.arange(I)] = 1.0
    f0 = native.FusedGemv(descs, [y[0:1] for y in outs])
    names = launched_kernels(lambda: f0(X[0:1]))
    assert not f0.separate and sum(ran([n], "gemv_lists_kernel") for n in names) == 1, names
    for f in range(I):
        native.FusedGemv(descs, [y[f:f + 1] for y in outs])(X[f:f + 1])
    torch.cuda.synchronize()


@pytest.mark.parametrize("group", ["qkv", "gate_up"])
def test_fused_and_dealt_probes_are_bit_identical(group):
    """Under probes the result does not depend on which warp sums which entries: a fused launch equals the separate
    launches, and lists in build order equal the bank-dealt lists, bit for bit."""
    shapes = [(4096, 4096), (4096, 1024), (4096, 1024)] if group == "qkv" else [(4096, 14336), (4096, 14336)]
    Ls = [layer(in_features=i, out_features=o, num_centroids=65536, num_res_centroids=256, seed=2000 + k)
          for k, (i, o) in enumerate(shapes)]
    mods = [module(L) for L in Ls]
    fused = [torch.full((4096, L.out_features), float("nan"), dtype=torch.float16, device="cuda") for L in Ls]
    _fused_probe([d for _, d in mods], Ls[0], fused)
    for L, (m, d), yf in zip(Ls, mods, fused):
        ys = probe_gemv(d, L)
        assert torch.equal(ys, yf), "fused launch != separate launches"
        mu, du = module(L, deal=False)
        assert bool(du.lists_stream)
        assert torch.equal(probe_gemv(du, L), ys), "undealt lists != dealt lists"
        report(f"lists {group} {L.in_features}x{L.out_features}", ys, to_dev(probe_expect(L, "lists"), L))


# ----------------------------------------------------------------------------------------------------------------
# 2. generic GEMV, 1 / 2 / 4 tokens per launch (C ABI), a different probe per token
# ----------------------------------------------------------------------------------------------------------------
GENERIC_CASES = {
    "outliers_vol4": dict(in_features=1024 + 128, out_features=512, num_centroids=4096, num_res_centroids=256,
                          outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096, bias=True),
    "outliers_vol8": dict(in_features=2048 + 64, out_features=264, num_centroids=65536, num_res_centroids=256,
                          outlier_size=64, outlier_vector_len=8, num_outlier_centroids=1024),
    "groups4": dict(in_features=4096, out_features=512, num_centroids=1024, num_res_centroids=256, num_codebooks=4),
    "groups16": dict(in_features=14336, out_features=256, num_centroids=4096, num_codebooks=16),
    "v2": dict(in_features=512, out_features=128, vector_len=2, num_centroids=256),
    "v4_bf16": dict(in_features=1024, out_features=250, vector_len=4, num_centroids=4096, num_res_centroids=16,
                    dtype="bf16", bias=True),
    "v6": dict(in_features=768, out_features=250, vector_len=6, num_centroids=4096),
    "v10": dict(in_features=512, out_features=200, vector_len=10, num_centroids=1024, num_res_centroids=16),
    "v12": dict(in_features=1536, out_features=264, vector_len=12, num_centroids=4096, num_res_centroids=256),
    "v16": dict(in_features=512, out_features=256, vector_len=16, num_centroids=4096, num_res_centroids=16),
    "small_k": dict(in_features=1000, out_features=96, num_centroids=16, enable_perm=False, bias=True),
    "lists_layer_k65536": LIST_CASES["k65536_r256"],
    "lists_layer_bf16": LIST_CASES["bf16"],
    "lists_layer_noperm": LIST_CASES["noperm_nonorm"],
    "llama_14336x4096": LIST_CASES["llama_14336x4096"],
}


@pytest.mark.parametrize("name,tokens", [(n, t) for n in GENERIC_CASES for t in (1, 2, 4)
                                          if t == 4 or not n.startswith("llama")])   # full size once
def test_generic_gemv_probes(name, tokens):
    L = layer(**GENERIC_CASES[name])
    m, d = module(L, lists=False)
    assert not d.lists_stream
    names = route_of_gemv(d, L, tokens)
    assert ran(names, "gemv_kernel") and not ran(names, "gemv_lists_kernel"), names
    Y = probe_gemv(d, L, tokens)
    report(f"generic {name} x{tokens}", Y, to_dev(probe_expect(L, "generic"), L))


# ----------------------------------------------------------------------------------------------------------------
# 3. prefill GEMM with x = identity: T = I tokens, one call
# ----------------------------------------------------------------------------------------------------------------
def _identity(I, dt):
    return torch.eye(I, dtype=dt, device="cuda")


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", list(LLAMA))
def test_prefill_direct_identity_is_exact(shape, dtype):
    """T = I tokens: thousands of 128x256 tiles over 132 CTAs.  y must be dequant()^T bit for bit (one product per
    output, no rowbias) and dequant() within 1 ulp of the simulation."""
    i, o = LLAMA[shape]
    L = layer(in_features=i, out_features=o, num_centroids=65536, num_res_centroids=256, dtype=dtype)
    m, _ = module(L, lists=False)
    x = _identity(i, m.centroids.weight.dtype)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "dequant_o8_kernel") and ran(names, "gemm_tn_wgmma") and not ran(names, "prefill_prep_x"), names
    y = m(x)
    W = m.dequant()
    torch.cuda.synchronize()
    assert torch.equal(y, W.t())
    report(f"direct {shape} {dtype}", y, to_dev(probe_expect(L, "direct"), L))


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_prefill_direct_identity_with_bias(dtype):
    L = layer(in_features=1024, out_features=1000, num_centroids=4096, num_res_centroids=256, bias=True, dtype=dtype)
    m, _ = module(L, lists=False)
    x = _identity(1024, m.centroids.weight.dtype)
    assert ran(launched_kernels(lambda: m(x)), "dequant_o8_kernel")
    y = m(x)
    expect = (m.dequant().float() + m.bias.float()[:, None]).to(y.dtype).t()
    assert torch.equal(y, expect)
    report(f"direct bias {dtype}", y, to_dev(probe_expect(L, "direct"), L))


PREP_CASES = {
    "forced_4096_fp16": (dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256), True),
    "forced_4096_bf16": (dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256,
                              dtype="bf16"), True),
    "forced_outliers_bias": (GENERIC_CASES["outliers_vol4"], True),
    "i1000_bias": (dict(in_features=1000, out_features=520, num_centroids=8192, num_res_centroids=16, bias=True), False),
    "i1004_scalar_prep": (dict(in_features=1004, out_features=1004, num_centroids=65536, num_res_centroids=256), False),
    "i1004_bf16_nonorm": (dict(in_features=1004, out_features=264, num_centroids=4096, enable_norm=False,
                               dtype="bf16", bias=True), False),
    "groups4_v6": (dict(in_features=768, out_features=250, vector_len=6, num_centroids=4096, num_codebooks=4), False),
}


@pytest.mark.parametrize("name", list(PREP_CASES))
def test_prefill_prep_identity(name, monkeypatch):
    kw, force = PREP_CASES[name]
    L = layer(**kw)
    if force:
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    m, _ = module(L, lists=False)
    x = _identity(L.in_features, m.centroids.weight.dtype)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "prefill_prep_x") and ran(names, "gemm_tn_wgmma") and not ran(names, "dequant_o8_kernel"), names
    y = m(x)
    torch.cuda.synchronize()
    report(f"prep {name}", y, to_dev(probe_expect(L, "prep"), L))


# ----------------------------------------------------------------------------------------------------------------
# 4. x = 0 on every route: y is the bias, or zero
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("route", ["lists", "generic", "direct", "prep"])
def test_zero_input_gives_the_bias(route, bias, monkeypatch):
    I = 1004 if route == "prep" else 1024
    L = layer(in_features=I, out_features=520, num_centroids=65536, num_res_centroids=256, bias=bias, seed=5)
    m, _ = module(L, lists=route == "lists")
    tokens = {"lists": 1, "generic": 2, "direct": 300, "prep": 300}[route]
    x = torch.zeros(tokens, I, dtype=torch.float16, device="cuda")
    names = launched_kernels(lambda: m(x))
    kernel = {"lists": "gemv_lists_kernel", "generic": "gemv_kernel", "direct": "dequant_o8_kernel",
              "prep": "prefill_prep_x"}[route]
    assert ran(names, kernel), names
    y = m(x)
    expect = m.bias.expand(tokens, -1) if bias else torch.zeros_like(y)
    assert torch.equal(y, expect)


# ----------------------------------------------------------------------------------------------------------------
# GEMM tile walk: nkb = 1, 3, 5 against a 4-stage ring, ragged edges, more than 4 tiles per CTA
# ----------------------------------------------------------------------------------------------------------------
SWEEP = [  # (tokens, out_features, in_features, dtype)
    (3, 8, 64, "fp16"), (127, 248, 64, "fp16"), (128, 256, 64, "bf16"), (129, 264, 64, "fp16"),
    (8193, 2056, 64, "fp16"), (8193, 264, 64, "bf16"),
    (255, 256, 192, "fp16"), (256, 248, 192, "fp16"), (257, 2056, 192, "bf16"), (8193, 2056, 192, "fp16"),
    (3, 264, 192, "fp16"),
    (127, 2056, 320, "fp16"), (129, 8, 320, "bf16"), (8193, 256, 320, "fp16"), (8193, 2056, 320, "bf16"),
    (256, 264, 320, "fp16"),
    (3, 248, 1004, "fp16"), (255, 2056, 1004, "fp16"), (8193, 2056, 1004, "fp16"), (257, 8, 1004, "bf16"),
    (128, 264, 1004, "bf16"),
]


@pytest.mark.parametrize("tokens,out_features,in_features,dtype", SWEEP)
def test_gemm_tile_walk_sweep(tokens, out_features, in_features, dtype):
    L = layer(in_features=in_features, out_features=out_features, num_centroids=4096, num_res_centroids=16,
              dtype=dtype, bias=True, seed=tokens + out_features)
    m, _ = module(L, lists=False)
    g = torch.Generator(device="cuda").manual_seed(tokens)
    x = torch.randn(tokens, in_features, device="cuda", generator=g).to(m.centroids.weight.dtype)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "prefill_prep_x" if in_features % 64 else "dequant_o8_kernel"), names
    y = m(x)
    ref = x.double() @ fp64_weight(L).T + fp64_bias(L)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    assert parity_error(y.double().cpu().numpy(), ref.cpu().numpy()) <= TOL[dtype]


# ----------------------------------------------------------------------------------------------------------------
# input and output layouts
# ----------------------------------------------------------------------------------------------------------------
def _layout_layer():
    return layer(in_features=1024, out_features=524, num_centroids=65536, num_res_centroids=256, bias=True, seed=8)


@pytest.mark.parametrize("extra", [64, 3])
def test_x_column_slice_of_a_wider_buffer(extra, monkeypatch):
    """pitch % 8 == 0: TMA reads x with its pitch (direct route); otherwise the prep pass reads it"""
    L = _layout_layer()
    m, _ = module(L)
    g = torch.Generator(device="cuda").manual_seed(1)
    wide = torch.randn(300, 1024 + extra, device="cuda", generator=g).half()
    xs = wide[:, :1024]
    names = launched_kernels(lambda: m(xs))
    if extra % 8 == 0:
        assert ran(names, "dequant_o8_kernel") and not ran(names, "prefill_prep_x"), names
        assert torch.equal(m(xs), m(xs.contiguous()))
    else:
        assert ran(names, "prefill_prep_x"), names
        y = m(xs)
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
        assert int(ulp_diff(y, m(xs.contiguous())).max()) <= 1
    ref = xs.double() @ fp64_weight(L).T + fp64_bias(L)
    assert parity_error(m(xs).double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]


def test_x_with_an_odd_storage_offset(monkeypatch):
    """x not 16-byte aligned: one token falls back from the list kernel to the generic kernel, 3+ tokens take the
    prep route; results match the aligned calls of the same kernels."""
    from vptq_b200 import native
    L = _layout_layer()
    m, d = module(L)
    mg, dg = module(L, lists=False)
    assert d.lists_stream
    g = torch.Generator(device="cuda").manual_seed(2)
    buf = torch.randn(3 + 300 * 1024, device="cuda", generator=g).half()
    x1 = buf[3:3 + 1024].view(1, 1024)
    assert x1.data_ptr() % 16
    names = launched_kernels(lambda: m(x1))
    assert ran(names, "gemv_kernel") and not ran(names, "gemv_lists_kernel"), names
    y1 = m(x1)
    ya = torch.empty_like(y1)
    native.quant_gemv(dg, x1.contiguous(), ya)
    assert torch.equal(y1, ya)
    xt = buf[3:3 + 300 * 1024].view(300, 1024)
    names = launched_kernels(lambda: m(xt))
    assert ran(names, "prefill_prep_x") and not ran(names, "dequant_o8_kernel"), names
    yt = m(xt)
    monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    assert int(ulp_diff(yt, m(xt.contiguous())).max()) <= 1
    ref = xt.double() @ fp64_weight(L).T + fp64_bias(L)
    assert parity_error(yt.double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]


@pytest.mark.parametrize("tokens", [1, 2, 3, 64])
def test_broadcast_x(tokens):
    """x = v.expand(T, I) has row stride 0: the same result as the materialised input, with and without autograd"""
    L = _layout_layer()
    m, _ = module(L)
    g = torch.Generator(device="cuda").manual_seed(3)
    v = torch.randn(1024, device="cuda", generator=g).half()
    xe = v.expand(tokens, 1024)
    assert tokens == 1 or xe.stride(0) == 0
    y = m(xe)
    assert torch.equal(y, m(xe.contiguous()))
    ref = xe.double() @ fp64_weight(L).T + fp64_bias(L)
    assert parity_error(y.double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]
    vg = v.clone().requires_grad_(True)
    with torch.enable_grad():
        yg = m(vg.expand(tokens, 1024))
        assert torch.equal(yg.detach(), y)
        yg.float().sum().backward()
    gref = tokens * fp64_weight(L).sum(0)
    assert parity_error(vg.grad.double().cpu().numpy(), gref.cpu().numpy()) <= TOL["fp16"]


SENTINEL = 0x7E5B   # a NaN payload no kernel produces


def _guarded(rows, cols, pitch, dt):
    """[rows, cols] view with row pitch `pitch` into a buffer that ends with one more (guard) row; every element
    outside the view holds SENTINEL"""
    buf = torch.full(((rows + 1) * pitch,), SENTINEL, dtype=torch.int16, device="cuda")
    y = buf.view(dt).as_strided((rows, cols), (pitch, 1))
    inside = torch.zeros(rows + 1, pitch, dtype=torch.bool, device="cuda")
    inside[:rows, :cols] = True
    return y, buf, ~inside.view(-1)


def _guards_intact(buf, outside):
    return bool((buf[outside] == SENTINEL).all())


@pytest.mark.parametrize("pad", [1, 8])
def test_y_pitch_and_guard_rows(pad):
    from vptq_b200 import native
    L = _layout_layer()
    m, d = module(L)
    dt = torch.float16
    O, I = L.out_features, L.in_features
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(300, I, device="cuda", generator=g).half()
    # GEMV: one token (list kernel) and two (generic kernel)
    for tokens, kernel in ((1, "gemv_lists_kernel"), (2, "gemv_kernel")):
        y, buf, outside = _guarded(tokens, O, O + pad, dt)
        assert ran(launched_kernels(lambda: native.quant_gemv(d, x[:tokens], y)), kernel)
        yc = torch.empty(tokens, O, dtype=dt, device="cuda")
        native.quant_gemv(d, x[:tokens], yc)
        assert _guards_intact(buf, outside) and torch.equal(y, yc), (tokens, pad)
    # prefill GEMM: pitch O + 1 is odd -> the scalar epilogue
    y, buf, outside = _guarded(300, O, O + pad, dt)
    assert ran(launched_kernels(lambda: native.quant_gemm(d, x, y)), "gemm_tn_wgmma")
    yc = torch.empty(300, O, dtype=dt, device="cuda")
    native.quant_gemm(d, x, yc)
    assert _guards_intact(buf, outside) and torch.equal(y, yc)
    # transposed GEMM (input gradient): dX with pitch I + pad
    dy = torch.randn(300, O, device="cuda", generator=g).half()
    dx, buf, outside = _guarded(300, I, I + pad, dt)
    native.quant_gemm_dgrad(d, dy, dx)
    dxc = torch.empty(300, I, dtype=dt, device="cuda")
    native.quant_gemm_dgrad(d, dy, dxc)
    assert _guards_intact(buf, outside) and torch.equal(dx, dxc)
    # dequant takes no pitch: a guard region after the end only
    w, buf, outside = _guarded(O, I, I, dt)
    native.dequant(d, w)
    assert _guards_intact(buf, outside) and torch.equal(w, m.dequant())
