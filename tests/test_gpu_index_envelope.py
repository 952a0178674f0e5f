"""The index envelope on the GPU: every packed field width b = 1..32, residual codebooks up to 65536 entries, skewed
index lists on the list kernel, both sides of every route cut-off, and unpacked checkpoints.

The other GPU tests draw every index uniformly from codebooks of at most 4096 residual entries (b <= 24).  Here the
index data is chosen (tests/_envelope.py): all-ones fields (idx = K - 1, ridx = Kr - 1, a 32-bit field fills whole
words), Zipf-distributed entries, rows whose fields all fall into one codebook slice, one constant index, and so on.

Bars, per route: basis probes within 1 ulp of the simulation of the route's arithmetic (tests/_probe.py); dequant()
equal to the prefill identity product; the input gradient against dY @ W in fp64 at TOL; weight gradients exact for
one-hot probes and at TOL against tests/_wgrad.py for random inputs.  Every test asserts the kernel it ran.
"""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _envelope import WIDTH_PAIRS, layer_with, list_shape_stats
from _probe import fp64_bias, fp64_weight, launched_kernels, probe_expect, ran, to_dev
from _util import TOL, parity_error
from _wgrad import quant_gemm_wgrad
from test_gpu_probes import module, probe_gemv, report, route_of_gemv
from test_gpu_wgrad import _assert_exact, _expected_probe, _generic_grads, _run_dequant_backward, _run_wgrad

pytestmark = pytest.mark.gpu


def _b(K, Kr):
    return int(np.log2(K)) + (int(np.log2(Kr)) if Kr > 0 else 0)


def _generic_names(d, L, tokens):
    names = route_of_gemv(d, L, tokens)
    assert not ran(names, "gemv_lists_kernel"), names
    assert ran(names, "gemv_kernel") or ran(names, "gemv_kernel_res_l2"), names
    return names


# ----------------------------------------------------------------------------------------------------------------
# B. field-width sweep: v = 8, one group, norm and perm, 1024 x 264
# ----------------------------------------------------------------------------------------------------------------
def _sweep_layer(K, Kr, kind, dtype="fp16", **kw):
    kw = {"in_features": 1024, "out_features": 264, "vector_len": 8, **kw}
    return layer_with(kind, num_centroids=K, num_res_centroids=Kr, dtype=dtype, seed=_b(K, Kr) * 7 + 1, **kw)


WIDTH_IDS = [f"k{K}_r{max(Kr, 0)}_b{_b(K, Kr)}" for K, Kr in WIDTH_PAIRS]


@pytest.mark.parametrize("kind", ["uniform", "ones"])
@pytest.mark.parametrize("K,Kr", WIDTH_PAIRS, ids=WIDTH_IDS)
def test_width_sweep_forward_routes(K, Kr, kind, monkeypatch):
    L = _sweep_layer(K, Kr, kind)
    # generic GEMV, lists off, 1 / 2 / 4 tokens per launch
    m, d = module(L, lists=False)
    assert not d.lists_stream
    gen = to_dev(probe_expect(L, "generic"), L)
    big_res = Kr * 16 > 200 * 1024           # 256 KiB and up cannot sit in shared memory next to the rest
    for tokens in (1, 2, 4):
        names = _generic_names(d, L, tokens)
        if big_res:
            assert ran(names, "gemv_kernel_res_l2"), names
        report(f"generic K={K} Kr={Kr} {kind} x{tokens}", probe_gemv(d, L, tokens), gen)
    # the list kernel wherever it is eligible
    ml, dl = module(L, lists=True)
    if dl.lists_stream:
        names = route_of_gemv(dl, L, 1)
        assert ran(names, "gemv_lists_kernel"), names
        report(f"lists K={K} Kr={Kr} {kind}", probe_gemv(dl, L), to_dev(probe_expect(L, "lists"), L))
    # dequant() within 1 ulp of the simulation; the prefill identity product equals it where the direct route runs
    # (dequant_o8_kernel: Kr <= 512 at this size), else it is the prep route's
    x = torch.eye(L.in_features, dtype=torch.float16, device="cuda")
    direct = Kr <= 512
    names = launched_kernels(lambda: m(x))
    assert ran(names, "gemm_tn_wgmma") and ran(names, "prefill_prep_x") != direct, names
    y = m(x)
    W = m.dequant()
    torch.cuda.synchronize()
    report(f"dequant K={K} Kr={Kr} {kind}", W.t().contiguous(), to_dev(probe_expect(L, "direct"), L))
    if direct:
        assert torch.equal(y, W.t())
    else:
        report(f"prep (default) K={K} Kr={Kr} {kind}", y, to_dev(probe_expect(L, "prep"), L))
    monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    names = launched_kernels(lambda: m(x))
    assert ran(names, "prefill_prep_x") and ran(names, "gemm_tn_wgmma"), names
    report(f"prep K={K} Kr={Kr} {kind}", m(x), to_dev(probe_expect(L, "prep"), L))


@pytest.mark.parametrize("K,Kr", WIDTH_PAIRS, ids=WIDTH_IDS)
def test_width_sweep_backward_routes(K, Kr):
    from test_gpu_wgrad import _module
    L = _sweep_layer(K, Kr, "uniform")
    m = _module(L)
    dt = m.centroids.weight.dtype
    # input gradient against dY @ W in fp64
    g = torch.Generator(device="cuda").manual_seed(K + Kr)
    x = torch.randn(5, L.in_features, device="cuda", generator=g).to(dt).requires_grad_(True)
    dy = torch.randn(5, L.out_features, device="cuda", generator=g).to(dt)
    names = launched_kernels(lambda: m(x).backward(dy))
    assert ran(names, "dequant_t8_kernel") or ran(names, "dequant_t_kernel"), names
    assert ran(names, "dequant_t8_kernel") == (Kr * 128 <= 64 * 1024), names
    x.grad = None
    m.zero_grad(set_to_none=True)
    m(x).backward(dy)
    ref = dy.double() @ fp64_weight(L)
    assert parity_error(x.grad.double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]
    # weight gradients: one-hot probes exact on both routes, random inputs at TOL
    o, f = L.out_features - 1, int(np.asarray(L.perm).astype(np.int64)[L.in_features - 1])
    want = _expected_probe(L, o, f)
    xe = torch.zeros(1, L.in_features, dtype=dt, device="cuda")
    xe[0, f] = 1
    de = torch.zeros(1, L.out_features, dtype=dt, device="cuda")
    de[0, o] = 1
    names = launched_kernels(lambda: _run_wgrad(m, xe, de))
    assert ran(names, "wg_finish") and ran(names, "wg_scatter") == (Kr > 256), names
    _assert_exact(_run_wgrad(m, xe, de), want, f"wgrad K={K} Kr={Kr}")
    _assert_exact(_generic_grads(m, xe, de), want, f"wgrad generic K={K} Kr={Kr}")
    gamma = torch.zeros(L.out_features, L.in_features, dtype=dt, device="cuda")
    gamma[o, f] = 1
    _assert_exact(_run_dequant_backward(m, gamma), want, f"dequant backward K={K} Kr={Kr}")
    x_np = vo.make_x(7, L.in_features, L.dtype, seed=1)
    dy_np = vo.make_x(7, L.out_features, L.dtype, seed=2)
    from _gpu import x_to_t
    got = _run_wgrad(m, x_to_t(x_np, L), x_to_t(dy_np, L))
    for n, w in quant_gemm_wgrad(x_np, dy_np, L).items():
        assert parity_error(got[n].float().cpu().numpy().reshape(w.shape), w) <= TOL["fp16"], n


# second set: other vector lengths, 4 groups, outliers of vector length 4
SECOND = [(v, b) for v in (2, 6, 12, 16) for b in (1, 17, 25, 31, 32) if not (b == 1 and v in (2, 6))]
_PAIR_OF_B = {1: (2, -1), 17: (32768, 4), 25: (65536, 512), 31: (32768, 65536), 32: (65536, 65536)}


@pytest.mark.parametrize("v,b", SECOND, ids=[f"v{v}_b{b}" for v, b in SECOND])
def test_width_sweep_groups_and_outliers(v, b):
    from _gpu import x_to_t
    from test_gpu_wgrad import _module
    K, Kr = _PAIR_OF_B[b]
    L = layer_with("ones" if b in (1, 32) else "uniform", in_features=1024 + 128, out_features=264, vector_len=v,
                   num_centroids=K, num_res_centroids=Kr, num_codebooks=4, outlier_size=128, outlier_vector_len=4,
                   num_outlier_centroids=256, bias=True, seed=b * 3 + v)
    m, d = module(L, lists=False)
    _generic_names(d, L, 1)
    report(f"generic v={v} b={b}", probe_gemv(d, L, 1), to_dev(probe_expect(L, "generic"), L))
    W = m.dequant()
    ref_w = fp64_weight(L)
    assert parity_error(W.double().cpu().numpy(), ref_w.cpu().numpy()) <= TOL["fp16"]
    x_np = vo.make_x(300, L.in_features, L.dtype, seed=5)
    x = x_to_t(x_np, L)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "gemm_tn_wgmma"), names
    ref = x.double() @ ref_w.T + fp64_bias(L)
    assert parity_error(m(x).double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]
    mg = _module(L)
    xg = x[:9].clone().requires_grad_(True)
    dy_np = vo.make_x(9, L.out_features, L.dtype, seed=6)
    dy = x_to_t(dy_np, L)
    mg(xg).backward(dy)
    assert parity_error(xg.grad.double().cpu().numpy(), (dy.double() @ ref_w).cpu().numpy()) <= TOL["fp16"]
    got = _run_wgrad(mg, x[:9], dy)
    for n, w in quant_gemm_wgrad(x_np[:9], dy_np, L).items():
        assert parity_error(got[n].float().cpu().numpy().reshape(w.shape), w) <= TOL["fp16"], n


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_full_size_k65536_r65536(dtype):
    """4096 x 4096, v = 8, K = Kr = 65536 (b = 32): the 1 MiB residual codebook is gathered through L1/L2."""
    from _gpu import x_to_t
    L = vo.make_layer(4096, 4096, vector_len=8, num_centroids=65536, num_res_centroids=65536, dtype=dtype, seed=77)
    L.meta = {}
    m, d = module(L, lists=False)
    W64 = fp64_weight(L)
    for tokens in (1, 2, 300):
        x_np = vo.make_x(tokens, 4096, dtype, seed=tokens)
        x = x_to_t(x_np, L)
        names = launched_kernels(lambda: m(x))
        if tokens < 3:
            assert ran(names, "gemv_kernel_res_l2"), names
        else:
            assert ran(names, "gemm_tn_wgmma"), names
        ref = x.double() @ W64.T
        err = parity_error(m(x).double().cpu().numpy(), ref.cpu().numpy())
        print(f"\n[full size K=Kr=65536 {dtype}] tokens={tokens}: {err:.3e}")
        assert err <= TOL[dtype]


# ----------------------------------------------------------------------------------------------------------------
# C. the list kernel on skewed lists
# ----------------------------------------------------------------------------------------------------------------
SKEWED = ("zipf_hot0", "zipf_spread", "row_slice", "constant", "ramp", "col_slice")
C_CONFIGS = {  # name: (in_features, out_features, K, Kr, dtype)
    "4096x4096_k65536_r256_fp16": (4096, 4096, 65536, 256, "fp16"),
    "4096x4096_k8192_r2_bf16": (4096, 4096, 8192, 2, "bf16"),
    "14336x4096_k65536_r2_bf16": (14336, 4096, 65536, 2, "bf16"),
    "14336x4096_k8192_r256_fp16": (14336, 4096, 8192, 256, "fp16"),
}
_C_LAYERS = {}


def _c_layer(cfg, kind):
    key = (cfg, kind)
    if key not in _C_LAYERS:
        I, O, K, Kr, dt = C_CONFIGS[cfg]
        _C_LAYERS.clear()
        _C_LAYERS[key] = layer_with(kind, in_features=I, out_features=O, num_centroids=K, num_res_centroids=Kr,
                                    dtype=dt, enable_perm=kind != "col_slice", seed=100 * SKEWED.index(kind) + K % 997)
    return _C_LAYERS[key]


def _lists_tol(L, y_star):
    from vptq_b200 import lists
    ns, nt, _ = lists.geometry(L.in_features, L.num_centroids)
    return TOL[L.dtype] * float(np.abs(y_star).max()) + ns * nt * 2.0 ** -31


def _lists_sim(L, x_np):
    """y of the list kernel's arithmetic in fp64: x' = rn16(x * scale), c + r rounded to fp16 for fp16 layers (fp32
    for bf16 ones), plus sum x * wbias"""
    from _wgrad import wq_original_order
    x = vo.to_f32(x_np, L.dtype).astype(np.float64).reshape(-1)
    s = vo.to_f32(L.weight_scale, L.dtype).astype(np.float64)
    wb = vo.to_f32(L.weight_bias, L.dtype).astype(np.float64)
    wq = wq_original_order(L)
    wq = (wq.astype(np.float16) if L.dtype == "fp16" else wq.astype(np.float32)).astype(np.float64)
    xq = vo.round_to((x * s).astype(np.float32), L.dtype).astype(np.float64)
    return (wq @ xq + float(x @ wb))[None, :]


def _tab_bounds(d):
    tab = d._keep[-1].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return tab & ((1 << 26) - 1), tab >> 26


_STATS = {}


@pytest.mark.parametrize("kind", SKEWED)
@pytest.mark.parametrize("cfg", list(C_CONFIGS))
def test_skewed_lists_against_fp64(cfg, kind, monkeypatch):
    from _gpu import x_to_t
    from vptq_b200 import lists, native
    L = _c_layer(cfg, kind)
    m, d = module(L)
    assert d.lists_stream
    # list shapes under the kernel's split of this layer over the SMs
    first, tail = _tab_bounds(d)
    ns, nt, _ = lists.geometry(L.in_features, L.num_centroids)
    Ro, Q = (L.out_features + 7) // 8, ns * nt
    ncta = min(torch.cuda.get_device_properties(0).multi_processor_count, Q * Ro)
    st = list_shape_stats(first, tail, Ro, Q, ncta)
    _STATS[(cfg, kind)] = st
    print(f"\n[list shapes] {cfg} {kind}: {st}")
    # random x against fp64
    x_np = vo.make_x(1, L.in_features, L.dtype, seed=11)
    x = x_to_t(x_np, L)
    names = launched_kernels(lambda: m(x))
    assert ran(names, "gemv_lists_kernel") and not ran(names, "gemv_kernel"), names
    y = m(x)
    y_star = (x.double() @ fp64_weight(L).T).cpu().numpy()
    err = float(np.abs(y.double().cpu().numpy() - y_star).max())
    # bar: the kernel's documented arithmetic in fp64 (x' = x * scale rounded to the layer's type, C + R rounded to
    # fp16 in fp16 layers), and the exact product within twice that.  With one slice per row or one constant index
    # the x' rounding errors of 14336 bf16 terms do not cancel against a varying weight: about TOL * max|y*| alone.
    y_sim = _lists_sim(L, x_np)
    err_sim = float(np.abs(y.double().cpu().numpy() - y_sim).max())
    print(f"\n[skewed lists] {cfg} {kind}: vs fp64 {err:.3e}, vs simulation {err_sim:.3e}, max|y*| {np.abs(y_star).max():.3e}")
    assert err_sim <= _lists_tol(L, y_sim), (err_sim, _lists_tol(L, y_sim))
    assert err <= 2 * _lists_tol(L, y_star), (err, _lists_tol(L, y_star))
    # the checked variant equals the default one on finite data
    monkeypatch.setenv("VPTQ_B200_LISTS_CHECKED", "1")
    assert torch.equal(m(x), y)
    monkeypatch.delenv("VPTQ_B200_LISTS_CHECKED")
    # 20 repeated calls bit-identical; the workspace's zero-at-rest head is zero afterwards
    ys = [m(x) for _ in range(20)]
    torch.cuda.synchronize()
    assert all(torch.equal(t, y) for t in ys)
    head = 65536 * 4 + 65536 * 64           # kZeroRegionBytes (csrc/kernels.h): counters + list accumulators
    ws = native.workspace(x.device, head)
    assert not bool(ws[:head].any())


@pytest.mark.parametrize("kind", SKEWED)
@pytest.mark.parametrize("cfg", ["4096x4096_k65536_r256_fp16", "4096x4096_k8192_r2_bf16"])
def test_skewed_lists_probes_dealt_and_undealt(cfg, kind):
    L = _c_layer(cfg, kind)
    m, d = module(L)
    assert ran(route_of_gemv(d, L, 1), "gemv_lists_kernel")
    Y = probe_gemv(d, L)
    report(f"lists {cfg} {kind}", Y, to_dev(probe_expect(L, "lists"), L))
    mu, du = module(L, deal=False)
    assert torch.equal(probe_gemv(du, L), Y), "undealt lists != dealt lists"


def test_skewed_patterns_reach_the_shapes_they_are_for():
    """From the tables of the layers above (host arithmetic): some unit spans at least 3 warps' runs, some CTA's range
    is mostly 1-step empty units, and some 8-step stage holds at least 2 unit ends."""
    from vptq_b200 import lists
    if len(_STATS) < len(C_CONFIGS) * len(SKEWED):   # run alone: compute the statistics here
        for cfg in C_CONFIGS:
            for kind in SKEWED:
                L = _c_layer(cfg, kind)
                I, O, K, Kr, _ = C_CONFIGS[cfg]
                pt = None if L.perm is None else torch.from_numpy(np.asarray(L.perm).astype(np.uint16).astype(np.int64))
                _, tab, _ = lists.build_lists(torch.from_numpy(np.ascontiguousarray(L.indices)).cuda(), num_centroids=K,
                                              num_res_centroids=Kr, in_features=I, out_features=O,
                                              perm=None if pt is None else pt.cuda(), deal=False)
                tb = tab.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
                ns, nt, _ = lists.geometry(I, K)
                Ro, Q = (O + 7) // 8, ns * nt
                ncta = min(torch.cuda.get_device_properties(0).multi_processor_count, Q * Ro)
                _STATS[(cfg, kind)] = list_shape_stats(tb & ((1 << 26) - 1), tb >> 26, Ro, Q, ncta)
    for k, s in sorted(_STATS.items()):
        print(f"\n[list shapes] {k}: {s}")
    assert max(s["max_warps_per_unit"] for s in _STATS.values()) >= 3
    assert max(s["empty_cta_share"] for s in _STATS.values()) > 0.5
    assert max(s["max_ends_per_stage"] for s in _STATS.values()) >= 2


def test_skewed_fused_qkv_equals_separate_launches():
    from vptq_b200 import native
    shapes = [(4096, 4096, "zipf_hot0"), (4096, 1024, "row_slice"), (4096, 1024, "ramp")]
    Ls = [layer_with(kind, in_features=i, out_features=o, num_centroids=65536, num_res_centroids=256, seed=300 + k)
          for k, (i, o, kind) in enumerate(shapes)]
    mods = [module(L) for L in Ls]
    I = 4096
    X = torch.zeros(I, I, dtype=torch.float16, device="cuda")
    X[torch.arange(I), torch.arange(I)] = 1.0
    fused = [torch.full((I, L.out_features), float("nan"), dtype=torch.float16, device="cuda") for L in Ls]
    f0 = native.FusedGemv([d for _, d in mods], [y[0:1] for y in fused])
    names = launched_kernels(lambda: f0(X[0:1]))
    assert not f0.separate and sum(ran([n], "gemv_lists_kernel") for n in names) == 1, names
    for f in range(I):
        native.FusedGemv([d for _, d in mods], [y[f:f + 1] for y in fused])(X[f:f + 1])
    torch.cuda.synchronize()
    for L, (m, d), yf in zip(Ls, mods, fused):
        assert torch.equal(probe_gemv(d, L), yf), "fused launch != separate launches"
        report(f"lists fused {L.in_features}x{L.out_features}", yf, to_dev(probe_expect(L, "lists"), L))


# ----------------------------------------------------------------------------------------------------------------
# D. route cut-offs: one layer on either side
# ----------------------------------------------------------------------------------------------------------------
def _fp64_check(m, L, tokens, seed=3):
    from _gpu import x_to_t
    x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)
    y = m(x)
    ref = x.double() @ fp64_weight(L).T + (fp64_bias(L) if L.bias is not None else 0)
    err = parity_error(y.double().cpu().numpy(), ref.cpu().numpy())
    assert err <= TOL[L.dtype], err


@pytest.mark.parametrize("K,main_smem", [(8192, True), (16384, False)])
def test_cutoff_main_codebook_in_shared_memory(K, main_smem):
    """generic GEMV: the main codebook is staged in shared memory iff K * 2v <= 128 KiB"""
    L = layer_with("uniform", in_features=1024, out_features=264, num_centroids=K, num_res_centroids=16, seed=5)
    m, d = module(L, lists=False)
    names = _generic_names(d, L, 1)
    assert any(f"gemv_kernel<__half, 8, 1, {'true' if main_smem else 'false'}, true>" in n for n in names), names
    report(f"generic K={K}", probe_gemv(d, L), to_dev(probe_expect(L, "generic"), L))
    _fp64_check(m, L, 2)


@pytest.mark.parametrize("Kr", [256, 512])
def test_cutoff_residual_replication(Kr):
    """v = 8: the residual codebook is replicated 8x in shared memory iff Kr * 16 * 8 <= 32 KiB (not visible in the
    kernel's name: both sides must give the probes' values)"""
    L = layer_with("uniform", in_features=1024, out_features=264, num_centroids=4096, num_res_centroids=Kr, seed=6)
    m, d = module(L, lists=False)
    names = _generic_names(d, L, 1)
    assert not ran(names, "gemv_kernel_res_l2"), names
    report(f"generic Kr={Kr}", probe_gemv(d, L), to_dev(probe_expect(L, "generic"), L))
    _fp64_check(m, L, 2)


@pytest.mark.parametrize("v,K,Kr,l2", [(8, 65536, 8192, False), (8, 65536, 16384, True), (8, 4096, 8192, False),
                                       (8, 4096, 16384, True), (16, 4096, 4096, False), (16, 4096, 8192, True),
                                       (2, 4096, 32768, False), (2, 4096, 65536, True),
                                       (12, 256, 8192, False), (12, 256, 16384, True)])
def test_cutoff_residual_codebook_through_l2(v, K, Kr, l2):
    """generic GEMV: a residual codebook that fits is staged in shared memory; one that does not is gathered through
    L1/L2 (before, such a layer had no decode plan at all)"""
    L = layer_with("uniform", in_features=1536, out_features=264, vector_len=v, num_centroids=K,
                   num_res_centroids=Kr, seed=7 + v)
    m, d = module(L, lists=False)
    gen = to_dev(probe_expect(L, "generic"), L)
    for tokens in (1, 2):
        names = _generic_names(d, L, tokens)
        assert ran(names, "gemv_kernel_res_l2") == l2, names
        report(f"generic v={v} K={K} Kr={Kr} x{tokens}", probe_gemv(d, L, tokens), gen)
    _fp64_check(m, L, 1)
    _fp64_check(m, L, 2)


def test_cutoff_residual_through_l2_in_a_fused_launch():
    """gemv_multi_kernel_res_l2: two v = 8 layers with Kr = 65536 in one launch equal the separate launches"""
    from vptq_b200 import native
    Ls = [layer_with("uniform", in_features=2048, out_features=o, num_centroids=4096, num_res_centroids=65536,
                     seed=400 + o) for o in (1024, 512)]
    mods = [module(L, lists=False) for L in Ls]
    x = torch.randn(2, 2048, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)).half()
    for tokens in (1, 2):
        ys = [torch.empty(tokens, L.out_features, dtype=torch.float16, device="cuda") for L in Ls]
        fg = native.FusedGemv([d for _, d in mods], ys)
        names = launched_kernels(lambda: fg(x[:tokens]))
        assert not fg.separate and ran(names, "gemv_multi_kernel_res_l2"), names
        fg(x[:tokens])
        torch.cuda.synchronize()
        for L, (m, d), y in zip(Ls, mods, ys):
            # (a fused launch plans each layer for its share of the SMs: its sums need not be the separate launch's
            # bits, so the bar is fp64)
            ref = x[:tokens].double() @ fp64_weight(L).T
            assert parity_error(y.double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]


@pytest.mark.parametrize("I,fast", [(41240, True), (41248, False)])
def test_cutoff_dequant_original_order_fast_path(I, fast):
    """dequant_o8_kernel needs Kr <= 512 and packed row + Kr * 128 <= 190 KiB (csrc/dequant.cu): with K = 65536 and
    Kr = 512 (b = 25) that is in_features <= 41240"""
    L = layer_with("ones", in_features=I, out_features=16, num_centroids=65536, num_res_centroids=512, seed=8)
    L.meta = {}
    m, _ = module(L, lists=False)
    names = launched_kernels(lambda: m.dequant())
    assert ran(names, "dequant_o8_kernel") == fast and ran(names, "dequant_kernel") != fast, names
    W = m.dequant()
    report(f"dequant I={I}", W.t().contiguous(), to_dev(probe_expect(L, "direct"), L))


@pytest.mark.parametrize("Kr,fast", [(512, True), (1024, False)])
def test_cutoff_prep_and_dgrad_fast_paths(Kr, fast, monkeypatch):
    """the quantised-order (prep) and transposed (dgrad) dequant fast paths need Kr * 128 <= 64 KiB"""
    L = layer_with("uniform", in_features=1024, out_features=264, num_centroids=4096, num_res_centroids=Kr, seed=9)
    monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    m, _ = module(L, lists=False)
    x = torch.eye(1024, dtype=torch.float16, device="cuda")
    names = launched_kernels(lambda: m(x))
    assert ran(names, "dequant_q8_kernel") == fast and ran(names, "prefill_prep_x"), names
    report(f"prep Kr={Kr}", m(x), to_dev(probe_expect(L, "prep"), L))
    xg = torch.randn(4, 1024, device="cuda").half().requires_grad_(True)
    dy = torch.randn(4, 264, device="cuda").half()
    names = launched_kernels(lambda: m(xg).backward(dy))
    assert ran(names, "dequant_t8_kernel") == fast and ran(names, "dequant_t_kernel") != fast, names
    xg.grad = None
    m(xg).backward(dy)
    assert parity_error(xg.grad.double().cpu().numpy(), (dy.double() @ fp64_weight(L)).cpu().numpy()) <= TOL["fp16"]


@pytest.mark.parametrize("Kr", [256, 512])
def test_cutoff_fused_weight_gradient(Kr):
    """the weight gradient is fused into the GEMM epilogue iff Kr <= 256; above, G goes through wg_scatter"""
    from test_gpu_wgrad import _module
    L = layer_with("uniform", in_features=1024, out_features=264, num_centroids=4096, num_res_centroids=Kr, seed=10)
    m = _module(L)
    dt = torch.float16
    o, f = 7, 5
    xe = torch.zeros(1, 1024, dtype=dt, device="cuda")
    xe[0, f] = 1
    de = torch.zeros(1, 264, dtype=dt, device="cuda")
    de[0, o] = 1
    names = launched_kernels(lambda: _run_wgrad(m, xe, de))
    assert ran(names, "wg_scatter") == (Kr > 256), names
    _assert_exact(_run_wgrad(m, xe, de), _expected_probe(L, o, f), f"wgrad Kr={Kr}")


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_cutoff_list_kernel_sm_count():
    """K = 65536 (NS = 16): NS * NT at and just past the SM count.  The layer past it gets no lists (the list launch
    would refuse it), runs the generic kernel, and prepare(drop_packed=True) refuses it up front."""
    from vptq_b200 import lists
    P = _sm_count()
    nt_in, nt_out = P // 16, P // 16 + 1
    for nt, inside in ((nt_in, True), (nt_out, False)):
        I = min(nt * 4096, 65535) if inside else min((nt - 1) * 4096 + 8, 65528)
        ns, got_nt, _ = lists.geometry(I, 65536)
        assert (ns * got_nt <= P) == inside, (I, ns, got_nt, P)
        L = layer_with("uniform", in_features=I, out_features=16, num_centroids=65536, num_res_centroids=256, seed=12)
        L.meta = {}
        m, d = module(L)
        names = route_of_gemv(d, L, 1)
        assert bool(d.lists_stream) == inside
        assert ran(names, "gemv_lists_kernel") == inside and ran(names, "gemv_kernel") != inside, names
        _fp64_check(m, L, 1)
        if not inside:
            with pytest.raises(RuntimeError, match="drop_packed"):
                m.prepare(drop_packed=True)
            assert m.indices.numel() > 0
            _fp64_check(m, L, 1)


def test_cutoff_fused_list_launch_past_the_sm_count():
    """4 fused layers with n * Q > SM count: the list launch refuses, the fused call still equals separate calls"""
    from vptq_b200 import lists, native
    P = _sm_count()
    I = 12288                                     # NT = 3, Q = 48 at K = 65536: 4 * 48 > P
    assert 4 * 16 * lists.geometry(I, 65536)[1] > P
    Ls = [layer_with("uniform", in_features=I, out_features=64, num_centroids=65536, num_res_centroids=256,
                     seed=500 + k) for k in range(4)]
    mods = [module(L) for L in Ls]
    x = torch.randn(1, I, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).half()
    ys = [torch.empty(1, 64, dtype=torch.float16, device="cuda") for _ in Ls]
    fg = native.FusedGemv([d for _, d in mods], ys)
    fg(x)
    torch.cuda.synchronize()
    for L, (m, d), y in zip(Ls, mods, ys):
        ref = x.double() @ fp64_weight(L).T
        assert parity_error(y.double().cpu().numpy(), ref.cpu().numpy()) <= TOL["fp16"]


# ----------------------------------------------------------------------------------------------------------------
# E. unpacked checkpoints: the packer runs at forward
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,Kr", [(256, -1), (4096, 4096), (65536, 65536)], ids=["b8", "b24", "b32"])
def test_unpacked_checkpoint_equals_packed(K, Kr):
    from _gpu import make_module
    from vptq_b200 import VQuantLinear
    L = layer_with("ones" if Kr == 65536 else "uniform", in_features=1024, out_features=264, num_centroids=K,
                   num_res_centroids=Kr, seed=13)
    mp = make_module(L)
    mu = VQuantLinear(1024, 264, vector_lens=[-1, 8], num_centroids=[-1, K], num_res_centroids=[-1, Kr], group_num=1,
                      group_size=1024, outlier_size=0, indices_as_float=True, enable_norm=True, enable_perm=True,
                      is_indice_packed=False, device="cuda", dtype=torch.float16, enable_proxy_error=False)
    with torch.no_grad():
        mu.indices.data = torch.from_numpy(L.meta["idx"].astype(np.uint16)).view(torch.int16).cuda()
        if Kr > 0:
            mu.res_indices.data = torch.from_numpy(L.meta["ridx"].astype(np.uint16)).view(torch.float16).cuda()
            mu.res_centroids.weight.data = mp.res_centroids.weight.data.clone()
        mu.centroids.weight.data = mp.centroids.weight.data.clone()
        mu.perm.data = torch.from_numpy(np.asarray(L.perm).astype(np.int64)).cuda()
        mu.weight_scale.data = mp.weight_scale.data.clone()
        mu.weight_bias.data = mp.weight_bias.data.clone()
    mu.eval()
    assert torch.equal(mu._packed_indices(), mp.indices)
    g = torch.Generator(device="cuda").manual_seed(K)
    for tokens in (1, 2, 300):
        x = torch.randn(tokens, 1024, device="cuda", generator=g).half()
        assert torch.equal(mu(x), mp(x)), tokens
    assert torch.equal(mu.dequant(), mp.dequant())
