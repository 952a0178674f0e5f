"""Every kernel route on inf / NaN inputs and on magnitudes far from 1, against an IEEE float64 reference
(tests/_extreme.py: the oracle's dense weight with the injected values, y* as element-wise products and sums).

Injections (NaN, +inf, -inf): one x feature of one token (dY for dgrad); one element of a main-codebook entry that
`isolate` confines to a few index rows -- an arbitrary entry, entry 0 and entry 4096 (entry 0 of slice 1: the
entries the padding lanes of the generic and the list kernel decode to); the same for residual entry k and
residual entry 0; weight_scale[f], weight_bias[f], bias[o] and one outlier-codebook entry.  For each:
  * isfinite(y) == isfinite(y*) element by element (y* rounded to the output type);
  * NaN injected: every non-finite output is NaN;
  * +-inf injected into a codebook or the bias (one non-finite term per output): the sign of y*, where the list
    kernel may return NaN instead; no route ever returns the opposite sign of y*;
  * every output the injection does not reach (y* finite) is bit-identical to the clean call, and a clean call
    after the poisoned one is bit-identical to the clean call before it (the workspace is back at rest).
Then: fp16 outputs that overflow, the list kernel's fixed-point range (fp16 products past 2^33, bf16 outputs of
2^36) and bf16 activations of 2^20; power-of-two scaling of x, which every route but the list kernel must carry
through bit for bit, while the list kernel keeps |y - y*| <= TOL max|y*| + Q 2^-31.  Every case asserts the
kernels it means to run (torch.profiler).  The list kernel runs as its checked variant
(VPTQ_B200_LISTS_CHECKED=1)."""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _extreme import (FINITE, NAN, NEG_INF, POS_INF, VALUES, classify, dense64, dgrad_star, encode, feature_of,
                      inject, isolate, isolated_column, y_star)
from _probe import launched_kernels, ran
from _util import TOL, parity_error

import _batch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _checked_lists(monkeypatch):
    """the list kernel's checked variant: the one whose results are defined for these inputs (the default variant
    leaves non-finite and out-of-range unit sums undefined, include/vptq_b200.h)"""
    monkeypatch.setenv("VPTQ_B200_LISTS_CHECKED", "1")

# index rows that use the isolated entries (every configuration has >= 9 index rows)
ROWS = {"C_arb": [1, 7], "C0": [2], "Cs": [3], "Rk": [4], "R0": [5, 8]}
K_ARB, R_ARB = 777, 5


def _dt(L):
    return torch.float16 if L.dtype == "fp16" else torch.bfloat16


def make_desc(L, lists):
    from _gpu import to_t
    from vptq_b200 import native
    outl = L.enable_outlier
    t = dict(indices=to_t(L.indices, L, "i32"), centroids=to_t(L.centroids, L),
             res_centroids=to_t(L.res_centroids, L) if L.res_bits else None,
             outlier_indices=to_t(L.outlier_indices, L, "u16") if outl else None,
             outlier_centroids=to_t(L.outlier_centroids, L) if outl else None,
             perm=to_t(L.perm, L, "u16") if L.perm is not None else None,
             weight_scale=to_t(L.weight_scale, L), weight_bias=to_t(L.weight_bias, L), bias=to_t(L.bias, L))
    d = native.make_desc(dtype=_dt(L), in_features=L.in_features, out_features=L.out_features,
                         vector_len=L.vector_len, num_centroids=L.num_centroids,
                         num_res_centroids=L.num_res_centroids, num_codebooks=L.num_codebooks,
                         group_size=L.group_size, outlier_size=L.outlier_size if outl else 0,
                         outlier_vector_len=L.outlier_vector_len, num_outlier_centroids=L.num_outlier_centroids,
                         lists=lists, **t)
    d._tensors = t
    assert bool(d.lists_stream) == lists
    return d


FIELD = {"C": "centroids", "R": "res_centroids", "Col": "outlier_centroids", "scale": "weight_scale",
         "wbias": "weight_bias", "bias": "bias"}


def upload(d, L, field):
    """write L's array `field` into the descriptor's tensor (and its quantised-order copy)"""
    from _gpu import to_t
    t = d._tensors[field]
    t.copy_(to_t(getattr(L, field), L).view_as(t))
    if field in ("weight_scale", "weight_bias") and d.weight_scale_q:
        pidx = d._tensors["perm"].view(torch.uint16).to(torch.int64)
        d._keep[0 if field == "weight_scale" else 1].copy_(t[pidx])


# ------------------------------------------------------------------------------------------------------------------
# layers and routes
# ------------------------------------------------------------------------------------------------------------------
CONFIGS = {
    "i1004": dict(in_features=1004, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True),
    "i1000_bf16": dict(in_features=1000, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True,
                       dtype="bf16"),
    "i9000": dict(in_features=9000, out_features=72, num_centroids=65536, num_res_centroids=256),
    "i1024": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True),
    "i1024_bf16": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True,
                       dtype="bf16"),
    "llama": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256),
    "v4_groups_outliers": dict(in_features=1000 + 128, out_features=250, vector_len=4, num_centroids=4096,
                               num_res_centroids=16, num_codebooks=2, outlier_size=128, outlier_vector_len=4,
                               num_outlier_centroids=256, bias=True),
    "fused_1": dict(in_features=1004, out_features=128, num_centroids=65536, num_res_centroids=256),
    "fused_2": dict(in_features=1004, out_features=136, num_centroids=65536, num_res_centroids=256, bias=True),
}
_CTX = {}


class Ctx:
    """one isolated layer, its fp64 weight, a clean x and descriptors with / without the lists"""

    def __init__(self, name):
        kw = {"vector_len": 8, "seed": 4242, **CONFIGS[name]}
        L = vo.make_layer(**kw)
        main = {K_ARB: ROWS["C_arb"], 0: ROWS["C0"]}
        if L.num_centroids >= 8192:
            main[4096] = ROWS["Cs"]
        self.L = isolate(L, main=main, res={R_ARB: ROWS["Rk"], 0: ROWS["R0"]} if L.res_bits else None)
        self.W = torch.from_numpy(dense64(self.L)).cuda()
        self.x = torch.from_numpy(vo.to_f32(vo.make_x(8, L.in_features, L.dtype, seed=17), L.dtype)).cuda().to(_dt(L))
        self.dy = torch.from_numpy(vo.to_f32(vo.make_x(3, L.out_features, L.dtype, seed=18), L.dtype)).cuda().to(_dt(L))
        self._d = {}

    def desc(self, lists):
        if lists not in self._d:
            self._d[lists] = make_desc(self.L, lists)
        return self._d[lists]


def ctx(name):
    if name not in _CTX:
        _CTX[name] = Ctx(name)
    return _CTX[name]


def _nan(shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def run(kind, c, x, descs=None):
    """one call of route `kind` on context c (x: activations, or dY for dgrad) -> output tensor"""
    from vptq_b200 import native
    L, dt = c.L, _dt(c.L)
    if kind in ("lists", "generic"):
        y = _nan((x.shape[0], L.out_features), dt)
        native.quant_gemv(c.desc(kind == "lists"), x, y)
    elif kind in ("direct", "prep"):
        y = _nan((x.shape[0], L.out_features), dt)
        native.quant_gemm(c.desc(False), x, y)
    elif kind == "dequant":
        y = _nan((L.out_features, L.in_features), dt)
        native.dequant(c.desc(False), y)
    elif kind == "dgrad":
        y = _nan((x.shape[0], L.in_features), dt)
        native.quant_gemm_dgrad(c.desc(False), x, y)
    elif kind == "fused":
        ys = [_nan((1, d.out_features), dt) for d in descs]
        f = native.FusedGemv(descs, ys)
        f(x)
        assert not f.separate
        y = torch.cat(ys, dim=1)
    elif kind == "batch":
        y = _batch.batch(c.desc(True), x)
    elif kind == "batch_fused":
        y = torch.cat(_batch.batch(descs, x), dim=1)
    else:
        raise ValueError(kind)
    return y


def kernels_ok(kind, names):
    dq = ran(names, "dequant_o8_kernel") or ran(names, "dequant_q8_kernel") or ran(names, "dequant_kernel")
    return {
        "lists": ran(names, "gemv_lists_kernel") and not ran(names, "gemv_kernel"),
        "fused": sum(ran([n], "gemv_lists_kernel") for n in names) == 1 and not ran(names, "gemv_kernel"),
        "batch": sum(ran([n], _batch.BATCH) for n in names) == 1 and not ran(names, "gemv_lists_kernel"),
        "batch_fused": sum(ran([n], _batch.BATCH) for n in names) == 1 and not ran(names, "gemv_lists_kernel"),
        "generic": ran(names, "gemv_kernel") and not ran(names, "gemv_lists_kernel"),
        "direct": ran(names, "dequant_o8_kernel") and ran(names, "gemm_tn_wgmma") and not ran(names, "prefill_prep_x"),
        "prep": ran(names, "prefill_prep_x") and ran(names, "gemm_tn_wgmma") and not ran(names, "dequant_o8_kernel"),
        "dequant": dq and not ran(names, "gemm_tn_wgmma"),
        "dgrad": (ran(names, "dequant_t8_kernel") or ran(names, "dequant_t_kernel")) and ran(names, "gemm_tn_wgmma"),
    }[kind]


def run_checked(kind, c, x, descs=None):
    out = []
    names = launched_kernels(lambda: out.append(run(kind, c, x, descs)))
    assert kernels_ok(kind, names), (kind, names)
    torch.cuda.synchronize()
    return out[0]


# route -> (configuration, kind, tokens)
ROUTES = {
    "lists_i1004": ("i1004", "lists", 1),
    "lists_i1000_bf16": ("i1000_bf16", "lists", 1),
    "lists_i9000": ("i9000", "lists", 1),
    "lists_llama": ("llama", "lists", 1),
    "lists_fused": ("i1004", "fused", 1),
    "generic1_i1004": ("i1004", "generic", 1),
    "generic2_i1004": ("i1004", "generic", 2),
    "generic2_i1000_bf16": ("i1000_bf16", "generic", 2),
    "generic1_v4_groups_outliers": ("v4_groups_outliers", "generic", 1),
    "generic2_v4_groups_outliers": ("v4_groups_outliers", "generic", 2),
    "direct_fp16": ("i1024", "direct", 3),
    "direct_bf16": ("i1024_bf16", "direct", 3),
    "prep_fp16": ("i1004", "prep", 3),
    "prep_bf16": ("i1000_bf16", "prep", 3),
    "dequant": ("i1004", "dequant", 0),
    "dgrad": ("i1004", "dgrad", 3),
    **{f"batch{t}_{cfg}": (cfg, "batch", t) for cfg in ("i1004", "i1000_bf16", "i9000", "llama") for t in (2, 5, 8)},
    "batch_fused": ("i1004", "batch_fused", 5),
}
LISTS_LIKE = ("lists", "fused", "batch", "batch_fused")     # kinds that run a list kernel (descriptors with lists)


def _sites(route):
    cfg, kind, _ = ROUTES[route]
    if route == "lists_llama":
        return ["x", "Cs"]
    if kind == "fused":
        return ["x", "C0", "Cs", "R0", "wbias"]
    kw = {"vector_len": 8, **CONFIGS[cfg]}
    s = ["C_arb", "C0", "Rk", "R0", "scale", "wbias"]
    if kind != "dequant":
        s.insert(0, "x")
    if kind in ("lists", "batch", "batch_fused"):
        s.append("Cs")
    if kw.get("bias") and kind not in ("dequant", "dgrad"):
        s.append("bias")
    if kw.get("outlier_size"):
        s.append("Col")
    return s


CASES = [(r, s) for r in ROUTES for s in _sites(r)]
SIGNED = ("C_arb", "C0", "Cs", "Rk", "R0", "bias", "Col")   # one non-finite term per affected output


def _injection(c, site, v):
    """-> (kwargs of _extreme.inject, field) for a layer site"""
    L = c.L
    e = min(3, L.vector_len - 1)
    if site in ("C_arb", "C0", "Cs"):
        return dict(site="C", k={"C_arb": K_ARB, "C0": 0, "Cs": 4096}[site], e=e), "centroids"
    if site in ("Rk", "R0"):
        return dict(site="R", k=R_ARB if site == "Rk" else 0, e=e), "res_centroids"
    if site == "Col":
        return dict(site="Col", k=int(L.outlier_indices[0, 1, 3]), e=1), "outlier_centroids"
    if site == "scale":
        return dict(site="scale", f=L.in_features // 3), "weight_scale"
    if site == "wbias":
        return dict(site="wbias", f=L.in_features - 2), "weight_bias"
    if site == "bias":
        return dict(site="bias", o=L.out_features - 3), "bias"
    raise ValueError(site)


def check_classes(y, ys, clean, vname, site, lists_like):
    cs, cy = classify(ys.to(y.dtype)), classify(y)
    fin = cs == FINITE
    bad = (cy == FINITE) != fin
    assert not bad.any(), f"{int(bad.sum())} outputs differ in finiteness from y* (first at {bad.nonzero()[0].tolist()})"
    assert not fin.all(), "the injection reached no output"
    if vname == "nan":
        assert bool((cy[~fin] == NAN).all()), "NaN injected, but a non-finite output is not NaN"
    opposite = ((cy == POS_INF) & (cs == NEG_INF)) | ((cy == NEG_INF) & (cs == POS_INF))
    assert not opposite.any(), f"{int(opposite.sum())} outputs have the opposite sign of y*"
    if vname != "nan" and site in SIGNED:
        inf = (cs == POS_INF) | (cs == NEG_INF)
        same = cy[inf] == cs[inf]
        if lists_like:
            same |= cy[inf] == NAN
        assert bool(same.all()), f"{int((~same).sum())} outputs lost the sign of y*"
    assert torch.equal(y[fin], clean[fin]), "an output the injection does not reach changed"


@pytest.mark.parametrize("route,site", CASES)
def test_injection(route, site, monkeypatch):
    cfg, kind, tokens = ROUTES[route]
    if kind == "prep":
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    c = ctx(cfg)
    descs = None
    if kind in ("fused", "batch_fused"):
        descs = [c.desc(True), ctx("fused_1").desc(True), ctx("fused_2").desc(True)]
    x = c.dy if kind == "dgrad" else c.x[:max(tokens, 1)]
    clean = run_checked(kind, c, x, descs)
    for vname, v in VALUES.items():
        Li, xi, W, field = c.L, x, c.W, None
        if site == "x":
            xi = x.clone()
            xi[xi.shape[0] // 2, (2 * xi.shape[1]) // 3] = v
        else:
            kw, field = _injection(c, site, v)
            Li = inject(c.L, value=v, **kw)
            upload(c.desc(kind in LISTS_LIKE), Li, field)
            if field != "bias":
                W = torch.from_numpy(dense64(Li)).cuda()
        try:
            y = run(kind, c, xi, descs)
        finally:
            if field is not None:
                upload(c.desc(kind in LISTS_LIKE), c.L, field)
        if kind == "dequant":
            ys = W
        elif kind == "dgrad":
            ys = dgrad_star(Li, xi, W)
        elif kind in ("fused", "batch_fused"):
            ys = torch.cat([y_star(Li, xi, W)] + [y_star(ctx(n).L, xi, ctx(n).W) for n in ("fused_1", "fused_2")], 1)
        else:
            ys = y_star(Li, xi, W)
        check_classes(y, ys, clean, vname, site, kind in LISTS_LIKE)
        assert torch.equal(run(kind, c, x, descs), clean), "a clean call after the poisoned one differs"


def test_lists_graph_replay_poisoned_then_clean():
    """CUDA graph of the list path: one capture, replayed with clean, poisoned and clean x again"""
    from vptq_b200 import native
    c = ctx("i1004")
    d = c.desc(True)
    xbuf = c.x[:1].clone()
    y = torch.empty(1, c.L.out_features, dtype=xbuf.dtype, device="cuda")
    assert kernels_ok("lists", launched_kernels(lambda: native.quant_gemv(d, xbuf, y)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            native.quant_gemv(d, xbuf, y, flags=native.FLAG_PDL)
    g.replay()
    torch.cuda.synchronize()
    clean = y.clone()
    for vname, v in VALUES.items():
        xi = c.x[:1].clone()
        xi[0, 10] = v
        xbuf.copy_(xi)
        y.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        check_classes(y, y_star(c.L, xi, c.W), clean, vname, "x", True)
        xbuf.copy_(c.x[:1])
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, clean), vname


# ------------------------------------------------------------------------------------------------------------------
# range: fp16 overflow, the list kernel's fixed point, bf16 magnitudes
# ------------------------------------------------------------------------------------------------------------------
RANGE_KINDS = [("lists", 1), ("generic", 1), ("generic", 2), ("direct", 3), ("prep", 3)]


class Plain:
    """a context around a given layer (no isolation)"""

    def __init__(self, L):
        self.L, self._d = L, {}
        self.W = torch.from_numpy(dense64(L)).cuda()

    desc = Ctx.desc


def _const_layer(value, **kw):
    L = vo.make_layer(in_features=1024, out_features=264, vector_len=8, num_centroids=8192, enable_perm=False,
                      enable_norm=False, seed=5, **kw)
    L.centroids = encode(np.full(L.centroids.shape, value), L.dtype)
    return L


@pytest.mark.parametrize("sign", [1, -1])
def test_fp16_output_overflow(sign, monkeypatch):
    """every intermediate finite, y = sign * 71680 > 65504: +-inf from every route"""
    c = Plain(_const_layer(1.0))
    x = torch.full((3, 1024), 70.0 * sign, dtype=torch.float16, device="cuda")
    assert float(y_star(c.L, x[:1], c.W).min()) * sign > 65520
    for kind, tokens in RANGE_KINDS:
        if kind == "prep":
            monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
        y = run_checked(kind, c, x[:tokens])
        assert bool((y == sign * float("inf")).all()), (kind, tokens)


@pytest.mark.parametrize("kind,tokens,second_unit", [
    ("lists", 1, False), ("lists", 1, True),
    ("generic", 1, True), ("generic", 2, True), ("direct", 3, True), ("prep", 3, True)])
def test_fp16_past_the_fixed_point_range(kind, tokens, second_unit, monkeypatch):
    """three features of one tile at 60000 with entries of 60000 in slice 0 (and, with `second_unit`, a fourth one in
    slice 1): y* >= 1.08e10 = +inf in fp16.  The list kernel's sums pass 2^33: +inf or NaN, never -inf, never
    finite.  (A lone unit past 2^33 once saturated to 2^63 - 1, which still reads as +inf; a second unit on top of
    it wrapped the 64-bit sum.)"""
    L = _const_layer(60000.0)
    idx = L.meta["idx"]
    idx[0, :, :3] = idx[0, :, :3] % 4096                     # slice 0 for the three columns in every row
    idx[0, :, 3] = 4096 + idx[0, :, 3] % 4096                # slice 1 for the fourth
    L.indices = vo.pack_index(idx, L.index_bits)
    c = Plain(L)
    x = torch.zeros(3, 1024, dtype=torch.float16, device="cuda")
    x[:, :4 if second_unit else 3] = 60000.0
    assert bool((y_star(L, x, c.W) > 1e10).all())
    if kind == "prep":
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    y = run_checked(kind, c, x[:tokens])
    if kind == "lists":
        assert bool(((y == float("inf")) | torch.isnan(y)).all()), y
    else:
        assert bool((y == float("inf")).all()), (kind, tokens)


def _bf16_layer():
    return vo.make_layer(in_features=1024, out_features=264, vector_len=8, num_centroids=65536, num_res_centroids=256,
                         dtype="bf16", bias=True, llm_like=False, seed=6)


def test_bf16_large_activations(monkeypatch):
    """|x * scale| = 2^20 on four features (outputs ~1e6): every route within the bf16 bar"""
    L = _bf16_layer()
    F = [3, 100, 517, 1000]
    s = vo.to_f32(L.weight_scale, "bf16")
    s[F] = 1.0
    L.weight_scale = encode(s, "bf16")
    c = Plain(L)
    x = torch.from_numpy(vo.to_f32(vo.make_x(3, 1024, "bf16", seed=2), "bf16")).cuda().to(torch.bfloat16)
    x[:, F] = torch.tensor([2.0 ** 20, -2.0 ** 20, 2.0 ** 20, 2.0 ** 20], dtype=torch.bfloat16, device="cuda")
    ys = y_star(L, x, c.W)
    assert float(ys.abs().max()) > 1e5
    for kind, tokens in RANGE_KINDS:
        if kind == "prep":
            monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
        y = run_checked(kind, c, x[:tokens])
        err = parity_error(y.double().cpu().numpy(), ys[:tokens].cpu().numpy())
        print(f"\n[extreme] bf16 2^20 activations, {kind} x{tokens}: {err:.2e}")
        assert torch.isfinite(y).all() and err <= TOL["bf16"], (kind, tokens, err)


@pytest.mark.parametrize("kind,tokens", RANGE_KINDS)
def test_bf16_outputs_beyond_the_fixed_point_range(kind, tokens, monkeypatch):
    """one main entry element of 2^36, used once in index rows 1 and 7 with x = 1 there: outputs of ~2^36 >= 2^33.
    The list kernel returns NaN or a correct value in exactly those outputs and is right everywhere else; the other
    routes are right everywhere"""
    L = _bf16_layer()
    L = isolate(L, main={K_ARB: [1, 7]})
    e = 3
    L = inject(L, "C", 2.0 ** 36, k=K_ARB, e=e)
    x = torch.from_numpy(vo.to_f32(vo.make_x(3, 1024, "bf16", seed=3), "bf16")).cuda().to(torch.bfloat16)
    for r in (1, 7):
        f = feature_of(L, isolated_column(L, r, K_ARB))
        x[:, f] = 1.0
        s = vo.to_f32(L.weight_scale, "bf16")
        s[f] = 1.0
        L.weight_scale = encode(s, "bf16")
    c = Plain(L)
    ys = y_star(L, x, c.W)
    hit = torch.zeros(L.out_features, dtype=torch.bool, device="cuda")
    hit[[8 + e, 56 + e]] = True
    assert bool((ys[:, hit].abs() >= 2.0 ** 33).all()) and bool((ys[:, ~hit].abs() < 1e3).all())
    if kind == "prep":
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    y = run_checked(kind, c, x[:tokens]).double()
    ref = ys[:tokens]
    rest = float((y[:, ~hit] - ref[:, ~hit]).abs().max() / ref[:, ~hit].abs().max())
    assert rest <= TOL["bf16"], (kind, tokens, rest)
    rel = (y[:, hit] - ref[:, hit]).abs() / ref[:, hit].abs()
    ok = rel <= TOL["bf16"]
    if kind == "lists":
        ok |= torch.isnan(y[:, hit])
    assert bool(ok.all()), (kind, tokens, y[:, hit])


# ------------------------------------------------------------------------------------------------------------------
# power-of-two scaling
# ------------------------------------------------------------------------------------------------------------------
def _sweep_layer(dtype, in_features):
    """no bias; weight_scale in [1, 2), so x' = x * scale stays a normal 16-bit number for |x| >= 2^-14"""
    L = vo.make_layer(in_features=in_features, out_features=264, vector_len=8, num_centroids=65536,
                      num_res_centroids=256, dtype=dtype, seed=8)
    s = 1.0 + np.abs(0.1 * np.random.default_rng(1).standard_normal(in_features))
    L.weight_scale = encode(np.minimum(s, 1.9), dtype)
    return L


def _sweep_x(rows, cols, dtype, seed):
    """|x| drawn in [2^-6, 2^2], random signs: 2^k x stays normal for k in [-8, 8]"""
    rng = np.random.default_rng(seed)
    a = np.sign(rng.standard_normal((rows, cols))) * 2.0 ** rng.uniform(-6, 2, (rows, cols))
    return torch.from_numpy(vo.to_f32(encode(a, dtype), dtype)).cuda().to(torch.bfloat16 if dtype == "bf16" else torch.float16)


MIN_NORMAL = {torch.float16: 2.0 ** -14, torch.bfloat16: 2.0 ** -126}
MIN_SUB = {torch.float16: 2.0 ** -24, torch.bfloat16: 2.0 ** -133}


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("kind,tokens", [("generic", 1), ("generic", 2), ("direct", 3), ("prep", 3), ("dgrad", 3)])
def test_power_of_two_scaling_is_exact(kind, tokens, dtype, monkeypatch):
    if kind == "prep":
        monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    c = Plain(_sweep_layer(dtype, 1024))
    x = _sweep_x(tokens, c.L.out_features if kind == "dgrad" else 1024, dtype, seed=11)
    y0 = run_checked(kind, c, x)
    dt = x.dtype
    for k in range(-8, 9):
        yk = run(kind, c, x * 2.0 ** k)
        want = y0.double() * 2.0 ** k
        # both y(x) and y(2^k x) normal: bit for bit
        normal = (yk.double().abs() >= MIN_NORMAL[dt]) & (y0.double().abs() >= MIN_NORMAL[dt])
        assert torch.equal(yk.double()[normal], want[normal]), (kind, k, int((yk.double()[normal] != want[normal]).sum()))
        # an output that cancels to a subnormal: one subnormal step of whichever side is subnormal (scaled by 2^k when
        # it is y(x), whose rounding the comparison multiplies by 2^k)
        sub = ~normal
        bound = MIN_SUB[dt] * max(1.0, 2.0 ** k)
        assert float((yk.double()[sub] - want[sub]).abs().max() if sub.any() else 0.0) <= bound, (kind, k)


@pytest.mark.parametrize("dtype,ks", [("fp16", range(-8, 9)), ("bf16", range(-24, 9, 2))], ids=["fp16", "bf16"])
def test_lists_scaling_within_the_documented_floor(dtype, ks):
    """list kernel: |y - y*| <= TOL max|y*| + Q 2^-31 at every scale (bf16 down to outputs around 2^-25)"""
    c = Plain(_sweep_layer(dtype, 1004))
    Q = (c.L.num_centroids // 4096) * ((c.L.in_features + 4095) // 4096)
    x = _sweep_x(1, 1004, dtype, seed=12)
    run_checked("lists", c, x)
    smallest = float("inf")
    for k in ks:
        xk = x * 2.0 ** k
        y = run("lists", c, xk).double()
        ys = y_star(c.L, xk, c.W)
        bound = TOL[dtype] * float(ys.abs().max()) + Q * 2.0 ** -31
        err = float((y - ys).abs().max())
        smallest = min(smallest, float(ys.abs().max()))
        assert err <= bound, (k, err, bound)
    if dtype == "bf16":
        assert smallest < 2.0 ** -22            # the sweep reached outputs where only the floor holds


# ------------------------------------------------------------------------------------------------------------------
# the batched list kernel (2..8 tokens per launch)
# ------------------------------------------------------------------------------------------------------------------
def test_batch_padding_targets_of_every_slice():
    """padding lanes decode to entry s 4096 of their unit's slice and to residual entry 0: all sixteen such main
    entries and residual entry 0, confined to rows 1..18 and set to NaN, reach no other output"""
    L = vo.make_layer(vector_len=8, seed=4243, **CONFIGS["i1004"])
    rows = {s * 4096: [1 + s] for s in range(16)}
    L = isolate(L, main=rows, res={0: [17, 18]})
    P, bad = {}, L
    for k in rows:
        for e in range(8):
            bad = inject(bad, "C", float("nan"), k=k, e=e)
    for e in range(8):
        bad = inject(bad, "R", float("nan"), k=0, e=e)
    d_clean, d_bad = _batch.desc_of(L), _batch.desc_of(bad)
    hit = torch.zeros(L.out_features, dtype=torch.bool, device="cuda")
    hit[8:19 * 8] = True
    x = ctx("i1004").x
    for tokens in (2, 5, 8):
        clean = _batch.batch(d_clean, x[:tokens])
        names = launched_kernels(lambda: P.update(y=_batch.batch(d_bad, x[:tokens])))
        assert kernels_ok("batch", names), names
        y = P["y"]
        assert torch.equal(y[:, ~hit], clean[:, ~hit]), tokens
        assert bool(torch.isnan(y[:, hit]).all()), tokens
    _batch.head_zero()


@pytest.mark.parametrize("second_unit", [False, True])
def test_batch_fp16_past_the_fixed_point_range_one_token_of_five(second_unit):
    """token 2 of 5 hits entries of 60000 with x = 60000: alone, one slice-0 unit of three such terms (1.08e10, past
    2^33); with `second_unit`, two units (slices 0 and 1) of two terms each (7.2e9 each: inside 2^33, past
    2^33 / 2^ceil(log2 Q) = 2^32, and their 2^-30 fixed-point sum past 2^63).  +inf or NaN, never -inf or finite;
    the other four tokens (small x) bit-identical to a batch in which token 2 is small too"""
    L = _const_layer(60000.0)
    idx = L.meta["idx"]
    split = 2 if second_unit else 3
    idx[0, :, :split] = idx[0, :, :split] % 4096                      # slice 0
    idx[0, :, split:4] = 4096 + idx[0, :, split:4] % 4096             # slice 1
    L.indices = vo.pack_index(idx, L.index_bits)
    c = Plain(L)
    x = (_sweep_x(5, 1024, "fp16", seed=13) * 2.0 ** -10).half()
    clean = run_checked("batch", c, x)
    assert torch.isfinite(clean).all()
    xb = x.clone()
    xb[2, :4 if second_unit else 3] = 60000.0
    assert bool((y_star(L, xb[2:3], c.W) > 1e10).all())
    y = run_checked("batch", c, xb)
    assert bool(((y[2] == float("inf")) | torch.isnan(y[2])).all()), y[2]
    others = [0, 1, 3, 4]
    assert torch.equal(y[others], clean[others])
    _batch.head_zero()


def test_batch_bf16_outputs_beyond_the_fixed_point_range():
    """the 2^36 entry of test_bf16_outputs_beyond_the_fixed_point_range in a 5-token batch: NaN or correct at the hit
    outputs, correct everywhere else"""
    L = _bf16_layer()
    L = isolate(L, main={K_ARB: [1, 7]})
    e = 3
    L = inject(L, "C", 2.0 ** 36, k=K_ARB, e=e)
    x = torch.from_numpy(vo.to_f32(vo.make_x(5, 1024, "bf16", seed=3), "bf16")).cuda().to(torch.bfloat16)
    for r in (1, 7):
        f = feature_of(L, isolated_column(L, r, K_ARB))
        x[:, f] = 1.0
        s = vo.to_f32(L.weight_scale, "bf16")
        s[f] = 1.0
        L.weight_scale = encode(s, "bf16")
    c = Plain(L)
    ys = y_star(L, x, c.W)
    hit = torch.zeros(L.out_features, dtype=torch.bool, device="cuda")
    hit[[8 + e, 56 + e]] = True
    assert bool((ys[:, hit].abs() >= 2.0 ** 33).all())
    y = run_checked("batch", c, x).double()
    rest = float((y[:, ~hit] - ys[:, ~hit]).abs().max() / ys[:, ~hit].abs().max())
    assert rest <= TOL["bf16"], rest
    ok = ((y[:, hit] - ys[:, hit]).abs() / ys[:, hit].abs() <= TOL["bf16"]) | torch.isnan(y[:, hit])
    assert bool(ok.all()), y[:, hit]
    _batch.head_zero()


@pytest.mark.parametrize("dtype,ks", [("fp16", (-8, -6, -4, -2, 0, 3, 6, 8)), ("bf16", (-24, -19, -14, -9, -4, 0, 4, 8))],
                         ids=["fp16", "bf16"])
def test_batch_magnitude_spread(dtype, ks):
    """one 8-token batch whose tokens are scaled by 2^k, k spread over the range: each token within its own bar (the
    kernel's arithmetic in fp64; twice that against the exact product) and the same bits as that token alone"""
    c = Plain(_sweep_layer(dtype, 1004))
    q = _batch.q_of(1004, c.L.num_centroids)
    x = _sweep_x(8, 1004, dtype, seed=14) * torch.tensor([2.0 ** k for k in ks], device="cuda")[:, None]
    x = x.to(_dt(c.L))
    y = run_checked("batch", c, x)
    kstar, ys = _batch.kernel_star(c.L, x), y_star(c.L, x, c.W)
    for t in range(8):
        _batch.assert_close(y[t:t + 1], kstar[t:t + 1], dtype, q)
        _batch.assert_close(y[t:t + 1], ys[t:t + 1], dtype, q, factor=2.0)
        assert torch.equal(run("batch", c, x[t:t + 1].clone()), y[t:t + 1]), t
    _batch.head_zero()


def test_batch_graph_replay_poisoned_then_clean():
    """CUDA graph of the batched route: one capture of a 5-token launch, replayed with clean, poisoned and clean x"""
    from vptq_b200 import native
    c = ctx("i1004")
    d = c.desc(True)
    xbuf = c.x[:5].clone()
    y = torch.empty(5, c.L.out_features, dtype=xbuf.dtype, device="cuda")
    fb = native.FusedGemvBatch([d], [y])
    assert kernels_ok("batch", launched_kernels(lambda: fb(xbuf)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fb(xbuf, native.FLAG_PDL)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fb(xbuf, native.FLAG_PDL)
    g.replay()
    torch.cuda.synchronize()
    clean = y.clone()
    for vname, v in VALUES.items():
        xi = c.x[:5].clone()
        xi[3, 10] = v
        xbuf.copy_(xi)
        y.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        check_classes(y, y_star(c.L, xi, c.W), clean, vname, "x", True)
        xbuf.copy_(c.x[:5])
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, clean), vname
    _batch.head_zero()


# ------------------------------------------------------------------------------------------------------------------
# the vector-length-16 list kernel (1..4 tokens per launch; its class records are always on)
# ------------------------------------------------------------------------------------------------------------------
def _v16_const_layer(value, dtype="fp16"):
    """v = 16, K = 8192 (NS = 2, Q = 2: unit sums are admitted below 2^33 / 2 = 2^32), no perm / norm, every main
    entry `value`"""
    L = vo.make_layer(in_features=1024, out_features=264, vector_len=16, num_centroids=8192, enable_perm=False,
                      enable_norm=False, seed=15, dtype=dtype)
    L.centroids = encode(np.full(L.centroids.shape, value), L.dtype)
    return L


def _v16(L, x, ys=None):
    from _lists16 import only_kernel, run
    d = _lists16_desc(L)
    y = run(d, x) if ys is None else ys
    only_kernel(lambda: run(d, x, [y]), launches=1)
    torch.cuda.synchronize()
    return y


def _lists16_desc(L):
    from _lists16 import desc_of
    key = id(L)
    if key not in _V16:
        _V16.clear()
        _V16[key] = (L, desc_of(L))
    return _V16[key][1]


_V16 = {}


@pytest.mark.parametrize("second_unit", [False, True])
def test_v16_fp16_past_the_fixed_point_range_one_token_of_four(second_unit):
    """token 2 of 4 hits entries of 60000 with x = 60000: alone, one slice-0 unit of three such terms (1.08e10, past
    2^33); with `second_unit`, two units (slices 0 and 1) of two terms each (7.2e9 each: inside 2^33, past
    2^33 / 2^ceil(log2 Q) = 2^32, and their 2^-30 fixed-point sum past 2^63).  +inf or NaN, never -inf or finite;
    the other three tokens bit-identical to a launch in which token 2 is small too"""
    L = _v16_const_layer(60000.0)
    idx = L.meta["idx"]
    split = 2 if second_unit else 3
    idx[0, :, :split] = idx[0, :, :split] % 4096                      # slice 0
    idx[0, :, split:4] = 4096 + idx[0, :, split:4] % 4096             # slice 1
    L.indices = vo.pack_index(idx, L.index_bits)
    W = torch.from_numpy(dense64(L)).cuda()
    x = (_sweep_x(4, 1024, "fp16", seed=13) * 2.0 ** -10).half()
    clean = _v16(L, x).clone()
    assert torch.isfinite(clean).all()
    xb = x.clone()
    xb[2, :4 if second_unit else 3] = 60000.0
    assert bool((y_star(L, xb[2:3], W) > 1e10).all())
    y = _v16(L, xb)
    assert bool(((y[2] == float("inf")) | torch.isnan(y[2])).all()), y[2]
    others = [0, 1, 3]
    assert torch.equal(y[others], clean[others])
    assert torch.equal(_v16(L, x), clean)                              # (the records were cleared)
    _batch.head_zero()


@pytest.mark.parametrize("sign", [1, -1])
def test_v16_fp16_output_overflow(sign):
    """every unit sum well inside the fixed point, y = sign * 71680 > 65504: +-inf at every token count"""
    L = _v16_const_layer(1.0)
    x = torch.full((4, 1024), 70.0 * sign, dtype=torch.float16, device="cuda")
    assert float(y_star(L, x[:1]).min()) * sign > 65520
    for tokens in (1, 2, 3, 4):
        y = _v16(L, x[:tokens].clone())
        assert bool((y == sign * float("inf")).all()), tokens
    _batch.head_zero()


def test_v16_bf16_outputs_beyond_the_fixed_point_range():
    """one main entry element of 2^36, used once in index rows 1 and 7 with x = 1 there: outputs of ~2^36 >= 2^33 in
    all four tokens.  NaN or correct there, correct everywhere else"""
    L = vo.make_layer(in_features=1024, out_features=264, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      dtype="bf16", bias=True, llm_like=False, seed=6)
    L = isolate(L, main={K_ARB: [1, 7]})
    e = 3
    L = inject(L, "C", 2.0 ** 36, k=K_ARB, e=e)
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 1024, "bf16", seed=3), "bf16")).cuda().to(torch.bfloat16)
    for r in (1, 7):
        f = feature_of(L, isolated_column(L, r, K_ARB))
        x[:, f] = 1.0
        s = vo.to_f32(L.weight_scale, "bf16")
        s[f] = 1.0
        L.weight_scale = encode(s, "bf16")
    ys = y_star(L, x)
    hit = torch.zeros(L.out_features, dtype=torch.bool, device="cuda")
    hit[[16 + e, 112 + e]] = True
    assert bool((ys[:, hit].abs() >= 2.0 ** 33).all()) and bool((ys[:, ~hit].abs() < 1e3).all())
    y = _v16(L, x).double()
    rest = float((y[:, ~hit] - ys[:, ~hit]).abs().max() / ys[:, ~hit].abs().max())
    assert rest <= TOL["bf16"], rest
    ok = ((y[:, hit] - ys[:, hit]).abs() / ys[:, hit].abs() <= TOL["bf16"]) | torch.isnan(y[:, hit])
    assert bool(ok.all()), y[:, hit]
    _batch.head_zero()


def _v16_sweep_layer(dtype):
    L = vo.make_layer(in_features=1004, out_features=264, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      dtype=dtype, seed=8)
    s = 1.0 + np.abs(0.1 * np.random.default_rng(1).standard_normal(1004))
    L.weight_scale = encode(np.minimum(s, 1.9), dtype)
    return L


@pytest.mark.parametrize("dtype,ks", [("fp16", (-8, -2, 3, 8)), ("bf16", (-24, -9, 0, 8))], ids=["fp16", "bf16"])
def test_v16_magnitude_spread(dtype, ks):
    """one 4-token launch whose tokens are scaled by 2^k, k spread over the range: each token within its own bar (the
    kernel's arithmetic in fp64; twice that against the exact product) and the same bits as that token alone"""
    L = _v16_sweep_layer(dtype)
    q = _batch.q_of(1004, 65536)
    x = _sweep_x(4, 1004, dtype, seed=14) * torch.tensor([2.0 ** k for k in ks], device="cuda")[:, None]
    x = x.to(_dt(L))
    y = _v16(L, x)
    kstar, ys = _batch.kernel_star(L, x), y_star(L, x)
    for t in range(4):
        _batch.assert_close(y[t:t + 1], kstar[t:t + 1], dtype, q)
        _batch.assert_close(y[t:t + 1], ys[t:t + 1], dtype, q, factor=2.0)
        assert torch.equal(_v16(L, x[t:t + 1].clone()), y[t:t + 1]), t
    _batch.head_zero()


@pytest.mark.parametrize("dtype,ks", [("fp16", range(-8, 9)), ("bf16", range(-24, 9, 2))], ids=["fp16", "bf16"])
def test_v16_scaling_within_the_documented_floor(dtype, ks):
    """|y - y*| <= TOL max|y*| + Q 2^-31 at every scale, 1 and 3 tokens (bf16 down to outputs around 2^-25)"""
    L = _v16_sweep_layer(dtype)
    Q = _batch.q_of(1004, 65536)
    x = _sweep_x(3, 1004, dtype, seed=12)
    W = torch.from_numpy(dense64(L)).cuda()
    smallest = float("inf")
    for k in ks:
        xk = x * 2.0 ** k
        for tokens in (1, 3):
            y = _v16(L, xk[:tokens].clone()).double()
            ys = y_star(L, xk[:tokens], W)
            bound = TOL[dtype] * float(ys.abs().max()) + Q * 2.0 ** -31
            err = float((y - ys).abs().max())
            smallest = min(smallest, float(ys.abs().max()))
            assert err <= bound, (k, tokens, err, bound)
    if dtype == "bf16":
        assert smallest < 2.0 ** -22            # the sweep reached outputs where only the floor holds
    _batch.head_zero()


def test_v16_graph_replay_clean_poisoned_clean():
    """CUDA graph of one 4-token v = 16 launch, replayed with clean, poisoned (NaN, +inf, -inf in one feature of
    token 3) and clean x: the poisoned token's classes those of the kernel's arithmetic in fp64, the other tokens and
    every clean replay the bits of the first clean replay"""
    from _lists16 import run
    from vptq_b200 import native
    L = vo.make_layer(in_features=1004, out_features=264, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      seed=17, bias=True)
    d = _lists16_desc(L)
    x0 = torch.from_numpy(vo.to_f32(vo.make_x(4, 1004, "fp16", seed=3), "fp16")).cuda().half()
    xbuf = torch.zeros(4, 1008, dtype=torch.float16, device="cuda")[:, :1004]
    xbuf.copy_(x0)
    y = torch.empty(4, 264, dtype=torch.float16, device="cuda")
    fb = native.FusedGemvLists16([d], [y])
    eager = run(d, x0.clone()).clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fb(xbuf, native.FLAG_PDL)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            fb(xbuf, native.FLAG_PDL)
    y.fill_(0)
    g.replay()
    torch.cuda.synchronize()
    clean = y.clone()
    assert torch.equal(clean, eager)
    for vname, v in VALUES.items():
        xi = x0.clone()
        xi[3, 10] = v
        xbuf.copy_(xi)
        y.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y[:3], clean[:3]), vname
        assert torch.equal(classify(y[3]), classify(_batch.kernel_star(L, xi)[3])), vname
        assert not torch.isfinite(y[3]).any(), vname
        xbuf.copy_(x0)
        y.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, clean), vname
    _batch.head_zero()
