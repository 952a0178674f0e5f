"""CPU checks of the extreme-value reference (tests/_extreme.py): its dense weight and its y* are compared with
oracle/torch_port.py, independent code in fp32, with inf / NaN injected into every kind of layer tensor and into x.
The class of every element (finite / +inf / -inf / NaN) must match exactly, finite values to fp32 rounding.  Also:
the layers built by `isolate` use the chosen entry in exactly the chosen rows."""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _extreme import VALUES, classify, copy_layer, dense64, ew_matmul, inject, isolate, rows_using, y_star
from _util import golden_names, load_golden

SYNTH = {
    "outliers_groups_v4": dict(in_features=1000 + 128, out_features=250, vector_len=4, num_centroids=4096,
                               num_res_centroids=16, num_codebooks=2, outlier_size=128, outlier_vector_len=4,
                               num_outlier_centroids=256, bias=True),
    "k65536_r256_bias": dict(in_features=1004, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True),
    "k8192_bf16": dict(in_features=1000, out_features=72, num_centroids=8192, num_res_centroids=16, dtype="bf16",
                       bias=True, llm_like=False),
}


def _port(L):
    f = (lambda a: None if a is None else (torch.from_numpy(np.asarray(a, dtype=np.float16).copy()) if L.dtype == "fp16"
         else torch.from_numpy(np.asarray(a, dtype=np.uint16).copy()).view(torch.bfloat16)))
    u = lambda a: None if a is None else torch.from_numpy(np.asarray(a, dtype=np.uint16).copy()).view(torch.int16)
    return dict(in_features=L.in_features, out_features=L.out_features, vector_len=L.vector_len,
                num_centroids=L.num_centroids, num_res_centroids=L.num_res_centroids, num_codebooks=L.num_codebooks,
                group_size=L.group_size, outlier_size=L.outlier_size if L.enable_outlier else 0,
                outlier_vector_len=L.outlier_vector_len, num_outlier_centroids=L.num_outlier_centroids,
                indices=torch.from_numpy(L.indices.copy()), centroids=f(L.centroids), res_centroids=f(L.res_centroids),
                outlier_indices=u(L.outlier_indices), outlier_centroids=f(L.outlier_centroids), perm=u(L.perm),
                weight_scale=f(L.weight_scale), weight_bias=f(L.weight_bias), bias=f(L.bias))


def _port_w(L):
    import torch_port as tp
    return tp.dequant(_port(L)).double()


def _same(a, b, rel=2.0 ** -21):
    """same class everywhere; finite values equal to fp32 rounding (b was computed in fp32)"""
    ca, cb = classify(a), classify(b)
    assert torch.equal(ca, cb), f"{int((ca != cb).sum())} elements differ in class"
    fin = ca == 0
    scale = max(float(a[fin].abs().max()) if fin.any() else 0.0, 1e-30)
    assert float((a[fin] - b[fin]).abs().max() if fin.any() else 0.0) <= rel * scale


def _sites(L):
    """(site, kwargs) injections that exist in L"""
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)   # entries row 0 uses
    out = [("C", dict(k=int(idx[0, 0, 1]), e=L.vector_len - 1)), ("scale", dict(f=L.in_features // 3)),
           ("wbias", dict(f=L.in_features - 1))]
    if L.res_bits:
        out.append(("R", dict(k=int(ridx[0, 0, 2]), e=1)))
    if L.enable_outlier:
        out.append(("Col", dict(k=int(L.outlier_indices[0, 0, 0]), e=0)))
    if L.bias is not None:
        out.append(("bias", dict(o=L.out_features - 1)))
    return [(s, kw) for s, kw in out if s not in ("scale", "wbias") or L.weight_scale is not None]


def _layers():
    for name in golden_names():
        yield name, load_golden(name)[0]
    for name, kw in SYNTH.items():
        yield name, vo.make_layer(seed=21, **kw)


LAYERS = dict(_layers())


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_dense64_matches_torch_port_with_injections(name):
    L = LAYERS[name]
    _same(torch.from_numpy(dense64(L)), _port_w(L))
    for site, kw in _sites(L):
        for vname, v in VALUES.items():
            Li = inject(L, site, v, **kw)
            if site == "bias":
                continue           # the weight does not hold the bias
            W = torch.from_numpy(dense64(Li))
            _same(W, _port_w(Li))
            assert not torch.isfinite(W).all(), (site, vname)


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_y_star_matches_torch_port_with_injections(name):
    L = LAYERS[name]
    x0 = torch.from_numpy(vo.to_f32(vo.make_x(3, L.in_features, L.dtype, seed=4), L.dtype)).to(
        torch.float16 if L.dtype == "fp16" else torch.bfloat16)
    cases = [(L, x0, None)] + [(inject(L, s, v, **kw), x0, (s, vn)) for s, kw in _sites(L) for vn, v in VALUES.items()]
    for vn, v in VALUES.items():
        x = x0.clone()
        x[1, L.in_features // 2] = v
        cases.append((L, x, ("x", vn)))
    for Li, x, what in cases:
        ys = y_star(Li, x)
        W = _port_w(Li)
        b = None if Li.bias is None else torch.from_numpy(vo.to_f32(Li.bias, Li.dtype).astype(np.float64))
        ref = ew_matmul(x.double(), W, b)
        _same(ys, ref, rel=2.0 ** -18)
        if what is not None:
            assert not torch.isfinite(ys).all(), what
        if what is not None and what[0] == "x":    # only the poisoned token
            assert torch.isfinite(ys[[0, 2]]).all() and not torch.isfinite(ys[1]).any(), what


def test_ew_matmul_keeps_ieee_zero_times_inf():
    a = torch.tensor([[0.0, 1.0], [1.0, 1.0]], dtype=torch.float64)
    b = torch.tensor([[float("inf"), 1.0], [float("inf"), float("-inf")], [2.0, 3.0]], dtype=torch.float64)
    y = ew_matmul(a, b, budget=2)
    assert torch.isnan(y[0, 0]) and torch.isnan(y[0, 1]) and y[0, 2] == 3.0
    assert y[1, 0] == float("inf") and torch.isnan(y[1, 1]) and y[1, 2] == 5.0


ISOLATE = {
    "k65536_r256": dict(in_features=1004, out_features=264, num_centroids=65536, num_res_centroids=256),
    "groups2_v4_outliers": SYNTH["outliers_groups_v4"],
}


@pytest.mark.parametrize("name", sorted(ISOLATE))
def test_isolated_entries_decode_to_their_rows_only(name):
    L = vo.make_layer(seed=22, **ISOLATE[name])
    K, v = L.num_centroids, L.vector_len
    k_pad = 4096 if K >= 8192 else 0
    main = {0: [1, 9], 77: [2, 5, 11], k_pad: [3, 20]} if k_pad else {0: [1, 9], 77: [2, 5, 11]}
    res = {0: [4, 6], 5: [7, 12]}
    Li = isolate(L, main=main, res=res)
    for k, rows in main.items():
        assert rows_using(Li, k) == {r: 1 for r in rows}, k
    for k, rows in res.items():
        assert rows_using(Li, k, residual=True) == {r: 1 for r in rows}, k
    # and the oracle agrees: NaN in element e of the entry reaches output r * v + e of those rows, in one column
    W0 = dense64(Li)
    for site, spec in (("C", main), ("R", res)):
        for k, rows in spec.items():
            e = 1
            W = dense64(inject(Li, site, float("nan"), k=k, e=e))
            bad_r, bad_c = np.nonzero(np.isnan(W))
            assert sorted(bad_r.tolist()) == [r * v + e for r in rows if r * v + e < L.out_features], (site, k)
            assert len(set(bad_c.tolist())) == len(bad_c)        # one column per row
            ok = ~np.isnan(W)
            np.testing.assert_array_equal(W[ok], W0[ok])


def test_copy_layer_does_not_share_arrays():
    L = vo.make_layer(in_features=64, out_features=16, num_centroids=256, seed=1)
    Li = inject(L, "C", float("inf"), k=3)
    assert np.isfinite(vo.to_f32(L.centroids, L.dtype)).all()
    assert not np.isfinite(vo.to_f32(Li.centroids, Li.dtype)).all()
    C = copy_layer(L)
    C.meta["idx"][0, 0, 0] += 1
    assert C.meta["idx"][0, 0, 0] != L.meta["idx"][0, 0, 0]
