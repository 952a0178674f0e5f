"""CPU checks of the probe simulation (tests/_probe.py) against the oracle's dequant: the GPU probe tests trust it to
the last bit, so it is pinned here on every golden fixture and on synthetic layers with outliers, groups and
several vector lengths."""
import dataclasses

import numpy as np
import pytest

import vptq_oracle as vo
from _probe import probe_expect
from _util import golden_names, load_golden

SYNTH = {
    "outliers_v4": dict(in_features=512 + 64, out_features=200, vector_len=4, num_centroids=1024, num_res_centroids=16,
                        outlier_size=64, outlier_vector_len=4, num_outlier_centroids=256, bias=True),
    "groups4_v6": dict(in_features=768, out_features=250, vector_len=6, num_centroids=4096, num_codebooks=4),
    "v12_bf16": dict(in_features=384, out_features=120, vector_len=12, num_centroids=256, num_res_centroids=256,
                     dtype="bf16", bias=True),
    "v16_noperm": dict(in_features=256, out_features=64, vector_len=16, num_centroids=512, enable_perm=False),
    "k65536_r256": dict(in_features=1024, out_features=264, vector_len=8, num_centroids=65536, num_res_centroids=256),
    "k8192_bf16_bias": dict(in_features=1000, out_features=72, vector_len=8, num_centroids=8192, num_res_centroids=16,
                            dtype="bf16", bias=True, llm_like=False),
}


def _layers():
    for name in golden_names():
        yield name, load_golden(name)[0]
    for name, kw in SYNTH.items():
        yield name, vo.make_layer(seed=13, **kw)


LAYERS = dict(_layers())


def _ulp16(a, dtype):
    """spacing of the 16-bit type at |a| (fp32 array)"""
    mant = 10 if dtype == "fp16" else 7
    e = np.floor(np.log2(np.maximum(np.abs(a), 2.0 ** -24 if dtype == "fp16" else 2.0 ** -126)))
    return 2.0 ** (e - mant)


def _dense(L):
    """vo.dequant (+ bias, in fp32) rounded once: the generic route's arithmetic, written independently"""
    W = vo.dequant(L)
    if L.bias is not None:
        W = W + vo.to_f32(L.bias, L.dtype)[:, None]
    return vo.round_to(W, L.dtype).T


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_generic_probe_is_the_rounded_oracle_dequant(name):
    L = LAYERS[name]
    e = probe_expect(L, "generic")
    assert e.shape == (L.in_features, L.out_features)
    np.testing.assert_array_equal(e, _dense(L))


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_other_routes_differ_from_generic_only_by_their_roundings(name):
    L = LAYERS[name]
    g = probe_expect(L, "generic").astype(np.float64)
    s = vo.to_f32(L.weight_scale, L.dtype) if L.weight_scale is not None else np.ones(L.in_features, np.float32)
    bare = dataclasses.replace(L, weight_scale=None, weight_bias=None, bias=None, meta=dict(L.meta))
    cr = np.abs(probe_expect(bare, "generic").astype(np.float64))    # |C + R| to 16 bits
    two_out_ulps = 2 * np.maximum(_ulp16(g, L.dtype), 2.0 ** -24)
    routes = ["direct", "prep"] + (["lists"] if L.num_codebooks == 1 and not L.enable_outlier else [])
    for route in routes:
        e = probe_expect(L, route).astype(np.float64)
        slack = two_out_ulps.copy()
        if route == "direct":   # the weight is rounded to 16 bits before the bias is added
            nobias = dataclasses.replace(L, bias=None, meta=dict(L.meta))
            slack += _ulp16(probe_expect(nobias, "generic"), L.dtype)
        if route in ("prep", "lists"):
            # C + R rounded to 16 bits (prep: both dtypes; lists: fp16); x' = s needs no rounding
            slack += np.abs(s[:, None]) * 0.5 * _ulp16(cr + 1e-30, L.dtype)
            slack += 2.0 ** -29
        assert np.all(np.abs(e - g) <= slack), (name, route, float(np.max(np.abs(e - g) - slack)))
        # the roundings move few outputs, and none by more than an output ulp or two
        assert np.mean(e == g) > 0.5, (name, route)


def test_probe_expect_sees_a_single_index_change():
    """The simulation itself must resolve one wrong codebook entry in one column (what a GPU probe catches)."""
    L = vo.make_layer(in_features=512, out_features=64, vector_len=8, num_centroids=65536, num_res_centroids=16, seed=3)
    base = {r: probe_expect(L, r) for r in ("generic", "lists")}
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    idx = idx.copy()
    idx[0, 5, 100] ^= 1
    L2 = vo.make_layer(in_features=512, out_features=64, vector_len=8, num_centroids=65536, num_res_centroids=16, seed=3)
    L2.indices = vo.pack_index(idx, L.index_bits, ridx, L.res_bits)
    f = int(L.perm[100])
    for r, b in base.items():
        moved = probe_expect(L2, r) != b
        assert moved[f, 40:48].any() and moved.sum() == moved[f, 40:48].sum(), r
