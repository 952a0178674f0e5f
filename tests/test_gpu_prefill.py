"""GPU parity of the prefill path (tokens >= 3): prep kernel + quantised-order dequant + wgmma GEMM,
through VQuantLinear.forward -> vptq.ops.quant_gemm -> C ABI, against the oracle.

Bar: max|y - y*| / max|y*| <= 1e-3 (fp16), 4e-3 (bf16); y* = fp64-accumulated math on the identical
tensors (oracle/vptq_oracle.py), and the reference's own python output for the golden fixtures.
"""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _util import TOL, golden_names, load_golden, parity_error

pytestmark = pytest.mark.gpu


def forward(L, x_np):
    from _gpu import from_t, make_module, x_to_t
    m = make_module(L)
    y = m(x_to_t(x_np, L))
    torch.cuda.synchronize()
    return from_t(y)


@pytest.mark.parametrize("name", golden_names())
def test_prefill_golden(name):
    L, x, ref = load_golden(name)          # 3 tokens -> the GEMM route (reference rule: tokens >= 3)
    y = forward(L, x)
    assert y.shape == ref["y_ref"].shape
    assert parity_error(y, vo.quant_gemm(x, L)) <= TOL[L.dtype]
    assert parity_error(y, ref["y_ref"]) <= TOL[L.dtype]


CASES = {
    "k65536_r256": (dict(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256), 200),
    "k256_multi_tile": (dict(in_features=2048, out_features=384, vector_len=8, num_centroids=256), 300),
    "ragged_everything": (dict(in_features=1000, out_features=344, vector_len=8, num_centroids=4096, num_res_centroids=32), 131),
    "outliers_bias": (dict(in_features=1024 + 128, out_features=512, vector_len=8, num_centroids=4096, num_res_centroids=256,
                           outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096, bias=True), 64),
    "groups4": (dict(in_features=2048, out_features=256, vector_len=8, num_centroids=1024, num_res_centroids=256,
                     num_codebooks=4), 33),
    "v6_pad": (dict(in_features=512, out_features=250, vector_len=6, num_centroids=4096), 17),
    "v16": (dict(in_features=512, out_features=256, vector_len=16, num_centroids=4096, num_res_centroids=16), 5),
    "noperm_nonorm": (dict(in_features=512, out_features=256, vector_len=8, num_centroids=256, enable_perm=False,
                           enable_norm=False, bias=True), 3),
    "bf16": (dict(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256,
                  dtype="bf16"), 150),
    "bf16_reftest_dist": (dict(in_features=1024, out_features=256, vector_len=8, num_centroids=8192, num_res_centroids=256,
                               dtype="bf16", llm_like=False), 40),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_prefill_vs_oracle(name):
    kw, tokens = CASES[name]
    L = vo.make_layer(seed=77, **kw)
    x = vo.make_x(tokens, L.in_features, L.dtype, seed=5)
    y = forward(L, x)
    err = parity_error(y, vo.quant_gemm(x, L))
    assert err <= TOL[L.dtype], f"{name}: {err:.3e}"


def test_prefill_3d_input_and_agreement_with_gemv():
    """[batch, seq, I] input; the GEMM route and the GEMV route agree on the same tokens."""
    from _gpu import make_module, x_to_t
    L = vo.make_layer(in_features=1024, out_features=512, vector_len=8, num_centroids=4096, num_res_centroids=256, seed=3)
    m = make_module(L)
    x_np = vo.make_x(8, L.in_features, L.dtype, seed=9)
    x = x_to_t(x_np, L)
    y_gemm = m(x.view(2, 4, -1))
    assert y_gemm.shape == (2, 4, 512)
    y_gemv = torch.cat([m(x[i:i + 2]) for i in range(0, 8, 2)])
    torch.cuda.synchronize()
    a, b = y_gemm.view(8, -1).float().cpu().numpy(), y_gemv.float().cpu().numpy()
    assert parity_error(a, b) <= 1e-3
    assert parity_error(a, vo.quant_gemm(x_np, L)) <= 1e-3


def test_prefill_large_tokens_property():
    """BASELINE configs[2] scale (seq 2048 x batch 4) on one 4096x4096 layer: too big for the numpy
    oracle in a unit test, so check linearity instead: f(a) + f(b) - f(0)*... via f(x1 + x2) = f(x1) + f(x2) - f(0)."""
    from _gpu import make_module
    L = vo.make_layer(in_features=4096, out_features=4096, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=8)
    m = make_module(L)
    g = torch.Generator(device="cuda").manual_seed(0)
    x1 = (0.5 * torch.randn(8192, 4096, device="cuda", generator=g)).half()
    x2 = (0.5 * torch.randn(8192, 4096, device="cuda", generator=g)).half()
    y1, y2, y12 = m(x1).float(), m(x2).float(), m((x1.float() + x2.float()).half()).float()
    y0 = m(torch.zeros(3, 4096, device="cuda", dtype=torch.float16)).float()[0]
    torch.cuda.synchronize()
    scale = y12.abs().max()
    # inputs were rounded to fp16 once more in x1 + x2; allow for that
    assert ((y1 + y2 - y0) - y12).abs().max() <= 4e-3 * scale
    # spot-check 64 random tokens against the GEMV route
    idx = torch.randint(0, 8192, (64,), generator=torch.Generator().manual_seed(1)).tolist()
    ref = torch.cat([m(x1[i:i + 1]) for i in idx]).float()
    assert (ref - y1[idx]).abs().max() <= 1e-3 * scale


def test_prep_path_still_matches(monkeypatch):
    """VPTQ_B200_GEMM_PREP=1 forces the round-1 route (x' prep pass + quantised-order Wq) for a shape that takes the
    prep-free route by default: both must match the oracle."""
    from _gpu import from_t, make_module, x_to_t
    L = vo.make_layer(in_features=1024, out_features=512, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=17)
    m = make_module(L)
    x_np = vo.make_x(200, 1024, "fp16", seed=3)
    x = x_to_t(x_np, L)
    y_star = vo.quant_gemm(x_np, L)
    y_direct = from_t(m(x))
    monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    y_prep = from_t(m(x))
    for y in (y_direct, y_prep):
        assert parity_error(y, y_star) <= TOL["fp16"]
