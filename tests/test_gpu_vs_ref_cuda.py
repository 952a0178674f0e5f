"""GPU-side anchor: our kernels vs the UNMODIFIED reference CUDA kernels on identical tensors.

What the reference kernels returned for these seeded cases (built by oracle/build_ref.sh and run on an H100 by
oracle/make_ref_cuda_golden.py) is stored in tests/golden/ref_cuda/outputs.npz as raw 16-bit words: the GEMV
outputs in full and a fixed, seeded sample of the dequantised weights.  The layers, activations and sample
positions are regenerated here from their seeds.

north_star: "Outputs match the reference kernels on identical (indices, centroids,
residual_centroids, perm, outliers, x) within 1e-3 relative fp16".  The reference GEMV accumulates
four columns per thread in fp16 (csrc/kernels/quant_gemv.cuh:34,140-141), so its own distance to
exact arithmetic is a few 1e-4; both distances are asserted.
"""
import os

import numpy as np
import pytest

import vptq_oracle as vo
from _util import GOLDEN_DIR, parity_error

pytestmark = pytest.mark.gpu
REF_GOLDEN = os.path.join(GOLDEN_DIR, "ref_cuda", "outputs.npz")
GEMV_SEED, DEQUANT_SEED = 2024, 2025


def sample_positions(size):
    """flat positions of the stored dequantised-weight sample (4096 of the matrix's elements)"""
    return np.sort(np.random.default_rng(0).choice(size, 8192, replace=False))[::2]


def to_bits(a, dtype):
    """16-bit values held in float32 -> their uint16 words (lossless)"""
    return np.asarray(a, np.float32).astype(np.float16).view(np.uint16) if dtype == "fp16" else vo.f32_to_bf16_bits(a)


def from_bits(w, dtype):
    return w.view(np.float16).astype(np.float32) if dtype == "fp16" else vo.bf16_bits_to_f32(w)


@pytest.fixture(scope="module")
def ref():
    return np.load(REF_GOLDEN, allow_pickle=False)


CASES = {
    "llama3_k65536_r256": dict(in_features=4096, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256),
    "k65536_r0": dict(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536),
    "cfg1_k256": dict(in_features=4096, out_features=4096, vector_len=8, num_centroids=256),
    "k4096_r4096_v12": dict(in_features=1536, out_features=768, vector_len=12, num_centroids=4096, num_res_centroids=4096),
    "outliers": dict(in_features=2048 + 128, out_features=1024, vector_len=8, num_centroids=4096, num_res_centroids=256,
                     outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096, bias=True),
    "bf16": dict(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256, dtype="bf16"),
}
DEQUANT_CASES = ["llama3_k65536_r256", "outliers", "bf16"]


def ref_tensors(L, m):
    G, v = L.num_codebooks, L.vector_len
    cent = m.centroids.weight.view(G, L.num_centroids, v)
    rcent = m.res_centroids.weight.view(G, L.num_res_centroids, v) if L.res_bits else None
    ocent = m.outlier_centroids.weight.view(1, L.num_outlier_centroids, L.outlier_vector_len) if L.enable_outlier else None
    return cent, rcent, ocent


@pytest.mark.parametrize("name", sorted(CASES))
def test_gemv_matches_reference_cuda(ref, name):
    import torch
    from _gpu import from_t, make_module, x_to_t
    L = vo.make_layer(seed=GEMV_SEED, **CASES[name])
    m = make_module(L)
    tol = 1e-3 if L.dtype == "fp16" else 8e-3
    for tokens in (1, 2):
        x_np = vo.make_x(tokens, L.in_features, L.dtype, seed=tokens)
        x = x_to_t(x_np, L)
        y_ours = from_t(m(x))
        y_ref = from_bits(ref[f"gemv__{name}__t{tokens}"], L.dtype)
        torch.cuda.synchronize()
        y_star = vo.quant_gemm(x_np, L)
        e_ours = parity_error(y_ours, y_star)
        assert e_ours <= tol
        if not np.isfinite(y_ref).all():
            # the reference kernel has returned NaN for the outlier configuration in some runs and finite values
            # in others on the same inputs; nothing to compare with then -- our distance to exact arithmetic is
            # asserted above
            print(f"{name} tokens={tokens}: ours-vs-exact {e_ours:.2e}  reference kernel output is not finite, skipped")
            continue
        assert y_ours.shape == y_ref.shape
        e_ref, e_mut = parity_error(y_ref, y_star), parity_error(y_ours, y_ref)
        print(f"{name} tokens={tokens}: ours-vs-exact {e_ours:.2e}  ref-vs-exact {e_ref:.2e}  ours-vs-ref {e_mut:.2e}")
        assert e_mut <= max(tol, 2 * e_ref), (e_mut, e_ref)


@pytest.mark.parametrize("name", ["llama3_k65536_r256", "k65536_r0", "bf16"])
def test_batched_decode_matches_reference_cuda(ref, name):
    """the batched list kernel (2 tokens, one launch) against the same record, with the same bars"""
    import torch
    from _batch import BATCH, batch, desc_of
    from _gpu import from_t, x_to_t
    from _probe import launched_kernels, ran
    L = vo.make_layer(seed=GEMV_SEED, **CASES[name])
    d = desc_of(L)
    tol = 1e-3 if L.dtype == "fp16" else 8e-3
    x_np = vo.make_x(2, L.in_features, L.dtype, seed=2)
    x = x_to_t(x_np, L)
    out = [torch.empty(2, L.out_features, dtype=x.dtype, device="cuda")]
    names = launched_kernels(lambda: batch(d, x, out))
    assert len(names) == 1 and ran(names, BATCH), names
    torch.cuda.synchronize()
    y_ours = from_t(out[0])
    y_ref = from_bits(ref[f"gemv__{name}__t2"], L.dtype)
    y_star = vo.quant_gemm(x_np, L)
    e_ours = parity_error(y_ours, y_star)
    assert e_ours <= tol
    assert np.isfinite(y_ref).all() and y_ours.shape == y_ref.shape
    e_ref, e_mut = parity_error(y_ref, y_star), parity_error(y_ours, y_ref)
    print(f"{name} batched x2: ours-vs-exact {e_ours:.2e}  ref-vs-exact {e_ref:.2e}  ours-vs-ref {e_mut:.2e}")
    assert e_mut <= max(tol, 2 * e_ref), (e_mut, e_ref)


@pytest.mark.parametrize("name", DEQUANT_CASES)
def test_dequant_matches_reference_cuda(ref, name):
    from _gpu import from_t, make_module
    L = vo.make_layer(seed=DEQUANT_SEED, **CASES[name])
    m = make_module(L)
    W = from_t(m.dequant())
    assert W.shape == tuple(ref[f"dequant__{name}__shape"])
    W = W.reshape(-1)[sample_positions(W.size)]
    W_ref = from_bits(ref[f"dequant__{name}__values"], L.dtype)
    # the reference rounds C+R to 16 bit and then fma-rounds again (csrc/kernels/dequant.cuh:87,98);
    # ours evaluates in fp32 and rounds once.  |diff| <= ulp * (|W| + 0.5*|C+R|*|scale|), and
    # |C+R|*|scale| <= |W| + |wbias|.
    ulp = 2.0 ** -10 if L.dtype == "fp16" else 2.0 ** -7
    wb = np.abs(vo.to_f32(L.weight_bias, L.dtype)).max()
    bound = 2 * ulp * (np.abs(W_ref) + wb) + 1e-7
    bad = np.abs(W - W_ref) > bound
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} sampled elements beyond the double-rounding bound"


# ------------------------------------------------------------------------------------------------ vector length 16
# The reference's quant_gemv dispatches group size 16 with 16 index bits and 8 (or no) residual bits.  Its outputs on
# these cases are in tests/golden/ref_cuda/v16.npz (oracle/make_ref_cuda_golden.py --v16); outputs.npz is unchanged.
REF16_GOLDEN = os.path.join(GOLDEN_DIR, "ref_cuda", "v16.npz")
V16_CASES = {
    "v16_k65536_r256": dict(in_features=4096, out_features=1024, vector_len=16, num_centroids=65536,
                            num_res_centroids=256),
    "v16_k65536_r256_bf16": dict(in_features=4096, out_features=1024, vector_len=16, num_centroids=65536,
                                 num_res_centroids=256, dtype="bf16"),
    "v16_k65536_r0": dict(in_features=2048, out_features=1024, vector_len=16, num_centroids=65536),
}
V16_DEQUANT_CASES = ["v16_k65536_r256", "v16_k65536_r256_bf16"]


@pytest.fixture(scope="module")
def ref16():
    return np.load(REF16_GOLDEN, allow_pickle=False)


@pytest.mark.parametrize("route", ["default", "lists16"])
@pytest.mark.parametrize("name", sorted(V16_CASES))
def test_v16_gemv_matches_reference_cuda(ref16, name, route):
    """the default v = 16 route (the generic GEMV) and the v = 16 list kernel (set_list_decode) at 1 and 2 tokens
    against the record, with the bars of test_gemv_matches_reference_cuda"""
    import torch
    from _gpu import from_t, make_module, x_to_t
    from _probe import launched_kernels, ran
    L = vo.make_layer(seed=GEMV_SEED, **V16_CASES[name])
    m = make_module(L)
    if route == "lists16":
        m.set_list_decode(True)
    tol = 1e-3 if L.dtype == "fp16" else 8e-3
    for tokens in (1, 2):
        x_np = vo.make_x(tokens, L.in_features, L.dtype, seed=tokens)
        x = x_to_t(x_np, L)
        with torch.no_grad():
            m(x)
            names = launched_kernels(lambda: m(x))
            assert ran(names, "gemv_lists16_kernel") == (route == "lists16"), names
            y_ours = from_t(m(x))
        y_ref = from_bits(ref16[f"gemv__{name}__t{tokens}"], L.dtype)
        torch.cuda.synchronize()
        y_star = vo.quant_gemm(x_np, L)
        e_ours = parity_error(y_ours, y_star)
        assert e_ours <= tol
        if not np.isfinite(y_ref).all():
            print(f"{name} {route} tokens={tokens}: ours-vs-exact {e_ours:.2e}  reference kernel output is not finite, "
                  "skipped")
            continue
        assert y_ours.shape == y_ref.shape
        e_ref, e_mut = parity_error(y_ref, y_star), parity_error(y_ours, y_ref)
        print(f"{name} {route} tokens={tokens}: ours-vs-exact {e_ours:.2e}  ref-vs-exact {e_ref:.2e}  "
              f"ours-vs-ref {e_mut:.2e}")
        assert e_mut <= max(tol, 2 * e_ref), (e_mut, e_ref)


@pytest.mark.parametrize("name", V16_DEQUANT_CASES)
def test_v16_dequant_matches_reference_cuda(ref16, name):
    from _gpu import from_t, make_module
    L = vo.make_layer(seed=DEQUANT_SEED, **V16_CASES[name])
    m = make_module(L)
    W = from_t(m.dequant())
    assert W.shape == tuple(ref16[f"dequant__{name}__shape"])
    W = W.reshape(-1)[sample_positions(W.size)]
    W_ref = from_bits(ref16[f"dequant__{name}__values"], L.dtype)
    ulp = 2.0 ** -10 if L.dtype == "fp16" else 2.0 ** -7
    wb = np.abs(vo.to_f32(L.weight_bias, L.dtype)).max()
    bound = 2 * ulp * (np.abs(W_ref) + wb) + 1e-7
    bad = np.abs(W - W_ref) > bound
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} sampled elements beyond the double-rounding bound"
