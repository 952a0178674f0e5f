"""GPU parity of the list-based decode kernel (csrc/gemv_lists.cu) through the C ABI.

Each case is run twice on the same tensors -- descriptor with the slice x tile lists (shared-memory
gathers) and without (generic kernel, L1/L2 gathers) -- and both are held to the oracle bar
(max|y - y*| / max|y*| <= 1e-3 fp16, 4e-3 bf16).  The list kernel rounds x * scale to the layer's 16-bit type and,
for fp16 layers, c + r to fp16, exactly as the reference's kernel does (csrc/kernels/quant_gemv.cuh:56,124-127), and
accumulates in fp32, then in 2^-30 fixed point across units (an absolute floor of Q * 2^-31 per output); the
generic kernel keeps those in fp32, so the two agree to a few output ulps, far inside the bar.  Non-finite and
out-of-range values: tests/test_gpu_extremes.py."""
import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _util import TOL, parity_error

pytestmark = pytest.mark.gpu


def _desc(L, lists):
    from _gpu import tdtype, to_t
    from vptq_b200 import native
    t = dict(indices=to_t(L.indices, L, "i32"), centroids=to_t(L.centroids, L),
             res_centroids=to_t(L.res_centroids, L) if L.res_bits else None,
             perm=to_t(L.perm, L, "u16") if L.perm is not None else None,
             weight_scale=to_t(L.weight_scale, L), weight_bias=to_t(L.weight_bias, L), bias=to_t(L.bias, L))
    d = native.make_desc(dtype=tdtype(L), in_features=L.in_features, out_features=L.out_features, vector_len=8,
                         num_centroids=L.num_centroids, num_res_centroids=L.num_res_centroids, num_codebooks=1,
                         group_size=L.group_size, outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1,
                         outlier_indices=None, outlier_centroids=None, lists=lists, **t)
    d._tensors = t
    assert bool(d.lists_stream) == lists
    return d


def _run(d, x, tokens=1):
    from vptq_b200 import native
    y = torch.full((tokens, d.out_features), float("nan"), dtype=x.dtype, device=x.device)
    native.quant_gemv(d, x[:tokens], y)
    torch.cuda.synchronize()
    return y


CASES = {
    "k65536_r256": dict(in_features=2048, out_features=1024, num_centroids=65536, num_res_centroids=256),
    "k65536_r256_bf16": dict(in_features=2048, out_features=1024, num_centroids=65536, num_res_centroids=256, dtype="bf16"),
    "k65536_r0_bias": dict(in_features=1024, out_features=2048, num_centroids=65536, bias=True),
    "k65536_r16_ragged": dict(in_features=1000, out_features=1004, num_centroids=65536, num_res_centroids=16),
    "k65536_i1004": dict(in_features=1004, out_features=512, num_centroids=65536, num_res_centroids=256),
    "k16384_r256": dict(in_features=1536, out_features=512, num_centroids=16384, num_res_centroids=256),
    "k8192_r256": dict(in_features=1536, out_features=512, num_centroids=8192, num_res_centroids=256),
    "k32768_plain": dict(in_features=1024, out_features=256, num_centroids=32768, enable_perm=False, enable_norm=False),
    "k32768_noperm_bf16": dict(in_features=1024, out_features=264, num_centroids=32768, num_res_centroids=64,
                               enable_perm=False, dtype="bf16", bias=True),
    "k65536_tiny_rows": dict(in_features=4096, out_features=24, num_centroids=65536, num_res_centroids=256),
    "k65536_one_row": dict(in_features=4096, out_features=8, num_centroids=65536, num_res_centroids=256),
    "k65536_wide": dict(in_features=14336, out_features=256, num_centroids=65536, num_res_centroids=256),
    "k65536_wide_odd": dict(in_features=9000, out_features=72, num_centroids=65536, num_res_centroids=256),
    "k65536_many_rows": dict(in_features=512, out_features=16384, num_centroids=65536, num_res_centroids=256),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_lists_vs_oracle_and_generic(name):
    from _gpu import from_t, x_to_t
    L = vo.make_layer(vector_len=8, seed=41, **CASES[name])
    x_np = vo.make_x(2, L.in_features, L.dtype, seed=7)
    x = x_to_t(x_np, L)
    y_star = vo.quant_gemm(x_np[:1], L)
    yl = from_t(_run(_desc(L, True), x))
    yg = from_t(_run(_desc(L, False), x))
    assert np.isfinite(yl).all()
    assert parity_error(yl, y_star) <= TOL[L.dtype], name
    assert parity_error(yg, y_star) <= TOL[L.dtype], name
    assert parity_error(yl, yg) <= (2.0 ** -9 if L.dtype == "fp16" else 2.0 ** -7), name


def test_lists_repeat_calls_leave_the_workspace_clean():
    """The arrival counters must be back at zero after every launch: 20 back-to-back calls on one workspace,
    interleaved with a generic-kernel layer that uses the same counter region."""
    from _gpu import from_t, x_to_t
    La = vo.make_layer(vector_len=8, seed=43, **CASES["k65536_r256"])
    Lb = vo.make_layer(vector_len=8, seed=44, in_features=2048, out_features=520, num_centroids=256)
    x_np = vo.make_x(1, 2048, "fp16", seed=3)
    x = x_to_t(x_np, La)
    da, db = _desc(La, True), _desc(Lb, False)
    ya0, yb0 = _run(da, x), _run(db, x)
    assert parity_error(from_t(ya0), vo.quant_gemm(x_np, La)) <= TOL["fp16"]
    for _ in range(10):
        assert torch.equal(_run(da, x), ya0)
        assert torch.equal(_run(db, x), yb0)


def test_two_tokens_take_the_generic_kernel():
    from _gpu import from_t, x_to_t
    L = vo.make_layer(vector_len=8, seed=42, **CASES["k65536_r256"])
    x_np = vo.make_x(2, L.in_features, L.dtype, seed=8)
    y = from_t(_run(_desc(L, True), x_to_t(x_np, L), tokens=2))
    assert parity_error(y, vo.quant_gemm(x_np, L)) <= TOL[L.dtype]


def test_lists_fused_launch_graph_and_repeatability():
    """q/k/v-style fused launch of list layers, under CUDA-graph replay with PDL; bit-identical from run to
    run (fixed summation order)."""
    from _gpu import from_t, x_to_t
    from vptq_b200 import native
    shapes = [(2048, 2048), (2048, 512), (2048, 520)]
    Ls = [vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                        seed=50 + k) for k, (i, o) in enumerate(shapes)]
    ds = [_desc(L, True) for L in Ls]
    x_np = vo.make_x(1, 2048, "fp16", seed=9)
    x = x_to_t(x_np, Ls[0])
    ys = [torch.full((1, L.out_features), float("nan"), dtype=x.dtype, device=x.device) for L in Ls]
    fused = native.FusedGemv(ds, ys)
    fused(x)
    torch.cuda.synchronize()
    assert not fused.separate
    first = [y.clone() for y in ys]
    for L, y, d in zip(Ls, ys, ds):
        assert parity_error(from_t(y), vo.quant_gemm(x_np, L)) <= TOL[L.dtype]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(3):
                fused(x, native.FLAG_PDL)
    for _ in range(10):
        for y in ys:
            y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        for y, f in zip(ys, first):
            assert torch.equal(y, f)


def test_chained_pdl_launches_read_fresh_activations():
    """y1 = L1(x), y2 = L2(y1) back to back with PDL inside a graph: the second launch must not read y1
    before the first has written it (griddepcontrol.wait) -- checked against eager, synchronised calls."""
    from _gpu import x_to_t
    from vptq_b200 import native
    L1 = vo.make_layer(in_features=2048, out_features=2048, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=60)
    L2 = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=61)
    d1, d2 = _desc(L1, True), _desc(L2, True)
    x = x_to_t(vo.make_x(1, 2048, "fp16", seed=10), L1)
    y1 = _run(d1, x)
    y2 = _run(d2, y1)
    a = torch.zeros_like(y1)
    b = torch.zeros_like(y2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        native.quant_gemv(d1, x, a, flags=native.FLAG_PDL)   # warm-up outside capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(4):
                native.quant_gemv(d1, x, a, flags=native.FLAG_PDL)
                native.quant_gemv(d2, a, b, flags=native.FLAG_PDL)
    for _ in range(5):
        a.zero_(); b.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(a, y1) and torch.equal(b, y2)


@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336), (14336, 4096), (8192, 1024), (28672, 1024)])
def test_lists_full_llama_shapes_match_generic(shape):
    """BASELINE configs[1] layer shapes at full size (and the 70B in_features): list kernel vs generic."""
    from _gpu import x_to_t
    i, o = shape
    L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=31)
    x = x_to_t(vo.make_x(1, i, "fp16", seed=5), L)
    yl, yg = _run(_desc(L, True), x).float(), _run(_desc(L, False), x).float()
    assert torch.isfinite(yl).all()
    assert float((yl - yg).abs().max()) <= 2.0 ** -9 * float(yg.abs().max())


def test_decode_only_module_drops_the_packed_words():
    """VQuantLinear.prepare(drop_packed=True): the lists replace the packed words (one copy of the indices); one-token
    calls are unchanged, multi-token calls and dequant refuse loudly, reloading the checkpoint restores everything."""
    from _gpu import from_t, make_module, x_to_t
    L = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=77)
    m = make_module(L)
    x_np = vo.make_x(3, 2048, "fp16", seed=1)
    x = x_to_t(x_np, L)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    y1 = m(x[:1]).clone()
    m.prepare(drop_packed=True)
    assert m.indices.numel() == 0 and not m._desc_cache[0].indices
    assert torch.equal(m(x[:1]), y1)
    assert parity_error(from_t(y1), vo.quant_gemm(x_np[:1], L)) <= TOL["fp16"]
    for bad in (x[:2], x):
        with pytest.raises(RuntimeError, match="decode-only"):
            m(bad)
    with pytest.raises(RuntimeError):
        m.dequant()
    m.load_state_dict(sd)
    assert parity_error(from_t(m(x)), vo.quant_gemm(x_np, L)) <= TOL["fp16"]
    assert torch.equal(m(x[:1]), y1)
