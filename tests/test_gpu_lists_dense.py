"""GPU checks of prefill, dequant and input gradient from the index lists (csrc/lists_dense.cu, include/
vptq_b200_lists_dense.h) and of the decode-only module routes that use them (VQuantLinear.set_lists_prefill).

* the weight: W and Wt written from the lists are bit-identical to the packed dequant kernels' on every list case of
  tests/test_gpu_lists.py and the Llama-3-8B shapes, fp16 and bf16; padding columns are zero, nothing outside the
  view is touched;
* the module: a decode-only copy with the opt-in against the full module -- bit-identical where the full module takes
  the prep-free prefill GEMM, within TOL of fp64 elsewhere; dequant(), dX and dbias bit-identical; batched decode
  still takes 2..8 tokens;
* extreme values: inf / NaN as the prefill route meets them; NaN in entry 0 of every slice and of the residual codebook
  reaches only the outputs whose fields use them (the padding entries of the lists are masked);
* lifecycle: CUDA graphs, inference mode, in-place updates, reloading the checkpoint, the zero-at-rest workspace head;
* model level: a fused decode-only model prefills and runs 2-token calls.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

import _extreme as ex
import vptq_oracle as vo
from _batch import BATCH, desc_of, head_zero
from _probe import launched_kernels, ran
from _util import TOL, parity_error
from test_gpu_lists import CASES

pytestmark = pytest.mark.gpu

LISTS_KERNEL = "lists_dense_kernel"
LLAMA = {"llama_4096x4096": dict(in_features=4096, out_features=4096, num_centroids=65536, num_res_centroids=256),
         "llama_14336x4096": dict(in_features=14336, out_features=4096, num_centroids=65536, num_res_centroids=256),
         "llama_4096x14336": dict(in_features=4096, out_features=14336, num_centroids=65536, num_res_centroids=256)}
SHAPES = dict(CASES, **LLAMA)
SENTINEL = 0x7A5A   # a finite 16-bit pattern in both types


def _bits(t):
    return t.contiguous().view(torch.int16)


def _packed_w(d, dt):
    from vptq_b200 import native
    w = torch.empty(d.out_features, d.in_features, dtype=dt, device="cuda")
    native.dequant(d, w)
    return w


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_weight_from_lists_is_bit_identical(name, dtype):
    from vptq_b200 import native
    L = vo.make_layer(vector_len=8, seed=41, **dict(SHAPES[name], dtype=dtype))
    dt = torch.float16 if dtype == "fp16" else torch.bfloat16
    d = desc_of(L)
    I, O = L.in_features, L.out_features
    w_ref = _packed_w(d, dt)
    # original order, ld > I, inside a sentinel-filled buffer with a row past O and a tail
    ld = (I + 7) // 8 * 8 + 16
    buf = torch.full(((O + 1) * ld + 64,), SENTINEL, dtype=torch.int16, device="cuda")
    native.lists_dequant(d, buf.view(dt), ld)
    v = buf[:O * ld].view(O, ld)
    assert torch.equal(v[:, :I], _bits(w_ref))
    assert not v[:, I:].any()
    assert bool((buf[O * ld:] == SENTINEL).all())
    # transposed, ld > O
    ldt = (O + 7) // 8 * 8 + 8
    buf = torch.full(((I + 1) * ldt + 64,), SENTINEL, dtype=torch.int16, device="cuda")
    native.lists_dequant(d, buf.view(dt), ldt, native.FLAG_TRANSPOSE)
    v = buf[:I * ldt].view(I, ldt)
    assert torch.equal(v[:, :O], _bits(w_ref.t()))
    assert not v[:, O:].any()
    assert bool((buf[I * ldt:] == SENTINEL).all())
    # Wt inside the input-gradient GEMM: dY = identity gives dX = W on both routes (by value: the fp32 accumulator
    # starts at +0, so a -0 weight comes out as +0)
    eye = torch.eye(O, dtype=dt, device="cuda")
    dx_l = torch.empty(O, I, dtype=dt, device="cuda")
    dx_p = torch.empty(O, I, dtype=dt, device="cuda")
    native.lists_quant_gemm(d, eye, dx_l, native.FLAG_TRANSPOSE)
    native.quant_gemm_dgrad(d, eye, dx_p)
    assert torch.equal(_bits(dx_l), _bits(dx_p)) and torch.equal(dx_l, w_ref)
    head_zero()


def _pair(L, batched=False):
    from _gpu import make_module
    full, dec = make_module(L), make_module(L)
    dec.prepare(drop_packed=True)
    dec.set_lists_prefill()
    if batched:
        full.set_batched_decode()
        dec.set_batched_decode()
    assert dec.indices.numel() == 0 and not dec._desc_cache[0].indices
    return full, dec


MODULE_LAYERS = {
    "direct": dict(in_features=1024, out_features=1004, num_centroids=65536, num_res_centroids=256, bias=True),
    "ragged_i": dict(in_features=1000, out_features=512, num_centroids=65536, num_res_centroids=16, bias=True),
}


@pytest.mark.parametrize("kind", sorted(MODULE_LAYERS))
def test_decode_only_module_prefills_like_the_full_module(kind):
    from _gpu import x_to_t
    L = vo.make_layer(vector_len=8, seed=5, **MODULE_LAYERS[kind])
    full, dec = _pair(L)
    W64 = torch.from_numpy(ex.dense64(L)).cuda()
    assert torch.equal(_bits(dec.dequant()), _bits(full.dequant()))
    for tokens in (2, 3, 9, 64, 300, 2048):
        x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=tokens), L)
        y_full, y_dec = full(x), dec(x)
        ystar = ex.y_star(L, x, W64).cpu().numpy()
        assert parity_error(y_dec.float().cpu().numpy(), ystar) <= TOL[L.dtype], tokens
        if kind == "direct" and tokens >= 3:   # the full module's prep-free prefill GEMM: the same W, the same GEMM
            assert torch.equal(_bits(y_dec), _bits(y_full)), tokens
        # input and bias gradients: the same Wt and GEMM on both modules, any token count
        xs = [x.clone().requires_grad_(), x.clone().requires_grad_()]
        dy = x_to_t(vo.make_x(tokens, L.out_features, L.dtype, seed=100 + tokens), L)
        for m, xx in zip((full, dec), xs):
            m.zero_grad()
            m(xx).backward(dy)
        assert torch.equal(_bits(xs[0].grad), _bits(xs[1].grad)), tokens
        assert torch.equal(_bits(full.bias.grad), _bits(dec.bias.grad)), tokens
        head_zero()
    assert dec.indices.numel() == 0 and not dec._desc_cache[0].indices


def test_gemm_prep_route_of_the_full_module_is_within_tol(monkeypatch):
    from _gpu import x_to_t
    monkeypatch.setenv("VPTQ_B200_GEMM_PREP", "1")
    L = vo.make_layer(vector_len=8, seed=6, **MODULE_LAYERS["direct"])
    full, dec = _pair(L)
    x = x_to_t(vo.make_x(64, L.in_features, L.dtype, seed=3), L)
    ystar = ex.y_star(L, x).cpu().numpy()
    for m in (full, dec):
        assert parity_error(m(x).float().cpu().numpy(), ystar) <= TOL[L.dtype]


def test_without_the_opt_in_a_decode_only_module_still_refuses():
    from _gpu import x_to_t
    L = vo.make_layer(vector_len=8, seed=7, **MODULE_LAYERS["direct"])
    _, dec = _pair(L)
    dec.set_lists_prefill(False)
    x = x_to_t(vo.make_x(9, L.in_features, L.dtype, seed=1), L)
    for bad in (x[:2], x):
        with pytest.raises(RuntimeError, match="decode-only"):
            dec(bad)
    with pytest.raises(RuntimeError):
        dec.dequant()


def test_batched_decode_keeps_2_to_8_tokens_and_the_lists_gemm_takes_the_rest():
    from _gpu import x_to_t
    L = vo.make_layer(vector_len=8, seed=8, in_features=2048, out_features=1024, num_centroids=65536,
                      num_res_centroids=256)
    full, dec = _pair(L, batched=True)
    for tokens in (2, 5, 8, 9, 64):
        x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=tokens), L)
        names = launched_kernels(lambda: dec(x))
        if tokens <= 8:
            assert ran(names, BATCH) and not ran(names, LISTS_KERNEL), names
            assert torch.equal(_bits(dec(x)), _bits(full(x))), tokens
        else:
            assert ran(names, LISTS_KERNEL) and ran(names, "gemm_tn_wgmma") and not ran(names, BATCH), names
            assert torch.equal(_bits(dec(x)), _bits(full(x))), tokens
    x1 = x_to_t(vo.make_x(1, L.in_features, L.dtype, seed=1), L)
    assert not ran(launched_kernels(lambda: dec(x1)), LISTS_KERNEL)
    assert torch.equal(_bits(dec(x1)), _bits(full(x1)))


@pytest.mark.parametrize("site", ["x", "C", "scale", "wbias", "bias"])
@pytest.mark.parametrize("value", sorted(ex.VALUES))
def test_extremes_as_the_prefill_route_meets_them(site, value):
    from _gpu import x_to_t
    L = vo.make_layer(vector_len=8, seed=9, **MODULE_LAYERS["direct"])
    x = x_to_t(vo.make_x(16, L.in_features, L.dtype, seed=2), L)
    if site == "x":
        x[3, 17] = ex.VALUES[value]
    else:
        L = ex.inject(L, site, ex.VALUES[value], k=int(vo.unpack_index(L.indices, L.index_bits, L.group_size,
                                                                         L.res_bits)[0][0][2, 5]), e=3, f=40, o=33)
    full, dec = _pair(L)
    y_full, y_dec = full(x), dec(x)
    assert torch.equal(_bits(y_dec), _bits(y_full))
    assert bool((ex.classify(y_dec) != ex.FINITE).any())
    assert torch.equal(_bits(dec.dequant()), _bits(full.dequant()))


def test_nan_in_entry_0_of_every_slice_reaches_only_its_rows():
    """Padding entries are zero words (entry 0 of slice 0, feature 0, residual 0): NaN there would spread if they were
    not masked.  Entry 0 of each slice and residual entry 0 are each used in one index row only."""
    from _gpu import x_to_t
    L = vo.make_layer(vector_len=8, seed=10, in_features=1024, out_features=512, num_centroids=65536,
                      num_res_centroids=256)
    ns = L.num_centroids // 4096
    L = ex.isolate(L, main={4096 * s: [2 * s + 1] for s in range(ns)}, res={0: [40]})
    for s in range(ns):
        L = ex.inject(L, "C", float("nan"), k=4096 * s, e=s % 8)
    L = ex.inject(L, "R", float("nan"), k=0, e=2)
    full, dec = _pair(L)
    x = x_to_t(vo.make_x(64, L.in_features, L.dtype, seed=4), L)
    want = ex.classify(ex.y_star(L, x))
    assert int((want == ex.NAN).sum()) == 64 * (ns + 1)
    assert torch.equal(ex.classify(dec(x)), want)
    w_cls = ex.classify(dec.dequant())
    assert torch.equal(w_cls, ex.classify(torch.from_numpy(ex.dense64(L)).cuda()))
    assert torch.equal(_bits(dec.dequant()), _bits(full.dequant()))


def test_cuda_graphs_inference_mode_and_in_place_updates():
    from _gpu import make_module, x_to_t
    L = vo.make_layer(vector_len=8, seed=11, **MODULE_LAYERS["direct"])
    full, dec = _pair(L)
    x = x_to_t(vo.make_x(300, L.in_features, L.dtype, seed=5), L)
    y_ref = full(x)
    with torch.no_grad():
        # capture on torch's capture stream, after eager calls that grow the workspace
        dec(x_to_t(vo.make_x(2048, L.in_features, L.dtype, seed=6), L))
        xs = x.clone()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ys = dec(xs)
        dec(x_to_t(vo.make_x(4096, L.in_features, L.dtype, seed=7), L))   # eager growth after the capture
        ys.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(ys), _bits(y_ref))
    head_zero()
    with torch.inference_mode():
        assert torch.equal(_bits(dec(x)), _bits(y_ref))
        assert torch.equal(_bits(dec.dequant()), _bits(full.dequant()))
    # in-place update of the codebooks: prepare(), then a fresh full module with the same tensors
    with torch.no_grad():
        dec.centroids.weight.mul_(0.5)
        dec.res_centroids.weight.mul_(0.25)
    dec.prepare()
    fresh = make_module(L)
    with torch.no_grad():
        fresh.centroids.weight.copy_(dec.centroids.weight)
        fresh.res_centroids.weight.copy_(dec.res_centroids.weight)
    assert torch.equal(_bits(dec(x)), _bits(fresh(x)))
    assert torch.equal(_bits(dec.dequant()), _bits(fresh.dequant()))
    head_zero()


def test_load_state_dict_brings_the_packed_routes_back():
    from _gpu import make_module, x_to_t
    L = vo.make_layer(vector_len=8, seed=12, **MODULE_LAYERS["direct"])
    sd = {k: v.clone() for k, v in make_module(L).state_dict().items()}
    full, dec = _pair(L)
    x = x_to_t(vo.make_x(64, L.in_features, L.dtype, seed=8), L)
    assert ran(launched_kernels(lambda: dec(x)), LISTS_KERNEL)
    dec.load_state_dict(sd)
    names = launched_kernels(lambda: dec(x))
    assert not ran(names, LISTS_KERNEL) and ran(names, "dequant_o8_kernel"), names
    assert dec.indices.numel() > 0 and dec._desc_cache[0].indices
    assert torch.equal(_bits(dec(x)), _bits(full(x)))
    assert not ran(launched_kernels(lambda: dec.dequant()), LISTS_KERNEL)


class _Block(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.attn, self.mlp = nn.Module(), nn.Module()
        self.attn.q_proj, self.attn.k_proj, self.attn.v_proj = layers[:3]
        self.mlp.gate_proj, self.mlp.up_proj = layers[3:]

    def forward(self, x):
        a = torch.cat([self.attn.q_proj(x), self.attn.k_proj(x), self.attn.v_proj(x)], -1)
        return torch.cat([a, self.mlp.gate_proj(x), self.mlp.up_proj(x)], -1)


def test_fused_decode_only_model_prefills_and_serves_two_tokens():
    import vptq_b200
    from _gpu import make_module, x_to_t
    Ls = [vo.make_layer(in_features=1024, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                        seed=20 + i) for i, o in enumerate((1024, 256, 256, 2048, 2048))]
    full = _Block([make_module(L) for L in Ls])
    dec = _Block([make_module(L).prepare(drop_packed=True) for L in Ls])
    vptq_b200.fuse(full)
    vptq_b200.fuse(dec)
    assert vptq_b200.set_lists_prefill(dec) == 5
    x = x_to_t(vo.make_x(300, 1024, "fp16", seed=9), Ls[0])
    with torch.no_grad():
        assert torch.equal(_bits(dec(x)), _bits(full(x)))
        x2 = x[:2].clone()
        y2 = dec(x2)
        # each member routed itself (the GEMM from the lists): the same values as the unfused decode-only layers
        vptq_b200.unfuse(dec)
        assert torch.equal(_bits(y2), _bits(dec(x2)))
    ystar = torch.cat([ex.y_star(L, x2) for L in Ls], -1).cpu().numpy()
    assert parity_error(y2.float().cpu().numpy(), ystar) <= TOL["fp16"]
    head_zero()
