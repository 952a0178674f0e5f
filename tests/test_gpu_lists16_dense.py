"""GPU checks of the dense weight from vector-length-16 index lists (csrc/lists_dense.cu at V = 16, include/
vptq_b200_lists_dense.h) and of decode-only v = 16 modules (set_list_decode + set_lists_prefill +
prepare(drop_packed=True)).

* the weight: W and Wt written from the v = 16 lists are bit-identical to the packed dequant (original order) and to
  the transposed dequant of the input-gradient GEMM, on every case of test_gpu_lists16.py in fp16 and bf16, on the
  Llama-3-70B shapes and Llama-3.1-405B q; one fp64 anchor per type;
* the module: bit-identical to a full module with set_list_decode at 1..max tokens (the same kernel); beyond, within
  TOL of fp64.  The full module's prefill pre-scales x at v = 16 and rounds differently, so there is no packed route
  to be bit-identical to: the comparison there with the GEMM from the lists on the full module's descriptor is a
  consistency check (the same kernels, decode-only against full descriptor), and the independent references are the
  fp64 bound and the weight's bit identity with the packed dequant (`_check_weight`).  dequant(), dX and dbias are
  bit-identical to the full module's; no kernel that reads packed words runs;
* values: NaN in unreferenced entry 0 of every slice and of the residual codebook stays out of W; inf / NaN in
  referenced entries land where the packed dequant puts them;
* a fused model, CUDA graphs, inference mode, in-place updates, reloading the checkpoint and the refusals.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

import _extreme as ex
import vptq_oracle as vo
from _batch import ZERO_HEAD, head_zero
from _lists16 import KERNEL, GpuLayer16, desc_of, repack
from _probe import launched_kernels, ran
from _util import TOL, parity_error
from test_gpu_lists16 import CASES

pytestmark = pytest.mark.gpu

DENSE = "lists_dense_kernel"
SENTINEL = 0x7A5A   # a finite 16-bit pattern in both types
FULL = {"70b_q_o": (8192, 8192), "70b_k_v": (8192, 1024), "70b_gate_up": (8192, 28672), "70b_down": (28672, 8192),
        "405b_q": (16384, 16384)}


def _bits(t):
    return t.contiguous().view(torch.int16)


def _dt(dtype):
    return torch.float16 if dtype == "fp16" else torch.bfloat16


def _packed_w(d, dt):
    from vptq_b200 import native
    w = torch.empty(d.out_features, d.in_features, dtype=dt, device="cuda")
    native.dequant(d, w)
    return w


def _packed_wt(d, dt):
    """Wt [in_features][ld] the transposed packed dequant wrote into the workspace of a 1-token input gradient
    (ld = out_features rounded up to 64, after the zero-at-rest head)"""
    from vptq_b200 import native
    I, O = d.in_features, d.out_features
    ld = (O + 63) // 64 * 64
    native.quant_gemm_dgrad(d, torch.zeros(1, O, dtype=dt, device="cuda"), torch.empty(1, I, dtype=dt, device="cuda"))
    ws = native.workspace(torch.device("cuda", torch.cuda.current_device()), 0)
    return ws[ZERO_HEAD:ZERO_HEAD + I * ld * 2].view(torch.int16).view(I, ld).clone(), ld


def _check_weight(d, dt):
    from vptq_b200 import native
    I, O = d.in_features, d.out_features
    w_ref = _packed_w(d, dt)
    # original order, ld > I, inside a sentinel-filled buffer: padding rows of the last index row never written
    ld = (I + 7) // 8 * 8 + 8
    buf = torch.full(((O + 1) * ld + 64,), SENTINEL, dtype=torch.int16, device="cuda")
    native.lists_dequant(d, buf.view(dt), ld)
    v = buf[:O * ld].view(O, ld)
    assert torch.equal(v[:, :I], _bits(w_ref))
    assert not v[:, I:].any()
    assert bool((buf[O * ld:] == SENTINEL).all())
    # transposed at the input-gradient GEMM's pitch: the packed route's Wt, zero columns included
    wt_ref, ldt = _packed_wt(d, dt)
    wt = torch.full((I, ldt), SENTINEL, dtype=torch.int16, device="cuda")
    native.lists_dequant(d, wt.view(dt), ldt, native.FLAG_TRANSPOSE)
    assert torch.equal(wt, wt_ref)
    # ld % 16 == 8: the second half of the last index row (and of the zero tail) lies past ld
    ldt = (O + 15) // 16 * 16 + 8
    buf = torch.full(((I + 1) * ldt + 64,), SENTINEL, dtype=torch.int16, device="cuda")
    native.lists_dequant(d, buf.view(dt), ldt, native.FLAG_TRANSPOSE)
    v = buf[:I * ldt].view(I, ldt)
    assert torch.equal(v[:, :O], _bits(w_ref.t()))
    assert not v[:, O:].any()
    assert bool((buf[I * ldt:] == SENTINEL).all())
    return w_ref


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_weight_from_v16_lists_is_bit_identical(name, dtype):
    L = vo.make_layer(vector_len=16, seed=61 + len(name), **dict(CASES[name], dtype=dtype))
    d = desc_of(L)
    w = _check_weight(d, _dt(dtype))
    names = launched_kernels(lambda: _check_weight(d, _dt(dtype)))
    assert ran(names, DENSE)
    head_zero()
    if name == "k65536_r256_fp16":   # one fp64 anchor per type
        W_star = vo.round_to(vo.dequant(L), dtype)
        tol = 2.0 ** -10 if dtype == "fp16" else 2.0 ** -7
        assert np.abs(w.float().cpu().numpy() - W_star).max() <= tol * np.abs(W_star).max() + 1e-7


@pytest.mark.parametrize("name", sorted(FULL) + ["70b_q_o_bf16"])
def test_full_size_weight_is_bit_identical(name):
    dtype = "bf16" if name.endswith("_bf16") else "fp16"
    I, O = FULL[name.replace("_bf16", "")]
    G = GpuLayer16(I, O, seed=700 + len(name), dtype=dtype)
    _check_weight(G.desc, _dt(dtype))
    del G
    torch.cuda.empty_cache()
    head_zero()


# ---------------------------------------------------------------- the module
MODULE = {"fp16": dict(in_features=4096, out_features=1048, num_centroids=65536, num_res_centroids=256, bias=True),
          "bf16": dict(in_features=2048, out_features=520, num_centroids=32768, num_res_centroids=64, bias=True,
                       dtype="bf16")}


def _packed_free(names):
    """no kernel that reads the packed index words ran"""
    assert not any("gemv_kernel" in n or "dequant" in n or "gemv_v2" in n for n in names), names


def _pair(L):
    from _gpu import make_module
    full = make_module(L).set_list_decode().prepare()
    dec = make_module(L).set_list_decode().set_lists_prefill()
    dec.prepare()
    packed = dec.indices.numel() * dec.indices.element_size()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    dec.prepare(drop_packed=True)
    torch.cuda.synchronize()
    assert before - torch.cuda.memory_allocated() >= packed
    assert dec.indices.numel() == 0 and not dec._desc_cache[0].indices and dec._desc_cache[0].lists_stream
    return full, dec


def _x(L, tokens, seed):
    from _gpu import x_to_t
    return x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)


def _ref(full, x):
    """what a decode-only copy of `full` must return: its own forward at 1..max tokens (the v = 16 list kernel), the
    GEMM from the lists on its descriptor beyond (the same kernels as the decode-only route: a consistency check,
    not an independent reference)"""
    from vptq_b200 import native
    d = full._desc_cache[0]
    if x.shape[0] <= native.lists16_max_tokens(d):
        return full(x)
    y = torch.empty(x.shape[0], full.out_features, dtype=x.dtype, device=x.device)
    native.lists_quant_gemm(d, x, y)
    return y


@pytest.mark.parametrize("kind", sorted(MODULE))
def test_decode_only_module_matches_the_full_module(kind):
    from _gpu import x_to_t
    from vptq_b200 import native
    L = vo.make_layer(vector_len=16, seed=17, **MODULE[kind])
    full, dec = _pair(L)
    mx = native.lists16_max_tokens(dec._desc_cache[0])
    assert mx >= 1
    with torch.no_grad():
        for tokens in list(range(1, mx + 1)) + [mx + 1, 9, 64, 2048]:
            x = _x(L, tokens, seed=tokens)
            names = launched_kernels(lambda: dec(x))
            _packed_free(names)
            assert ran(names, KERNEL) == (tokens <= mx) and ran(names, DENSE) == (tokens > mx), (tokens, names)
            y = dec(x)
            assert torch.equal(_bits(y), _bits(_ref(full, x))), tokens
            ystar = ex.y_star(L, x).cpu().numpy()
            assert parity_error(y.float().cpu().numpy(), ystar) <= TOL[L.dtype], tokens
        # a misaligned 1-token x: the list kernel on an aligned copy, the aligned result
        buf = _x(L, 2, seed=5).reshape(-1)
        x1 = buf[1:1 + L.in_features].view(1, -1)
        assert x1.data_ptr() % 16
        names = launched_kernels(lambda: dec(x1))
        _packed_free(names)
        assert ran(names, KERNEL)
        assert torch.equal(_bits(dec(x1)), _bits(dec(x1.clone())))
        assert torch.equal(_bits(dec.dequant()), _bits(full.dequant()))
        _packed_free(launched_kernels(lambda: dec.dequant()))
    # input and bias gradients: the same Wt and GEMM on both modules
    for tokens in (1, 5, 128, 2048):
        x = _x(L, tokens, seed=40 + tokens)
        dy = x_to_t(vo.make_x(tokens, L.out_features, L.dtype, seed=90 + tokens), L)
        xs = [x.clone().requires_grad_(), x.clone().requires_grad_()]
        for m, xx in zip((full, dec), xs):
            m.zero_grad()
            m(xx).backward(dy)
        assert torch.equal(_bits(xs[0].grad), _bits(xs[1].grad)), tokens
        assert torch.equal(_bits(full.bias.grad), _bits(dec.bias.grad)), tokens
        xx = x.clone().requires_grad_()
        _packed_free(launched_kernels(lambda: dec(xx).backward(dy)))
    head_zero()


def test_unreferenced_nan_stays_out_and_referenced_extremes_land_as_packed():
    L = vo.make_layer(vector_len=16, seed=23, in_features=2048, out_features=264, num_centroids=65536,
                      num_res_centroids=256)
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    idx = np.where(idx % 4096 == 0, idx + 1, idx)            # entry 0 of every slice: referenced by no field
    ridx = np.where(ridx == 0, 1, ridx)
    L = repack(L, idx, ridx)
    for s in range(L.num_centroids // 4096):
        for e in (0, 9, 15):
            L = ex.inject(L, "C", float("nan"), k=4096 * s, e=e)
    for e in (0, 8):
        L = ex.inject(L, "R", float("nan"), k=0, e=e)
    d = desc_of(L)
    w = _check_weight(d, torch.float16)
    assert bool(torch.isfinite(w).all())
    # referenced entries: inf / NaN where the packed dequant puts them
    k, kr = int(idx[0][3, 100]), int(ridx[0][5, 7])
    L = ex.inject(L, "C", float("inf"), k=k, e=2)
    L = ex.inject(L, "C", float("nan"), k=k, e=13)
    L = ex.inject(L, "R", float("-inf"), k=kr, e=10)
    w = _check_weight(desc_of(L), torch.float16)
    assert bool((~torch.isfinite(w)).any())
    head_zero()


# ---------------------------------------------------------------- model level and lifecycle
class _Block(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.attn, self.mlp = nn.Module(), nn.Module()
        self.attn.q_proj, self.attn.k_proj, self.attn.v_proj = layers[:3]
        self.mlp.gate_proj, self.mlp.up_proj = layers[3:]

    def forward(self, x):
        a = torch.cat([self.attn.q_proj(x), self.attn.k_proj(x), self.attn.v_proj(x)], -1)
        return torch.cat([a, self.mlp.gate_proj(x), self.mlp.up_proj(x)], -1)


def test_fused_decode_only_model():
    import vptq_b200
    from _gpu import make_module
    Ls = [vo.make_layer(in_features=2048, out_features=o, vector_len=16, num_centroids=65536, num_res_centroids=256,
                        seed=30 + i) for i, o in enumerate((2048, 512, 512, 4096, 4096))]
    members = [make_module(L).set_list_decode() for L in Ls]
    full = _Block(members)
    dec = _Block([make_module(L).set_list_decode().set_lists_prefill().prepare(drop_packed=True) for L in Ls])
    vptq_b200.fuse(full)
    vptq_b200.fuse(dec)
    with torch.no_grad():
        for tokens in (1, 2, 3, 4, 64):
            x = _x(Ls[0], tokens, seed=tokens)
            names = launched_kernels(lambda: dec(x))
            _packed_free(names)
            if tokens <= 4:   # one launch per group
                assert sum(ran([n], KERNEL) for n in names) == 2 and not ran(names, DENSE), names
            else:             # each member's own GEMM from its lists
                assert sum(ran([n], DENSE) for n in names) == 5 and not ran(names, KERNEL), names
            want = full(x) if tokens <= 4 else torch.cat([_ref(m, x) for m in members], -1)
            assert torch.equal(_bits(dec(x)), _bits(want)), tokens
    head_zero()


def test_lifecycle_and_refusals():
    from _gpu import make_module
    L = vo.make_layer(vector_len=16, seed=19, **MODULE["fp16"])
    sd = {k: v.clone() for k, v in make_module(L).state_dict().items()}
    full, dec = _pair(L)
    x1, xp = _x(L, 1, seed=1), _x(L, 64, seed=2)
    with torch.no_grad():
        y1, yp = _ref(full, x1), _ref(full, xp)
        # graphs at 1 token and at a prefill count, captured after eager calls that grew the workspace
        dec(_x(L, 2048, seed=3))
        g1, gp = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        s1, sp = x1.clone(), xp.clone()
        with torch.cuda.graph(g1):
            o1 = dec(s1)
        with torch.cuda.graph(gp):
            op = dec(sp)
        o1.zero_(), op.zero_()
        g1.replay(), gp.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(o1), _bits(y1)) and torch.equal(_bits(op), _bits(yp))
    with torch.inference_mode():
        assert torch.equal(_bits(dec(x1)), _bits(y1)) and torch.equal(_bits(dec(xp)), _bits(yp))
    # refusals: raise, and the module keeps working
    for bad in (lambda: dec.set_quant_grad(True), lambda: dec.prepare(rebuild=True), lambda: dec.state_dict(),
                lambda: dec.set_list_decode(False), lambda: dec.set_lists_prefill(False)):
        with pytest.raises(RuntimeError, match="decode-only"):
            bad()
    with torch.no_grad():
        assert torch.equal(_bits(dec(x1)), _bits(y1)) and torch.equal(_bits(dec(xp)), _bits(yp))
    # in-place codebook update, prepare(): outputs follow the new codebook
    with torch.no_grad():
        dec.centroids.weight.mul_(0.5)
        dec.res_centroids.weight.mul_(0.25)
    dec.prepare()
    fresh = make_module(L).set_list_decode()
    with torch.no_grad():
        fresh.centroids.weight.copy_(dec.centroids.weight)
        fresh.res_centroids.weight.copy_(dec.res_centroids.weight)
        fresh.prepare()
        assert torch.equal(_bits(dec(x1)), _bits(_ref(fresh, x1)))
        assert torch.equal(_bits(dec(xp)), _bits(_ref(fresh, xp)))
        assert torch.equal(_bits(dec.dequant()), _bits(fresh.dequant()))
    # reloading the checkpoint: a full module again, routed as a fresh one
    dec.load_state_dict(sd)
    with torch.no_grad():
        names = launched_kernels(lambda: dec(xp))
        assert not ran(names, DENSE) and dec.indices.numel() > 0 and dec._desc_cache[0].indices, names
        assert torch.equal(_bits(dec(x1)), _bits(y1)) and torch.equal(_bits(dec(xp)), _bits(full(xp)))
    assert dec.state_dict()["indices"].numel() > 0           # a full module saves again
    dec.set_list_decode(False).set_lists_prefill(False)      # allowed again on a full module
    head_zero()
