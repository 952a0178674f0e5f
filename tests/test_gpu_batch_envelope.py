"""The batched list kernel (csrc/gemv_lists_batch.cu) across its partition regimes, its workspace and shared-memory
cut-offs, its token masking and its output footprint.

The kernel runs B = floor(SMs / Q) CTAs per combo (Q = codebook slices x column tiles); these tests reach B = 1
(Q = 128), k = Ro (one index row per CTA), Ro = 1, a fused set with n = B, ragged last column tiles with several
tiles, NS = 2, 4, 8, 16, the full Llama-3 8B / 70B decode sets, the 65536-row workspace limit, the 3- / 2-stage ring
switch and the last shared-memory layout that fits.  Every shape used for a cut-off is also asserted on the CPU
against the integer mirror (tests/test_batch_decode_host.py).

Bars, per token t: |y - y*| <= TOL max|y*_t| + Q 2^-31 against the fp64 evaluation of the kernel's arithmetic,
twice that against the exact product.  Layers whose fp64 weight would be large are checked on a seeded sample of
index rows.  Every test asserts which kernels ran and that every workspace head is zero at rest afterwards."""
import gc

import pytest
import torch

from _batch import BATCH, GpuLayer, batch, head_zero, rand_x
from _probe import launched_kernels, ran

pytestmark = pytest.mark.gpu

SAMPLE = 40        # index rows checked per layer


@pytest.fixture(autouse=True)
def _own_workspaces():
    """the workspace-limit tests fill the whole zero-at-rest head: start and end without cached workspaces"""
    from vptq_b200 import native
    torch.cuda.synchronize()
    gc.collect()
    native.release_workspaces()
    yield
    torch.cuda.synchronize()
    gc.collect()
    native.release_workspaces()


def _one_batched_launch(descs, x, ys):
    batch(descs, x, ys)                           # (allocates the stream's workspace once)
    names = launched_kernels(lambda: batch(descs, x, ys))
    assert len(names) == 1 and ran(names, BATCH), names


def _run_set(layers, tokens_list=(2, 5, 8), seed=1, sample=SAMPLE):
    """one batched launch of the fused set per token count; every member on sampled rows against fp64; a token's
    outputs the same bits whatever the token count"""
    from vptq_b200 import native
    descs = [l.desc for l in layers]
    assert native.batch_max_tokens(descs) == 8
    x = rand_x(8, layers[0].I, layers[0].dtype, seed)
    y8 = None
    for tokens in sorted(tokens_list, reverse=True):
        ys = [torch.full((tokens, l.O), float("nan"), dtype=x.dtype, device="cuda") for l in layers]
        _one_batched_launch(descs, x[:tokens], ys)
        torch.cuda.synchronize()
        for k, (l, y) in enumerate(zip(layers, ys)):
            l.check(x[:tokens], y, l.sample(sample, seed=k + tokens))
            if y8 is not None:
                assert torch.equal(y, y8[k][:tokens]), (k, tokens)
        if y8 is None:
            y8 = ys
    head_zero()


# ------------------------------------------------------------------------------------------------------- A1 full size
FUSED_SETS = {
    "8b_qkv": (4096, [4096, 1024, 1024]), "8b_o": (4096, [4096]), "8b_gate_up": (4096, [14336, 14336]),
    "8b_down": (14336, [4096]), "70b_qkv": (8192, [8192, 1024, 1024]), "70b_o": (8192, [8192]),
    "70b_gate_up": (8192, [28672, 28672]), "70b_down": (28672, [8192]),
    "n_equals_b": (14336, [4096, 4096]),          # Q = 64, B = 2, k = [1, 1]
}
FULL = [(n, "fp16") for n in FUSED_SETS] + [("8b_qkv", "bf16"), ("70b_down", "bf16")]


@pytest.mark.parametrize("name,dtype", FULL, ids=[f"{n}-{d}" for n, d in FULL])
def test_full_size_fused_sets(name, dtype):
    I, outs = FUSED_SETS[name]
    layers = [GpuLayer(I, o, dtype=dtype, bias=k == 1, seed=10 * len(outs) + k) for k, o in enumerate(outs)]
    _run_set(layers, seed=len(name))


# ------------------------------------------------------------------------------------------------ A2 slices x tiles
SWEEP = [(ns, i, kr, pn) for ns in (2, 4, 8, 16) for i in (4096, 4100, 9004) for kr, pn in ((0, True), (2, False),
                                                                                          (256, True))]


@pytest.mark.parametrize("ns,I,kr,perm_norm", SWEEP, ids=[f"ns{a}-i{b}-kr{c}-{'pn' if d else 'plain'}"
                                                          for a, b, c, d in SWEEP])
def test_slices_and_ragged_tiles(ns, I, kr, perm_norm):
    """K = 4096 NS; I = 4100 gives TCW = 2056 with a last tile of 2044 columns, I = 9004 three tiles of 3008 / 3008 /
    2988 (and a row length that is not a multiple of 8)"""
    l = GpuLayer(I, 520, K=4096 * ns, Kr=kr, perm=perm_norm, norm=perm_norm, bias=not perm_norm, seed=ns + I + kr)
    _run_set([l], tokens_list=(3, 8), seed=ns)


# ----------------------------------------------------------------------------------------------- A3 partition extremes
@pytest.mark.parametrize("case", ["ro1", "k_equals_ro", "b1_q128"])
def test_partition_extremes(case):
    I, O, K = {"ro1": (1024, 8, 65536), "k_equals_ro": (1024, 264, 8192), "b1_q128": (32768, 4096, 65536)}[case]
    l = GpuLayer(I, O, K=K, bias=True, seed=len(case))
    _run_set([l], tokens_list=(1, 2, 7, 8), seed=3)


def test_q_equal_to_the_sm_count_is_not_reachable():
    """power-of-two codebooks give NS in {2, 4, 8, 16} and in_features <= 65535 gives NT <= 16: NS NT equals the SM
    count only where the SM count factorises so (not on a 132-SM H100, whose largest reachable Q, 128, runs above)"""
    from vptq_b200 import lists
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    shapes = [(ns, nt) for ns in (2, 4, 8, 16) for nt in range(1, 17) if ns * nt == sms]
    if not shapes:
        pytest.skip(f"{sms} SMs: no NS x NT of a valid layer equals it")
    ns, nt = shapes[0]
    I = 4096 * nt
    assert lists.geometry(I, 4096 * ns)[:2] == (ns, nt)
    _run_set([GpuLayer(I, 1024, K=4096 * ns, seed=5)], tokens_list=(2, 8))


# ------------------------------------------------------------------------------------------------ A4 workspace limit
def test_workspace_limit_accepted():
    """sum Ro x 8 = 65536: the [row][NTOK][8] accumulators fill the whole zero-at-rest head"""
    _run_set([GpuLayer(4096, 65536, seed=1)], tokens_list=(2, 8), sample=24)
    _run_set([GpuLayer(4096, 16384, seed=2 + k, bias=k == 3) for k in range(4)], tokens_list=(5, 8), sample=16)


def _module_of(l):
    from vptq_b200 import VQuantLinear
    t = l.t
    m = VQuantLinear(l.I, l.O, vector_lens=[-1, 8], num_centroids=[-1, l.K], num_res_centroids=[-1, l.Kr],
                     group_num=1, group_size=l.I, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                     enable_norm=t["weight_scale"] is not None, enable_perm=t["perm"] is not None,
                     bias=t["bias"] is not None, device="cuda", dtype=t["centroids"].dtype, enable_proxy_error=False)
    with torch.no_grad():
        m.indices.data = t["indices"]
        m.centroids.weight.data = t["centroids"]
        m.res_centroids.weight.data = t["res_centroids"]
        if t["perm"] is not None:
            m.perm.data = t["perm"]
        if t["weight_scale"] is not None:
            m.weight_scale.data, m.weight_bias.data = t["weight_scale"], t["weight_bias"]
        if t["bias"] is not None:
            m.bias.data = t["bias"]
    return m.eval()


def _module_fallback(l, refused_by):
    """batched decode refused for this layer: 2 tokens take the generic GEMV, 3..8 the prefill GEMM, right values"""
    from vptq_b200 import native
    assert native.batch_max_tokens(l.desc) == 0
    with pytest.raises(RuntimeError, match=refused_by):
        batch(l.desc, rand_x(2, l.I, l.dtype, 0))
    m = _module_of(l).set_batched_decode(True)
    x = rand_x(8, l.I, l.dtype, 4)
    with torch.no_grad():
        for tokens in (2, 3, 8):
            names = launched_kernels(lambda: m(x[:tokens]))
            assert not ran(names, BATCH), names
            if tokens == 2:
                assert ran(names, "gemv_kernel") and not ran(names, "gemm_tn_wgmma"), names
            else:
                assert ran(names, "gemm_tn_wgmma"), names
            l.check(x[:tokens], m(x[:tokens]), l.sample(24, seed=tokens), factor_exact=True)
    head_zero()


def test_workspace_limit_refused_falls_back():
    """out = 65544: one index row past the head"""
    _module_fallback(GpuLayer(4096, 65544, seed=3), "index rows")


# ------------------------------------------------------------------------------------------ A5 shared-memory cut-offs
def test_two_and_three_stage_rings_agree():
    """I = 12288 with two 20480-output layers: NTOK = 8 runs 2 ring stages, NTOK = 2 and 4 run 3 (mirror: carve()).
    The ring depth changes no arithmetic: a token's outputs are the same bits at every token count and position."""
    layers = [GpuLayer(12288, 20480, seed=40 + k, bias=k == 0) for k in range(2)]
    descs = [l.desc for l in layers]
    _run_set(layers, tokens_list=(2, 4, 8), seed=6, sample=24)
    x = rand_x(8, 12288, "fp16", 7)
    ref = batch(descs, x)
    for tokens in (1, 2, 3, 4, 5, 8):
        for start in (0, 8 - tokens):
            ys = batch(descs, x[start:start + tokens])
            for y, r in zip(ys, ref):
                assert torch.equal(y, r[start:start + tokens]), (tokens, start)
    head_zero()


def test_last_layout_that_fits():
    """I = 20480 (Q = 80), Kr = 256: out = 51192 needs exactly the 232448-byte opt-in at NTOK = 8"""
    _run_set([GpuLayer(20480, 51192, seed=8)], tokens_list=(2, 8), sample=24)


def test_no_layout_fits_falls_back():
    """out = 51200: 128 bytes more than the opt-in"""
    _module_fallback(GpuLayer(20480, 51200, seed=9), "shared-memory")


# ---------------------------------------------------------------------------------------------- A6 fused refusal
def test_fused_group_past_the_sm_count():
    """three layers at I = 12288 (Q = 48, B = 2): the group is refused; 2 tokens take the generic GEMV (one launch
    per member here: the fused generic launch cannot plan these shapes together), 3..8 tokens each member's own
    batched launch"""
    import vptq_b200
    from vptq_b200 import native
    layers = [GpuLayer(12288, o, seed=50 + k) for k, o in enumerate((4096, 1024, 1024))]
    assert native.batch_max_tokens([l.desc for l in layers]) == 0
    assert all(native.batch_max_tokens(l.desc) == 8 for l in layers)

    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj, self.v_proj = (_module_of(l) for l in layers)

        def forward(self, x):
            return self.q_proj(x), self.k_proj(x), self.v_proj(x)

    model = Attn()
    assert len(vptq_b200.fuse(model)) == 1
    assert vptq_b200.set_batched_decode(model) == 3
    x = rand_x(8, 12288, "fp16", 10)
    with torch.no_grad():
        for tokens in (2, 3, 8):
            model(x[:tokens])
            names = launched_kernels(lambda: model(x[:tokens]))
            if tokens == 2:
                assert all(ran([n], "gemv_kernel") or ran([n], "gemv_multi_kernel") for n in names), names
                assert len(names) in (1, 3), names
            else:
                assert len(names) == 3 and all(ran([n], BATCH) for n in names), names
            for l, y in zip(layers, model(x[:tokens])):
                l.check(x[:tokens], y, l.sample(24, seed=tokens))
    head_zero()


# ------------------------------------------------------------------------------------------------- B. masking
@pytest.fixture(scope="module")
def small():
    return [GpuLayer(1004, o, seed=60 + k, bias=k == 1) for k, o in enumerate((264, 100, 136))]


@pytest.mark.parametrize("tokens", [1, 3, 5, 7])
def test_rows_past_the_token_count_are_never_read(small, tokens):
    """x = the first t rows of an 8-row buffer whose other rows hold NaN, +inf and -inf: the same bits as clean"""
    l = small[0]
    x = rand_x(8, l.I, l.dtype, 11)
    clean = batch(l.desc, x[:tokens].clone())
    poisoned = x.clone()
    fill = (float("nan"), float("inf"), float("-inf"))
    for r in range(tokens, 8):
        poisoned[r] = fill[r % 3]
    y = torch.full((tokens, l.O), float("nan"), dtype=x.dtype, device="cuda")
    _one_batched_launch(l.desc, poisoned[:tokens], [y])
    assert torch.equal(y, clean)
    l.check(x[:tokens], y, l.sample(SAMPLE))
    head_zero()


@pytest.mark.parametrize("pitch", ["aligned", "odd"])
@pytest.mark.parametrize("fused", [False, True], ids=["one", "fused"])
def test_outputs_stay_inside_their_views(small, pitch, fused):
    """y views into a sentinel-filled buffer (gaps between the fused slices): rows >= t, columns past each slice and
    the gaps keep the sentinel"""
    layers = small if fused else small[:1]
    descs = [l.desc for l in layers]
    x = rand_x(8, 1004, "fp16", 12)
    sentinel = 1234.0
    gap = 5
    width = sum(l.O for l in layers) + gap * len(layers)
    pitch_el = (width + 7) // 8 * 8 if pitch == "aligned" else width + 3
    for tokens in (2, 5, 8):
        ref = batch(descs, x[:tokens]) if fused else [batch(descs[0], x[:tokens])]
        buf = torch.full((8 * pitch_el,), sentinel, dtype=torch.float16, device="cuda")
        grid = buf.view(8, pitch_el)
        views, mask, a = [], torch.zeros_like(grid, dtype=torch.bool), 0
        for l in layers:
            views.append(grid[:tokens, a:a + l.O])
            mask[:tokens, a:a + l.O] = True
            a += l.O + gap
        _one_batched_launch(descs, x[:tokens], views)
        torch.cuda.synchronize()
        assert bool((grid[~mask] == sentinel).all()), (tokens, int((grid[~mask] != sentinel).sum()))
        for v, r in zip(views, ref):
            assert torch.equal(v, r)
    head_zero()


def test_misaligned_weight_scale_is_refused_without_a_launch(small):
    from vptq_b200 import native
    l = small[0]
    base = l.desc
    d = native.LinearDesc()
    for f, _ in native.LinearDesc._fields_:
        setattr(d, f, getattr(base, f))
    d.weight_scale = base.weight_scale + 2
    assert native.batch_max_tokens(d) == 0
    x = rand_x(2, l.I, l.dtype, 13)
    batch(base, x)                                # (allocates the stream's workspace)
    y = torch.zeros(2, l.O, dtype=x.dtype, device="cuda")
    assert launched_kernels(lambda: pytest.raises(RuntimeError, batch, d, x, [y])) == []
    assert bool((y == 0).all())


def test_misaligned_x_takes_the_default_route(small):
    l = small[0]
    m = _module_of(l).set_batched_decode(True)
    x = rand_x(4, l.I, l.dtype, 14)
    buf = torch.zeros(4 * l.I + 8, dtype=x.dtype, device="cuda")
    xm = buf[1:1 + 4 * l.I].view(4, l.I)
    xm.copy_(x)
    with torch.no_grad():
        for tokens in (2, 4):
            xt = xm[:tokens]
            names = launched_kernels(lambda: m(xt))
            assert not ran(names, BATCH), names
            l.check(x[:tokens], m(xt), l.sample(SAMPLE))
