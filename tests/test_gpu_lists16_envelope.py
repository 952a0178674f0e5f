"""The vector-length-16 list kernel (csrc/gemv_lists16.cu) across its partition regimes, its index-data extremes, its
shared-memory and row-token cut-offs, its token masking and its output footprint.

The kernel runs B = floor(SMs / Q) CTAs per combo (Q = codebook slices x column tiles); these tests reach NS = 2, 4, 8,
16 at one and at ragged multi-tile widths, Ro = 1 (O = 8: the whole hi plane is padding), B = 1 (Q = 128), one index
row per CTA with one slice per row (a unit split across all 16 warps' runs, and CTAs whose warps mostly get no steps),
all-ones index fields, every residual replication and ring depth the carve chooses, the exact shared-memory fit, the
4 -> 2 -> 1 -> 0 token limits and a fused group past the SM count.  Every shape used for a cut-off is also asserted
against the integer mirror on the CPU (tests/test_lists16_host.py; the shapes themselves are in tests/_lists16.py).

Bars, per token t: |y - y*| <= TOL max|y*_t| + Q 2^-31 against the fp64 evaluation of the kernel's arithmetic,
twice that against the exact product; one-hot probes exact to the bit.  Layers whose fp64 weight would be large are
checked on a seeded sample of index rows.  Every test asserts which kernels ran and that every workspace head is zero
at rest afterwards."""
import gc

import numpy as np
import pytest
import torch

import vptq_oracle as vo
from _batch import head_zero, kernel_star, q_of, rand_x, assert_close
from _lists16 import (CARVE, EXACT_FIT, KERNEL, PAST_FIT, QKV_405B, ROW_TOKENS, SM_COUNT, SMEM_OPTIN, GpuLayer16,
                      desc_of, module_of, only_kernel, repack, run)
from _probe import launched_kernels, probe_expect, ran

pytestmark = pytest.mark.gpu

SAMPLE = 40        # index rows checked per large layer


@pytest.fixture(autouse=True)
def _own_workspaces():
    """the row-token-limit tests fill the whole zero-at-rest head: start and end without cached workspaces"""
    from vptq_b200 import native
    torch.cuda.synchronize()
    gc.collect()
    native.release_workspaces()
    yield
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    native.release_workspaces()


@pytest.fixture()
def h100():
    """the cut-off shapes hold for a 132-SM device with the 232448-byte shared-memory opt-in"""
    p = torch.cuda.get_device_properties(0)
    optin = getattr(p, "shared_memory_per_block_optin", None)
    if optin != SMEM_OPTIN or p.multi_processor_count != SM_COUNT:
        pytest.skip(f"{p.multi_processor_count} SMs, opt-in {optin}: the cut-off shapes are for {SM_COUNT} / {SMEM_OPTIN}")


def _invariant_tokens(descs, x, check):
    """1..4 tokens: one v = 16 launch each, `check(tokens, ys)`, and each token's bits the same at every token count and
    position as in the 4-token launch"""
    single = not isinstance(descs, (list, tuple))
    descs = [descs] if single else list(descs)
    y4 = run(descs, x[:4])
    only_kernel(lambda: run(descs, x[:4], y4), launches=1)
    torch.cuda.synchronize()
    check(4, y4)
    for tokens in (1, 2, 3):
        for start in range(0, 5 - tokens):
            ys = run(descs, x[start:start + tokens].clone())
            for y, r in zip(ys, y4):
                assert torch.equal(y, r[start:start + tokens]), (tokens, start)
            if start == 0:
                check(tokens, ys)
    return y4


def _check_layers(layers, x, sample=SAMPLE):
    def check(tokens, ys):
        for k, (G, y) in enumerate(zip(layers, ys)):
            G.check(x[:tokens], y, rows=G.sample(sample, seed=k + tokens))
    return check


# ------------------------------------------------------------------------------------------------ partition
SWEEP = [(ns, i, kr, pn) for ns in (2, 4, 8, 16) for i in (4096, 4100, 9004) for kr, pn in ((0, True), (2, False),
                                                                                          (256, True))]


@pytest.mark.parametrize("ns,I,kr,perm_norm", SWEEP, ids=[f"ns{a}-i{b}-kr{c}-{'pn' if d else 'plain'}"
                                                          for a, b, c, d in SWEEP])
def test_slices_and_ragged_tiles(ns, I, kr, perm_norm):
    """K = 4096 NS; I = 4100 gives TCW = 2056 with a last tile of 2044 columns, I = 9004 three tiles of 3008 / 3008 /
    2988 (and a row length that is not a multiple of 8); out = 520: a last index row half padding"""
    from vptq_b200 import native
    G = GpuLayer16(I, 520, K=4096 * ns, Kr=kr, perm=perm_norm, norm=perm_norm, bias=not perm_norm, seed=ns + I + kr)
    assert native.lists16_max_tokens(G.desc) == 4
    x = rand_x(4, I, "fp16", seed=ns)
    _invariant_tokens(G.desc, x, _check_layers([G], x))
    head_zero()


@pytest.mark.parametrize("O", [8, 16])
def test_one_index_row(O):
    """Ro = 1: one CTA per combo; at O = 8 the outputs of the hi plane are all padding and must not be written"""
    G = GpuLayer16(1024, O, bias=True, seed=O)
    x = rand_x(4, 1024, "fp16", seed=O)
    buf = torch.full((4, 24), 1234.0, dtype=torch.float16, device="cuda")
    y4 = _invariant_tokens(G.desc, x, _check_layers([G], x))
    run(G.desc, x, [buf[:, :O]])
    assert torch.equal(buf[:, :O], y4[0]) and bool((buf[:, O:] == 1234.0).all())
    G.probe(range(0, 1024, 97), rows=[0])
    head_zero()


def test_q128_one_cta_per_combo(h100):
    """I = 32768, K = 65536: Q = 16 x 8 = 128 combos, B = 1"""
    assert q_of(32768, 65536) == 128
    G = GpuLayer16(32768, 4096, bias=True, seed=3)
    x = rand_x(4, 32768, "fp16", seed=3)
    _invariant_tokens(G.desc, x, _check_layers([G], x, sample=24))
    head_zero()


def test_one_slice_per_row_one_row_per_cta(h100):
    """I = 4096, K = 65536, out = 128: Q = 16, B = 8 = Ro, so every CTA holds one unit.  Row r draws its fields from
    slice (5 r) mod 16 only: that unit has 128 steps, split over all 16 warps' runs; every other unit of the row is
    one padding step, so 15 of its CTA's warps get no step at all"""
    L0 = vo.make_layer(in_features=4096, out_features=128, vector_len=16, num_centroids=65536, num_res_centroids=256,
                       seed=71, bias=True)
    idx = L0.meta["idx"].copy()
    sl = (5 * np.arange(8)) % 16
    idx[0] = sl[:, None] * 4096 + idx[0] % 4096
    L = repack(L0, idx=idx)
    d = desc_of(L)
    tab = d._keep[-1].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    first = tab & ((1 << 26) - 1)
    steps = (first[1:] - first[:-1]).reshape(16, 8)         # [combo = slice (one tile)][row]
    for r in range(8):
        assert steps[sl[r], r] == 128 and all(steps[s, r] <= 1 for s in range(16) if s != sl[r]), steps[:, r]
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 4096, "fp16", seed=8), "fp16")).cuda().half()

    def check(tokens, y):
        assert_close(y[0], kernel_star(L, x[:tokens]), "fp16", q_of(4096, 65536))
    _invariant_tokens(d, x, check)
    dt = torch.float16
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)
    for f in ((0, 4095), (1, 2, 3), (100, 2000, 3000, 4000)):
        xp = torch.zeros(len(f), 4096, dtype=dt, device="cuda")
        xp[torch.arange(len(f)), torch.tensor(f, device="cuda")] = 1.0
        assert torch.equal(run(d, xp).view(torch.int16), expect[list(f)].view(torch.int16)), f
    head_zero()


# ------------------------------------------------------------------------------------------------ all-ones fields
ONES = [(k, kr, dt) for k in (8192, 65536) for kr in (2, 256) for dt in ("fp16", "bf16")]


@pytest.mark.parametrize("K,Kr,dtype", ONES, ids=[f"k{a}-r{b}-{c}" for a, b, c in ONES])
def test_all_ones_fields(K, Kr, dtype):
    """idx = K - 1, ridx = Kr - 1 everywhere: the last entry of the last slice in both planes, the last residual copy,
    and (Kr = 256) entry words >= 2^31; every unit but the last slice's is empty.  Against the exact product only
    in fp16: with one weight per column the bf16 roundings of x' = x * scale (part of the kernel's arithmetic, held
    to the first bar) do not average out over the 4096 terms, and alone come to about 3 TOL max|y*|"""
    L0 = vo.make_layer(in_features=4096, out_features=264, vector_len=16, num_centroids=K, num_res_centroids=Kr,
                       seed=K + Kr, dtype=dtype, bias=True)
    shape = L0.meta["idx"].shape
    L = repack(L0, idx=np.full(shape, K - 1, dtype=np.int64), ridx=np.full(shape, Kr - 1, dtype=np.int64))
    d = desc_of(L)
    if Kr == 256:
        words = d._keep[-2].cpu().numpy().reshape(-1).view(np.uint32)
        assert (words >= 1 << 31).any()
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 4096, dtype, seed=9), dtype)).cuda()
    x = x.to(torch.float16 if dtype == "fp16" else torch.bfloat16)
    import _extreme as ex
    kstar, exact = kernel_star(L, x), ex.y_star(L, x)

    def check(tokens, y):
        assert_close(y[0], kstar[:tokens], dtype, q_of(4096, K))
        if dtype == "fp16":
            assert_close(y[0], exact[:tokens], dtype, q_of(4096, K), factor=2.0)
    _invariant_tokens(d, x, check)
    dt = x.dtype
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)
    rng = np.random.default_rng(K + Kr)
    for tokens in (1, 2, 3, 4):
        f = rng.choice(4096, size=tokens, replace=False)
        xp = torch.zeros(tokens, 4096, dtype=dt, device="cuda")
        xp[torch.arange(tokens), torch.from_numpy(f).cuda()] = 1.0
        assert torch.equal(run(d, xp).view(torch.int16), expect[torch.from_numpy(f).cuda()].view(torch.int16)), f
    G = GpuLayer16(4096, 2048, K=K, Kr=Kr, dtype=dtype, seed=K + Kr, all_ones=True)    # the same on the GPU builder
    xg = rand_x(4, 4096, dtype, seed=10)
    y = run(G.desc, xg)
    if dtype == "fp16":
        G.check(xg, y, rows=G.sample(16))
    else:
        Ls, cols, keep = G.oracle(G.sample(16))
        ys = y[:, torch.from_numpy(cols[keep]).cuda()]
        assert_close(ys, kernel_star(Ls, xg)[:, torch.from_numpy(np.nonzero(keep)[0]).cuda()], dtype, q_of(4096, K))
    G.probe((0, 4095, 1234, 77), rows=[0, G.Ro - 1])
    head_zero()


# ------------------------------------------------------------------------------------------------ shared-memory carve
@pytest.mark.parametrize("regime", sorted(CARVE), ids=[f"rep{r}-st{s}" for r, s in sorted(CARVE)])
def test_carve_regimes_probed_exactly(regime, h100):
    """one shape per (residual replication, ring stages) the carve chooses (the mirror's figures); one-hot probes on
    both planes exact, random x within the bars.  Replication 1 / 2 stages is the exact fit (I = 32768, out = 72176)"""
    from vptq_b200 import native
    I, O, Kr, tokens = CARVE[regime]
    big = I * O > 1 << 26
    G = GpuLayer16(I, O, Kr=Kr, bias=not big, seed=sum(regime) + Kr)
    assert native.lists16_max_tokens(G.desc) == 4
    rows = G.sample(8 if big else 64, seed=1)
    rng = np.random.default_rng(Kr + I)
    feats = [int(f) for f in rng.choice(I, size=4 * tokens, replace=False)] + [0, I - 1]
    L, cols, keep = G.oracle(rows)
    dt = G.t["centroids"].dtype
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)[:, torch.from_numpy(keep).cuda()]
    c = torch.from_numpy(cols[keep]).cuda()
    for a in range(0, len(feats), tokens):
        f = feats[a:a + tokens]
        xp = torch.zeros(len(f), I, dtype=dt, device="cuda")
        xp[torch.arange(len(f)), torch.tensor(f, device="cuda")] = 1.0
        y = run(G.desc, xp)
        if a == 0:
            only_kernel(lambda: run(G.desc, xp, [y]), launches=1)
        torch.cuda.synchronize()
        assert torch.equal(y[:, c].view(torch.int16), expect[torch.tensor(f, device="cuda")].view(torch.int16)), f
    x = rand_x(tokens, I, "fp16", seed=5)
    y = run(G.desc, x)
    G.check(x, y, rows=rows)
    if regime == (1, 2):
        assert (I, O) == EXACT_FIT
        assert torch.equal(run(G.desc, x[:1].clone()), y[:1])     # (the 1-token instance: replication 4)
    del G
    head_zero()


def test_one_row_past_the_exact_fit_takes_two_tokens(h100):
    """I = 32768, out = 72192: NTOK = 4 needs 128 bytes more than the opt-in, so the layer takes 1..2 tokens.  At
    module level 1 and 2 tokens run the v = 16 kernel, 3 and 4 the prefill GEMM, all within the bars"""
    from vptq_b200 import native
    G = GpuLayer16(*PAST_FIT, seed=12)
    assert native.lists16_max_tokens(G.desc) == 2
    x = rand_x(4, PAST_FIT[0], "fp16", seed=12)
    with pytest.raises(RuntimeError, match="1..2"):
        run(G.desc, x[:3])
    m = module_of(G).set_list_decode(True)
    rows = G.sample(16, seed=2)
    with torch.no_grad():
        for tokens in (1, 2, 3, 4):
            names = launched_kernels(lambda: m(x[:tokens]))
            if tokens <= 2:
                assert len(names) == 1 and ran(names, KERNEL), names
            else:
                assert not ran(names, KERNEL) and ran(names, "gemm_tn_wgmma"), names
            G.check(x[:tokens], m(x[:tokens]), rows=rows)
    del m, G
    head_zero()


# ------------------------------------------------------------------------------------------------ row-token limit
@pytest.mark.parametrize("O", sorted(ROW_TOKENS))
def test_row_token_limit(O, h100):
    """I = 4096: sum Ro x NTOK <= 32768 accumulators of 16 outputs.  out = 131072 takes 4 tokens, 262144 two, 524288
    one (its accumulators fill the 4 MiB head exactly), 524304 none.  The module routes the calls past the limit as
    before: 2 tokens to the generic GEMV, 3 and more to the prefill GEMM"""
    from vptq_b200 import native
    want = ROW_TOKENS[O]
    G = GpuLayer16(4096, O, seed=O % 1000)
    assert native.lists16_max_tokens(G.desc) == want
    x = rand_x(4, 4096, "fp16", seed=O % 997)
    rows = G.sample(16, seed=O % 13)
    if want:
        y = run(G.desc, x[:want])
        only_kernel(lambda: run(G.desc, x[:want], [y]), launches=1)
        G.check(x[:want], y, rows=rows)
        if want > 1:
            assert torch.equal(run(G.desc, x[:1].clone()), y[:1])
    else:
        with pytest.raises(RuntimeError, match="index rows"):
            run(G.desc, x[:1])
    m = module_of(G).set_list_decode(True)
    with torch.no_grad():
        for tokens in sorted({max(want, 1), want + 1} - {0}):
            if tokens > 4 or (O > 262144 and tokens > 2):
                continue                       # (the prefill GEMM would dequantise a 4 GiB weight)
            names = launched_kernels(lambda: m(x[:tokens]))
            if tokens <= want:
                assert len(names) == 1 and ran(names, KERNEL), names
            elif tokens < 3:
                assert ran(names, "gemv_kernel") and not ran(names, KERNEL), names
            else:
                assert ran(names, "gemm_tn_wgmma") and not ran(names, KERNEL), names
            G.check(x[:tokens], m(x[:tokens]), rows=rows)
    del m, G
    head_zero()


# ------------------------------------------------------------------------------------------------ fused refusal
def test_fused_405b_qkv_is_refused_and_each_member_runs_alone(h100):
    """Llama-3.1-405B q/k/v at I = 16384: Q = 64 leaves B = 2 combo copies for three layers, so the group is refused;
    with the opt-in each member runs its own v = 16 launch, with the right values"""
    import vptq_b200
    from vptq_b200 import native
    I, outs = QKV_405B
    layers = [GpuLayer16(I, o, seed=80 + k, bias=k == 1) for k, o in enumerate(outs)]
    assert native.lists16_max_tokens([G.desc for G in layers]) == 0
    assert all(native.lists16_max_tokens(G.desc) == 4 for G in layers)

    class Attn(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj, self.v_proj = (module_of(G) for G in layers)

        def forward(self, x):
            return self.q_proj(x), self.k_proj(x), self.v_proj(x)

    model = Attn()
    assert len(vptq_b200.fuse(model)) == 1
    assert vptq_b200.set_list_decode(model) == 3
    x = rand_x(4, I, "fp16", seed=11)
    with torch.no_grad():
        for tokens in (1, 3, 4):
            model(x[:tokens])
            names = launched_kernels(lambda: model(x[:tokens]))
            assert len(names) == 3 and all(ran([n], KERNEL) for n in names), names
            for k, (G, y) in enumerate(zip(layers, model(x[:tokens]))):
                assert torch.equal(y, run(G.desc, x[:tokens]))
                G.check(x[:tokens], y, rows=G.sample(16, seed=k))
    del model, layers
    head_zero()


# ------------------------------------------------------------------------------------------------ masking, footprint
@pytest.fixture(scope="module")
def small():
    return [vo.make_layer(in_features=4100, out_features=o, vector_len=16, num_centroids=65536, num_res_centroids=256,
                          seed=60 + k, bias=k == 1) for k, o in enumerate((264, 104, 136))]


@pytest.mark.parametrize("tokens", [1, 2, 3])
def test_rows_past_the_token_count_are_never_read(small, tokens):
    """x = the first t rows of a 4-row buffer whose other rows hold NaN, +inf and -inf: the same bits as clean (3
    tokens run the 4-token instance)"""
    L = small[0]
    d = desc_of(L)
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 4100, "fp16", seed=11), "fp16")).cuda().half()
    buf = torch.zeros(4, 4104, dtype=torch.float16, device="cuda")[:, :4100]    # (16-byte aligned rows)
    buf.copy_(x)
    clean = run(d, buf[:tokens].clone())
    fill = (float("nan"), float("inf"), float("-inf"))
    for r in range(tokens, 4):
        buf[r] = fill[r % 3]
    y = torch.full((tokens, L.out_features), float("nan"), dtype=x.dtype, device="cuda")
    only_kernel(lambda: run(d, buf[:tokens], [y]), launches=1)
    assert torch.equal(y, clean)
    assert_close(y, kernel_star(L, x[:tokens]), "fp16", q_of(4100, 65536))
    head_zero()


@pytest.mark.parametrize("pitch", ["aligned", "odd"])
@pytest.mark.parametrize("fused", [False, True], ids=["one", "fused"])
def test_outputs_stay_inside_their_views(small, pitch, fused):
    """y views into a sentinel-filled buffer (gaps between the fused slices): rows >= t, columns past each slice and
    the gaps keep the sentinel; an odd pitch sends rows to the kernel's unaligned store path"""
    layers = small if fused else small[:1]
    descs = [desc_of(L) for L in layers]
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 4100, "fp16", seed=12), "fp16")).cuda().half()
    x = x.clone()
    sentinel, gap = 1234.0, 5
    width = sum(L.out_features for L in layers) + gap * len(layers)
    pitch_el = (width + 7) // 8 * 8 if pitch == "aligned" else width + 3
    for tokens in (1, 2, 3, 4):
        ref = run(descs, x[:tokens].clone())
        buf = torch.full((4 * pitch_el,), sentinel, dtype=torch.float16, device="cuda")
        grid = buf.view(4, pitch_el)
        views, mask, a = [], torch.zeros_like(grid, dtype=torch.bool), 0
        for L in layers:
            views.append(grid[:tokens, a:a + L.out_features])
            mask[:tokens, a:a + L.out_features] = True
            a += L.out_features + gap
        xt = x[:tokens].clone()
        only_kernel(lambda: run(descs, xt, views), launches=1)
        torch.cuda.synchronize()
        assert bool((grid[~mask] == sentinel).all()), (tokens, int((grid[~mask] != sentinel).sum()))
        for v, r in zip(views, ref):
            assert torch.equal(v, r)
    head_zero()


def test_misaligned_weight_scale_is_refused_without_a_launch(small):
    from vptq_b200 import native
    L = small[0]
    base = desc_of(L)
    d = native.LinearDesc()
    for f, _ in native.LinearDesc._fields_:
        setattr(d, f, getattr(base, f))
    d.weight_scale = base.weight_scale + 2
    assert native.lists16_max_tokens(d) == 0
    x = torch.from_numpy(vo.to_f32(vo.make_x(2, 4100, "fp16", seed=13), "fp16")).cuda().half()
    run(base, x)                                  # (allocates the stream's workspace)
    y = torch.zeros(2, L.out_features, dtype=x.dtype, device="cuda")
    assert launched_kernels(lambda: pytest.raises(RuntimeError, run, d, x, [y])) == []
    assert bool((y == 0).all())
    head_zero()


def test_misaligned_x_takes_the_default_route(small):
    from _gpu import make_module
    L = small[0]
    m = make_module(L).set_list_decode(True)
    x = torch.from_numpy(vo.to_f32(vo.make_x(4, 4100, "fp16", seed=14), "fp16")).cuda().half()
    buf = torch.zeros(4 * 4100 + 8, dtype=x.dtype, device="cuda")
    xm = buf[1:1 + 4 * 4100].view(4, 4100)
    xm.copy_(x)
    import _extreme as ex
    exact = ex.y_star(L, x)
    with torch.no_grad():
        for tokens in (1, 2, 4):
            xt = xm[:tokens]
            names = launched_kernels(lambda: m(xt))
            assert not ran(names, KERNEL), names
            assert_close(m(xt), exact[:tokens], "fp16", q_of(4100, 65536))
        assert ran(launched_kernels(lambda: m(x[:2])), KERNEL)       # (aligned: the v = 16 kernel)


def test_probes_resolve_the_fixed_point_quantum():
    """bf16, weight_scale about 2^-17 and no weight_bias: most probe outputs c x' lie in (2^-25, 2^-22), where a bf16
    ulp is at most the 2^-30 step of the fixed point, so the kernel's round-to-nearest-even of each unit sum shows in
    the output bits (truncating the unit sums instead changes about 40 % of these outputs)"""
    import _extreme as ex
    L = vo.make_layer(in_features=1024, out_features=264, vector_len=16, num_centroids=65536, num_res_centroids=256,
                      seed=73, dtype="bf16")
    s = np.random.default_rng(2).uniform(1.0, 2.0, 1024) * 2.0 ** -17
    L = ex.copy_layer(L)
    L.weight_scale, L.weight_bias = ex.encode(s, "bf16"), ex.encode(np.zeros(1024), "bf16")
    d = desc_of(L)
    expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(torch.bfloat16)
    mag = expect.double().abs()
    assert float(mag.max()) < 2.0 ** -19 and float(((mag > 2.0 ** -25) & (mag < 2.0 ** -22)).double().mean()) > 0.5
    rng = np.random.default_rng(3)
    for rep in range(3):
        for tokens in (1, 2, 3, 4):
            f = rng.choice(1024, size=tokens, replace=False)
            xp = torch.zeros(tokens, 1024, dtype=torch.bfloat16, device="cuda")
            xp[torch.arange(tokens), torch.from_numpy(f).cuda()] = 1.0
            y = run(d, xp)
            if rep == 0 and tokens == 4:
                only_kernel(lambda: run(d, xp, [y]), launches=1)
            torch.cuda.synchronize()
            # (by value: an output whose unit sums all round to 0 is a zero of either sign)
            assert torch.equal(y.float(), expect[torch.from_numpy(f).cuda()].float()), (rep, f)
    head_zero()
