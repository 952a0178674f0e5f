"""The generic decode GEMV in every launch plan its planner chooses on an H100, against fp64.

The shapes come from the census of tests/_gemv_plan.py (the smallest shape of each plan class: warps, codebook
placement and replication, ring depth, chunk count, cluster or global reduction on both sides of the 16 KiB
partial-sum limit, wsplit 1 / 2 / 4 and an empty warp sub-range, one or several rows per CTA, outliers, every
vector length).  Every test asserts the launch it means to run: kernel name, grid, block and dynamic shared memory
from torch.profiler's trace, equal to the mirror's plan.  Cluster plans may be clamped to the co-residency the
device reports; the clamped CTAs per chunk are read back as grid / nch and printed ("[clusters]").

Bars: every token within TOL max|y*_t| of fp64; one-hot probes bit-exact against the simulation of the kernel's
arithmetic (tests/_probe.py); a repeated call gives the same bits; the workspace head is zero afterwards.
"""
import json
import os
import tempfile
import time

import numpy as np
import pytest
import torch

import _extreme as ex
import _gemv_plan as gp
import vptq_oracle as vo
from _batch import head_zero
from _probe import probe_expect, to_dev, ulp_diff
from _util import TOL

pytestmark = pytest.mark.gpu

DT = {"fp16": 0, "bf16": 1}


# ------------------------------------------------------------------------------------------------------------------
# launches as the profiler records them
# ------------------------------------------------------------------------------------------------------------------
def launches(fn):
    """[(name, grid, block, dynamic shared memory)] of the kernels one call of `fn` launched, from torch.profiler's
    chrome trace.  `fn` runs between two marker kernels, `lead` seconds inside both ends of the session (see
    _probe.launched_kernels); the call is repeated with a longer lead until both markers are recorded."""
    from torch.profiler import ProfilerActivity, profile
    marker = torch.zeros(1, dtype=torch.int64, device="cuda")
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        for lead in (0.0, 0.05, 0.25, 1.0, 4.0):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                time.sleep(lead)
                marker.add_(1)
                torch.cuda.synchronize()
                fn()
                torch.cuda.synchronize()
                marker.add_(1)
                torch.cuda.synchronize()
                time.sleep(lead)
            prof.export_chrome_trace(path)
            with open(path) as f:
                ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
            ev.sort(key=lambda e: e["ts"])
            mk = [i for i, e in enumerate(ev) if "CUDAFunctorOnSelf_add<long>" in e["name"]]
            if len(mk) == 2:
                return [(e["name"], e["args"]["grid"][0], e["args"]["block"][0], e["args"]["shared memory"])
                        for e in ev[mk[0] + 1:mk[1]]]
    raise AssertionError("torch.profiler did not record both marker kernels: the launch cannot be asserted")


def _is(name, template_id):
    """the profiler's name is `void vptq_b200::<template-id>(vptq_b200::GemvParams)`"""
    return f"vptq_b200::{template_id}(" in name


def device_plan(d, tokens, launch):
    """The mirror's plan for what the device launched (name, grid, block, shared memory).  The planner asks the device
    how many clusters of each size it can hold; the answers depend on the die, so they are read back from the launch:
    the answer table (nearest the recorded H100's first) under which the mirror gives the launched grid, block and
    shared memory.  They are printed for the record.  Fails only if no answers explain the launch."""
    name, grid, block, smem = launch

    def run(clusters):
        p = gp.make_plan(d, tokens, clusters=clusters)
        return (p.grid, p.threads, p.smem_bytes), p
    found = gp.explain_answers(run, (grid, block, smem))
    assert found, f"no co-residency answers give the launch {launch} (no-device plan {gp.make_plan(d, tokens)})"
    table, p = found
    if p.cpc < p.cpc_unclamped or table != {k: v for k, v in gp.H100_CLUSTERS.items() if k in table}:
        print(f"\n[clusters] answers {table}: nch={p.nch} cpc {p.cpc_unclamped} -> {p.cpc}", end="")
    return p, table


def assert_launch(d, dtype, got, tokens):
    """the launches `got` of one call with `tokens` tokens are the passes of the mirror's plan (4 -> 2 -> 1 tokens
    each), every one with its kernel, grid, block and shared memory; returns the plan and the device's answers"""
    assert got and all("gemv_kernel" in n for n, *_ in got), got
    p, table = device_plan(d, min(tokens, 4), got[0])
    want = p.passes(tokens)
    assert len(got) == len(want), (got, want)
    for (name, grid, block, smem), nt in zip(got, want):
        assert _is(name, p.kernel_name(DT[dtype], nt)), (name, p.kernel_name(DT[dtype], nt), p)
        assert (grid, block, smem) == (p.grid, p.threads, p.smem_bytes), ((grid, block, smem), p)
    return p, table


# ------------------------------------------------------------------------------------------------------------------
# layers, references
# ------------------------------------------------------------------------------------------------------------------
def make(d, dtype, seed):
    """oracle layer of the census shape d (norm, perm, bias; outliers of vector length 4) and its descriptor without
    index lists (the generic kernel is the only decode route)"""
    from test_gpu_probes import module
    L = vo.make_layer(in_features=d.I, out_features=d.O, vector_len=d.v, num_centroids=d.K,
                      num_res_centroids=d.Kr, num_codebooks=d.G, outlier_size=d.S,
                      outlier_vector_len=4 if d.S else -1, num_outlier_centroids=64 if d.S else -1, bias=True,
                      dtype=dtype, seed=seed)
    assert L.group_size == d.gs
    m, desc = module(L, lists=False)
    assert not desc.lists_stream
    return L, m, desc


def rand_x(L, tokens, seed):
    from _gpu import x_to_t
    return x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)


def gemv(desc, x, O):
    from vptq_b200 import native
    y = torch.full((x.shape[0], O), float("nan"), dtype=x.dtype, device="cuda")
    native.quant_gemv(desc, x, y)
    return y


def gemv_launches(desc, x, O):
    """launches() of one quant_gemv call (its output allocated outside the profiled region)"""
    from vptq_b200 import native
    y = torch.empty(x.shape[0], O, dtype=x.dtype, device="cuda")
    return launches(lambda: native.quant_gemv(desc, x, y))


def assert_fp64(y, ystar, dtype, what):
    """per token: max|y - y*| <= TOL max|y*_t|"""
    assert torch.isfinite(y).all(), what
    for t in range(y.shape[0]):
        err = float((y[t].double() - ystar[t]).abs().max())
        bar = TOL[dtype] * float(ystar[t].abs().max())
        assert err <= bar, (what, t, err, bar)


def probe_features(L, p, n_rand=16, seed=0):
    """input features whose one-hot probes reach every chunk at its first and last column and at every warp
    sub-range boundary, the outlier columns, and a few others"""
    q = set()
    if L.enable_outlier:
        q |= {0, L.outlier_size - 1}
    S = L.outlier_size if L.enable_outlier else 0
    for g in range(L.num_codebooks):
        for c in range(p.cpg):
            f0 = c * p.chunk_cols
            f1 = min(L.group_size, f0 + p.chunk_cols)
            for s in range(f0, f1, p.sub_cols):
                q |= {S + g * L.group_size + s, S + g * L.group_size + min(f1, s + p.sub_cols) - 1}
    q |= set(np.random.default_rng(seed).integers(0, L.in_features, n_rand).tolist())
    perm = np.asarray(L.perm).astype(np.uint16).astype(np.int64) if L.perm is not None else np.arange(L.in_features)
    return sorted({int(perm[c]) for c in q})


def assert_probes(L, run, feats, tokens, what):
    """one-hot probes e_f, `tokens` per call of run(X, Y), bit-exact against probe_expect(L, "generic")"""
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    n = len(feats)
    X = torch.zeros(n, (L.in_features + 7) // 8 * 8, dtype=dt, device="cuda")[:, :L.in_features]
    X[torch.arange(n), torch.tensor(feats)] = 1.0
    Y = torch.full((n, L.out_features), float("nan"), dtype=dt, device="cuda")
    for i in range(0, n, tokens):
        run(X[i:i + tokens], Y[i:i + tokens])
    torch.cuda.synchronize()
    want = to_dev(probe_expect(L, "generic")[feats], L)
    d = ulp_diff(Y, want)
    assert int(d.max()) == 0, f"{what}: {int(d.max())} ulp at {np.unravel_index(int(d.argmax()), d.shape)}"


# ------------------------------------------------------------------------------------------------------------------
# 1. every census shape at 1 and 2 tokens
# ------------------------------------------------------------------------------------------------------------------
def _census_shapes():
    """distinct census shapes, each with the classes it stands for"""
    by = {}
    for name, (d, p) in gp.census().items():
        by.setdefault(d, []).append(name)
    return sorted(by.items(), key=lambda kv: gp.shape_size(kv[0]))


SHAPES = _census_shapes()


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("d,classes", SHAPES, ids=["+".join(c) for _, c in SHAPES])
def test_census_plan(d, classes, dtype):
    """launch = the mirror's plan and still in its classes; fp64 bar per token; exact probes; same bits twice;
    workspace head zero"""
    from vptq_b200 import native
    L, m, desc = make(d, dtype, seed=11 + d.v + d.G)
    W = torch.from_numpy(ex.dense64(L)).cuda()
    for tokens in (1, 2):
        x = rand_x(L, tokens, seed=tokens)
        got = gemv_launches(desc, x, L.out_features)
        p, table = assert_launch(d, dtype, got, tokens)
        # the census is of single-token plans, robust to the answers of gp.census_models()
        if tokens == 1 and gp.within_census_range(table):
            lost = [c for c in classes if not gp.CLASSES[c](d, p)]
            assert not lost, (lost, p)
        elif tokens == 1:
            print(f"\n[clusters] answers {table} outside the census range: classes {classes} not asserted", end="")
        y = gemv(desc, x, L.out_features)
        assert_fp64(y, ex.y_star(L, x, W), dtype, f"{classes} x{tokens}")
        y2 = gemv(desc, x, L.out_features)
        assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), "a repeated call changed bits"
        head_zero()
        assert_probes(L, lambda X, Y: native.quant_gemv(desc, X, Y), probe_features(L, p), tokens,
                      f"{classes} {dtype} x{tokens}")
    head_zero()


# ------------------------------------------------------------------------------------------------------------------
# 2. tail passes of plans sized for 4 tokens
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", sorted(gp.TAIL_SHAPES))
def test_tail_passes(kind):
    """3, 5, 6 and 7 tokens on an nt = 4 plan: passes 4 / 2 / 1 from the launched kernels, each token at the fp64
    bar, same bits twice"""
    d = gp.TAIL_SHAPES[kind]
    L, m, desc = make(d, "fp16", seed=21)
    W = torch.from_numpy(ex.dense64(L)).cuda()
    for tokens in (3, 5, 6, 7):
        x = rand_x(L, tokens, seed=100 + tokens)
        got = gemv_launches(desc, x, L.out_features)
        p, _ = assert_launch(d, "fp16", got, tokens)
        assert p.nt == (4 if tokens >= 4 else 2) and len(got) == len(p.passes(tokens)) > 1
        y = gemv(desc, x, L.out_features)
        assert_fp64(y, ex.y_star(L, x, W), "fp16", f"{kind} x{tokens}")
        assert torch.equal(y.view(torch.int16), gemv(desc, x, L.out_features).view(torch.int16))
    head_zero()


# ------------------------------------------------------------------------------------------------------------------
# 3. fused launches of 2-4 layers on one x
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("group", sorted(gp.FUSED_GROUPS))
def test_fused_launch(group):
    """one gemv_multi_kernel launch whose grid is the sum of the members' grids and whose shared memory is their
    maximum; each member's slice at the fp64 bar with exact probes.  A group the C side refuses runs one launch
    per layer inside native.FusedGemv, bit-identical to the layers called alone."""
    from vptq_b200 import native
    descs, fused = gp.FUSED_GROUPS[group]
    layers = [make(d, "fp16", seed=31 + i) for i, d in enumerate(descs)]
    I = descs[0].I
    for tokens in (1, 2):
        x = rand_x(layers[0][0], tokens, seed=200 + tokens)
        ys = [torch.full((tokens, d.O), float("nan"), dtype=torch.float16, device="cuda") for d in descs]
        fg = native.FusedGemv([c for _, _, c in layers], ys)
        fg(x)                  # (the first call may allocate the workspace)
        got = launches(lambda: fg(x))
        if fused:
            assert not fg.separate and len(got) == 1, got
            name, grid, block, smem = got[0]

            def run(clusters):
                plans, g, s = gp.multi_plan(descs, tokens, clusters=clusters)
                return (g, plans[0].threads, s), (plans, g, s)
            found = gp.explain_answers(run, (grid, block, smem))
            assert found, (got, gp.multi_plan(descs, tokens))
            table, (plans, g_want, s_want) = found
            print(f"\n[clusters] fused {group} x{tokens}: answers {table}", end="")
            assert g_want == sum(p.grid for p in plans) and s_want == max(p.smem_bytes for p in plans)
            assert _is(name, plans[0].kernel_name(0, tokens, multi=True)), (name, plans[0])
        else:
            assert fg.separate, "the C side took a group it should refuse"
            assert len(got) == len(descs), got
            for launch, d in zip(got, descs):
                assert_launch(d, "fp16", [launch], tokens)
        fg(x)
        torch.cuda.synchronize()
        first = [y.clone() for y in ys]
        fg(x)
        torch.cuda.synchronize()
        for (L, _, desc), y, y0, d in zip(layers, ys, first, descs):
            assert torch.equal(y.view(torch.int16), y0.view(torch.int16)), f"{group}: a repeated call changed bits"
            assert_fp64(y, ex.y_star(L, x), "fp16", f"{group} O={d.O} x{tokens}")
            if not fused:
                alone = gemv(desc, x, d.O)
                assert torch.equal(y.view(torch.int16), alone.view(torch.int16)), "fallback != the layer alone"
        head_zero()
    # probes through the fused launch, member by member
    feats = sorted(set(np.random.default_rng(5).integers(0, I, 24).tolist()) | {0, I - 1})
    dt = torch.float16
    X = torch.zeros(len(feats), I, dtype=dt, device="cuda")
    X[torch.arange(len(feats)), torch.tensor(feats)] = 1.0
    Ys = [torch.full((len(feats), d.O), float("nan"), dtype=dt, device="cuda") for d in descs]
    for i in range(len(feats)):
        native.FusedGemv([c for _, _, c in layers], [Y[i:i + 1] for Y in Ys])(X[i:i + 1])
    torch.cuda.synchronize()
    for (L, _, _), Y in zip(layers, Ys):
        want = to_dev(probe_expect(L, "generic")[feats], L)
        assert int(ulp_diff(Y, want).max()) == 0, group
