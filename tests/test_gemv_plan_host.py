"""The generic decode GEMV's launch planner without a GPU (tests/_gemv_plan.py mirrors gemv_make_plan and the fused
launch's shares):

* the mirror against the library's own planner over a seeded sweep of descriptors the C ABI accepts, through
  vptq_b200_workspace_bytes(OP_GEMV) on the H100 geometry (counter head + global partial sums: pins the chunk count,
  cluster or global reduction, and refusals);
* the census of plan classes the cost model reaches on an H100, each with its smallest test shape (the GPU file
  tests/test_gpu_gemv_plans.py runs those shapes and asserts their launches);
* the invariants every plan must keep under any cluster co-residency answer the device may give.
"""
import numpy as np
import pytest

import _gemv_plan as gp

VS = (2, 4, 6, 8, 10, 12, 16)
TOKENS = (1, 2, 3, 4, 5, 8)


def _sweep(n=3000, seed=20261018):
    """seeded descriptors the C ABI accepts: every v, K and Kr up to 65536 (b <= 32), 1..16 groups, ragged group
    sizes, outliers, in_features up to 65535, up to ~100k output rows, the token counts of decode"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        v = int(rng.choice(VS))
        K = 1 << int(rng.integers(1, 17))
        Kr = -1 if rng.random() < 0.3 else 1 << int(rng.integers(1, 17))
        if Kr > 0 and gp.ilog2(K) + gp.ilog2(Kr) > 32:
            continue
        G = int(rng.integers(1, 17)) if rng.random() < 0.5 else int(rng.choice((1, 2, 4, 8, 16)))
        S = int(rng.integers(1, 513)) if rng.random() < 0.15 else 0
        gmax = (65535 - S) // G
        if gmax < 1:
            continue
        r = rng.random()
        if r < 0.3:
            gs = int(rng.integers(1, max(2, gmax // 128 + 1))) * 128          # whole 128-column blocks
        elif r < 0.5:
            gs = int(rng.integers(1, min(gmax, 512) + 1))                       # narrow, ragged
        else:
            gs = int(np.exp(rng.uniform(0, np.log(gmax + 1))))                  # log-uniform, ragged
        gs = max(1, min(gs, gmax))
        O = max(1, int(np.exp(rng.uniform(0, np.log(100000)))))
        out.append((gp.Desc(v=v, K=K, Kr=Kr, G=G, gs=gs, O=O, S=S, dtype=int(rng.integers(0, 2))),
                    int(rng.choice(TOKENS))))
    return out


SWEEP = _sweep()


def _mirror_workspace(d, tokens):
    try:
        return gp.make_plan(d, tokens).workspace_bytes
    except gp.Refused:
        return 0


def test_mirror_matches_the_library_planner():
    """workspace bytes of the mirror == the library's, descriptor by descriptor (0 where both refuse)"""
    lib = gp.library_workspaces_without_device(SWEEP)
    bad = []
    kinds = {"nch1": 0, "cluster": 0, "global": 0, "refused": 0}
    for (d, t), (ws, err) in zip(SWEEP, lib):
        want = _mirror_workspace(d, t)
        if ws != want:
            bad.append((d, t, ws, want, err))
        if not ws:
            kinds["refused"] += 1
            assert gp.NO_LAYOUT in err or "index rows" in err, (d, t, err)
            continue
        p = gp.make_plan(d, t)
        kinds["nch1" if p.nch == 1 else "cluster" if p.cluster else "global"] += 1
    print(f"\n[plans] {len(SWEEP)} descriptors: {kinds}")
    assert not bad, f"{len(bad)} mismatches, first {bad[:5]}"
    # the sweep reaches every reduction kind and the refusal
    assert all(kinds.values()), kinds


def test_census_covers_every_plan_class():
    """every class has a shape (the smallest), and the fused-launch and tail-pass shapes plan as the GPU file needs"""
    c = gp.census()
    missing = sorted(set(gp.CLASSES) - set(c))
    assert not missing, missing
    for name, (d, p) in sorted(c.items()):
        assert gp.CLASSES[name](d, p)
        print(f"\n[census] {name:24s} v={d.v} K={d.K} Kr={d.Kr} G={d.G} gs={d.gs} O={d.O} S={d.S}: "
              f"threads={p.threads} nch={p.nch} cpc={p.cpc} wsplit={p.wsplit} stages={p.stages} "
              f"main={'smem x%d' % p.main_rep if p.main_in_smem else 'L2'} "
              f"res={('smem x%d' % p.res_rep if p.res_rep else 'L2') if p.has_res else 'none'} "
              f"cluster={p.cluster} smem={p.smem_bytes}", end="")
    # both sides of the cluster partial-sum limit, at the same chunk count
    at, over = c["cluster_part_at_limit"][1], c["global_part_over_limit"][1]
    assert gp.part_bytes(at) == gp.MAX_CLUSTER_PART_BYTES < gp.part_bytes(over) and at.nch == over.nch
    # the shapes the GPU file runs through the tail passes and the fused launches
    for name, d in gp.TAIL_SHAPES.items():
        for tokens, passes in ((3, [2, 1]), (5, [4, 1]), (6, [4, 2]), (7, [4, 2, 1])):
            p = gp.make_plan(d, tokens, clusters=gp.h100_clusters)   # the library plans for the call's token count
            assert {"cluster": p.cluster == 1, "global": p.nch > 1 and not p.cluster, "nch1": p.nch == 1}[name], p
            assert p.passes(tokens) == passes, (name, tokens, p)
    for name, (descs, fused) in gp.FUSED_GROUPS.items():
        for tokens in (1, 2):
            if not fused:
                with pytest.raises(gp.Refused, match="one launch configuration"):
                    gp.multi_plan(descs, tokens, clusters=gp.h100_clusters)
                continue
            plans, grid, smem = gp.multi_plan(descs, tokens, clusters=gp.h100_clusters)
            alone = [gp.make_plan(d, tokens, clusters=gp.h100_clusters) for d in descs]
            # some member is planned differently than alone: the share and the imposed cpg move it
            assert any((p.cpc, p.cpg) != (a.cpc, a.cpg) for p, a in zip(plans, alone)), name
            assert (plans[0].cluster == 1) == ("cluster" in name), name


def test_invariants_under_every_cluster_answer():
    """For every sweep descriptor and every co-residency answer n (cudaOccupancyMaxActiveClusters, 1..66):
    the rows a CTA owns after the clamp fit the tables the carve sized for them (s_part, s_wsum, s_wcnt), the layout
    fits the opt-in, a cluster grid is whole clusters, and the global reduction's row counters stay inside the
    256 KiB head"""
    checked, clamped, recarved = 0, 0, 0
    for d, t in SWEEP[:1000]:
        try:
            base = gp.make_plan(d, t)
        except gp.Refused:
            continue
        for n in list(range(1, gp.H100_SMS // 2 + 1)) + [gp.H100_SMS]:
            try:
                p = gp.make_plan(d, t, clusters=lambda nch, threads, smem, n=n: n)
            except gp.Refused:
                continue
            checked += 1
            clamped += p.cpc < p.cpc_unclamped
            recarved += p.rows_alloc > base.rows_alloc
            if p.cluster or p.wsplit > 1:
                assert p.rows_cta <= p.rows_alloc, (d, t, n, p)
            if p.cluster:
                assert 2 <= p.nch <= 8 and p.grid % p.nch == 0 and gp.part_bytes(p) <= gp.MAX_CLUSTER_PART_BYTES
            assert p.smem_bytes <= gp.H100_OPTIN - gp.SMEM_RESERVE, (d, t, n, p)
            assert p.grid == p.nch * p.cpc and 1 <= p.cpc <= p.Ro
            if p.nch > 1 and not p.cluster:
                assert p.Ro * 4 <= gp.COUNTER_REGION_BYTES
                assert p.ws_partials_bytes >= p.nch * p.nt * p.Ro * p.v * 4
            # an answer of at least cpc clamps nothing: the plan is the no-device plan
            if n >= gp.H100_SMS:
                assert p == base
    print(f"\n[invariants] {checked} plans, {clamped} clamped, {recarved} carved again after the clamp")
    assert clamped and recarved


def test_recarve_after_the_clamp():
    """A cluster plan with split rows whose co-residency clamp leaves more rows per CTA than the partial-sum table
    holds: the planner falls back to the global reduction and sizes s_wsum / s_wcnt for the clamped rows (before,
    their rows past the carve ran into the residual codebook behind them)"""
    d = gp.Desc(v=2, K=256, Kr=-1, G=2, gs=2048, O=64)
    base = gp.make_plan(d, 1)
    assert base.cluster and base.wsplit == 2
    # the cost model's own query (at 200 KiB) sees room for every cluster, the query at the plan's footprint for one
    p = gp.make_plan(d, 1, clusters=lambda nch, threads, smem: gp.H100_SMS if smem == 200 * 1024 else 1)
    assert p.cpc == 1 and not p.cluster and p.wsplit == 2
    assert p.rows_alloc == p.rows_cta == d.Ro > base.rows_alloc
    assert p.ws_partials_bytes == gp.align_up(p.nch * p.nt * d.Ro * d.v * 4, 256)


@pytest.mark.parametrize("table", [{4: 30, 8: 15}, {4: 31, 8: 16}, {2: 64, 4: 29, 8: 14}, {3: 40, 6: 20, 7: 16}],
                         ids=lambda t: "-".join(f"{k}:{v}" for k, v in t.items()))
def test_answers_are_read_back_from_a_launch(table):
    """what the GPU file does with a launch: for a device answering `table`, the answers found from the launched
    grid, block and shared memory give that device's plan, for every census shape and fused group"""
    dev = gp.table_clusters(table)
    for d, _ in gp.census().values():
        want = gp.make_plan(d, 1, clusters=dev)

        def run(clusters):
            p = gp.make_plan(d, 1, clusters=clusters)
            return (p.grid, p.threads, p.smem_bytes), p
        found = gp.explain_answers(run, (want.grid, want.threads, want.smem_bytes))
        assert found and found[1] == want, (d, table, found)
    for descs, fused in gp.FUSED_GROUPS.values():
        if fused:
            want = gp.multi_plan(descs, 1, clusters=dev)

            def run(clusters):
                plans, g, s = gp.multi_plan(descs, 1, clusters=clusters)
                return (g, plans[0].threads, s), (plans, g, s)
            found = gp.explain_answers(run, (want[1], want[0][0].threads, want[2]))
            assert found and found[1][1:] == want[1:], (descs, table, found)
