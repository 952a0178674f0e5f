"""Integer mirror of the generic decode GEMV's planner: gemv_make_plan and the share / forced-cpg logic of
gemv_multi_launch (vptq_b200/csrc/gemv.cu).  Written from the C++ as it stands; the tests decide whether the two
agree (tests/test_gemv_plan_host.py against the library's own planner, tests/test_gpu_gemv_plans.py against the
launches an H100 records).

`clusters(nch, threads, smem)` stands for cudaOccupancyMaxActiveClusters of the kernel at that cluster size, block
size and dynamic shared memory (<= 0: unknown).  `clusters=None` means "no device", as on a CPU-only host: no
occupancy query is made and no clamp is applied.  `tune` mirrors the developer knob VPTQ_B200_GEMV_TUNE
(keys rep, stages, seg, warps, cpg, cluster, wsplit).
"""
import ctypes
import dataclasses
import json
import os
import subprocess
import sys
from typing import Callable, Optional

MAX_CHUNK_COLS = 4096
SMEM_RESERVE = 2048
MAX_CLUSTER_PART_BYTES = 16384
MAX_INDEX_ROWS = 65536
ZERO_REGION_BYTES = MAX_INDEX_ROWS * 4 + MAX_INDEX_ROWS * 64     # kZeroRegionBytes: counters, then accumulators
COUNTER_REGION_BYTES = MAX_INDEX_ROWS * 4
MAX_FUSED = 4
H100_SMS, H100_OPTIN = 132, 232448                                # the geometry the CPU path assumes
NO_LAYOUT = "no shared-memory layout fits"
# cudaOccupancyMaxActiveClusters of the GEMV kernels (one CTA per SM) by cluster size, as one H100 SXM (132 SMs)
# answered them; sizes not listed clamped no tested plan there.  The answer depends on how many SMs each GPC of a
# given die has, so another H100 may answer differently: tests/test_gpu_gemv_plans.py reads the answers of the device
# it runs on back from its launches (explain_answers).
H100_CLUSTERS = {4: 30, 8: 15}
# the census keeps a shape in a class only if it stays there for every answer from this fraction of
# floor(132 / size) up to floor(132 / size) (no clamp)
CENSUS_ANSWER_FLOOR = 0.85


def table_clusters(table):
    """the co-residency query as a table {cluster size: answer} (sizes not in it: no answer, no clamp)"""
    return lambda nch, threads, smem: table.get(nch, -1)


h100_clusters = table_clusters(H100_CLUSTERS)


def max_answer(k, sms=H100_SMS):
    return sms // k


def queried_sizes(run):
    """the cluster sizes `run(clusters)` asks about (the sizes asked do not depend on the answers)"""
    sizes = set()

    def rec(nch, threads, smem):
        sizes.add(nch)
        return -1
    run(rec)
    return sorted(sizes)


def explain_answers(run, observed, recorded=H100_CLUSTERS, budget=40000):
    """The co-residency answers under which `run(clusters)` gives `observed`: {size: answer} tables over the sizes
    `run` queries, tried in order of their distance from `recorded` (answers >= floor(132 / size) clamp nothing and
    count as that value).  Returns (table, result of run), or None when no table explains the observation."""
    import itertools
    sizes = queried_sizes(run)
    axes = []
    for k in sizes:
        top = max_answer(k)
        ref = min(recorded.get(k, top), top)
        axes.append(sorted(range(1, top + 1), key=lambda n: (abs(n - ref), -n)))
    combos = sorted(itertools.product(*[range(len(a)) for a in axes]), key=sum)[:budget]
    for c in combos:
        table = {k: axes[i][j] for i, (k, j) in enumerate(zip(sizes, c))}
        try:
            got = run(table_clusters(table))
        except Refused:
            continue
        if got[0] == observed:
            return table, got[1]
    return None


def within_census_range(table):
    """every answer of `table` lies in the range the census made its classes robust to"""
    return all(max_answer(k) * CENSUS_ANSWER_FLOOR <= n for k, n in table.items())


def ilog2(v):
    return int(v).bit_length() - 1


def align_up(v, a):
    return (v + a - 1) // a * a


@dataclasses.dataclass(frozen=True)
class Desc:
    """The descriptor fields the planner reads.  Kr <= 0: no residual codebook; S: outlier columns (0: none)."""
    v: int
    K: int
    Kr: int
    G: int
    gs: int
    O: int
    S: int = 0
    dtype: int = 0          # 0 fp16, 1 bf16 (picks the kernel, not the plan)

    @property
    def I(self):
        return self.S + self.G * self.gs

    @property
    def Ro(self):
        return (self.O + self.v - 1) // self.v


@dataclasses.dataclass
class Plan:
    threads: int
    grid: int
    nch: int
    cpg: int
    chunk_cols: int
    cpc: int
    wsplit: int
    sub_cols: int
    stages: int
    main_in_smem: int
    main_rep: int
    res_rep: int            # 0: residual gathered through L1/L2 (or no residual codebook: see has_res)
    cluster: int
    nt: int
    smem_bytes: int
    ws_partials_bytes: int
    rows_alloc: int         # index rows per CTA the carve sized s_part, s_wsum and s_wcnt for
    cpc_unclamped: int      # min(slots / nch, Ro): cpc before the cluster co-residency clamp
    has_res: bool
    v: int
    Ro: int

    @property
    def rows_cta(self):
        """index rows the CTA owning the first row of a chunk works on (the kernel's nrows_cta at cta_in_chunk 0)"""
        return (self.Ro + self.cpc - 1) // self.cpc

    @property
    def res_l2(self):
        return self.has_res and self.res_rep == 0

    @property
    def workspace_bytes(self):
        """what vptq_b200_workspace_bytes(OP_GEMV) reports for this plan (a descriptor without index lists)"""
        return ZERO_REGION_BYTES + self.ws_partials_bytes

    def kernel_name(self, dtype, nt=None, multi=False):
        """the template-id of the kernel a pass of `nt` tokens launches, as the profiler prints it"""
        nt = self.nt if nt is None else nt
        T = "__half" if dtype == 0 else "__nv_bfloat16"
        b = lambda x: "true" if x else "false"
        base = "gemv_multi_kernel" if multi else "gemv_kernel"
        if self.res_l2:
            return f"{base}_res_l2<{T}, {self.v}, {nt}, {b(self.main_in_smem)}>"
        return f"{base}<{T}, {self.v}, {nt}, {b(self.main_in_smem)}, {b(self.has_res)}>"

    def passes(self, tokens):
        """tokens per launch of a call with `tokens` tokens: full passes of nt, then the tail 4 -> 2 -> 1"""
        out, t0 = [], 0
        while t0 < tokens:
            nt = self.nt
            while nt > tokens - t0:
                nt >>= 1
            out.append(nt)
            t0 += nt
        return out


class Refused(Exception):
    pass


def make_plan(d: Desc, tokens: int, sms: int = H100_SMS, optin: int = H100_OPTIN,
              clusters: Optional[Callable[[int, int, int], int]] = None, slots_override: int = 0, force_cpg: int = 0,
              tune: Optional[dict] = None) -> Plan:
    """gemv_make_plan.  Raises Refused (with the library's reason) where the C++ returns VPTQ_ERR_UNSUPPORTED."""
    tn = dict(rep=-1, stages=0, seg=0, warps=0, cpg=0, cluster=-1, wsplit=0)
    tn.update(tune or {})
    v, G, gs = d.v, d.G, d.gs
    Ro = d.Ro
    ib = ilog2(d.K)
    rb = ilog2(d.Kr) if d.Kr > 0 else 0
    b = ib + rb
    S = d.S
    EB = 2 * v
    if Ro > MAX_INDEX_ROWS:
        raise Refused("index rows exceed the supported maximum")
    nt = (4 if tokens >= 4 else 2 if tokens >= 2 else 1) if v == 8 else 1
    seg_fields = tn["seg"] or 512
    stage_bytes = align_up(seg_fields * b // 8 + 16, 16)

    main_bytes = d.K * EB
    res_bytes = d.Kr * EB if rb else 0
    main_fits = main_bytes <= 131072
    main_rep_smem = 8 if (v == 8 and main_bytes * 8 <= 32768) else 1
    res_rep_want = (8 if tn["rep"] else 1) if tn["rep"] >= 0 else 8
    res_rep_max = res_rep_want if (rb and v == 8 and res_bytes * 8 <= 32768) else 1
    smem_limit = optin - SMEM_RESERVE
    slots = min(slots_override, sms) if slots_override > 0 else sms
    query = clusters is not None and tn["cluster"] != 0

    attempts = [(16, True, True), (8, True, True), (16, False, True), (8, False, True),
                (16, True, False), (8, True, False), (16, False, False), (8, False, False)]
    for warps, main_smem, res_smem in attempts:
        if main_smem and not main_fits:
            continue
        if not res_smem and not rb:
            continue
        if tn["warps"] and warps != tn["warps"]:
            continue
        res_smem_bytes = res_bytes if res_smem else 0

        # ---- column chunks x warps per row: the cost model
        best_cpg, best_cc, best_ws, best_cost = 0, 0, 1, 1e300
        cpg = 1
        while cpg <= 64:
            if (tn["cpg"] and cpg != tn["cpg"]) or (force_cpg and cpg != force_cpg):
                cpg *= 2
                continue
            cc = align_up((gs + cpg - 1) // cpg, 128)
            if cc > MAX_CHUNK_COLS:
                cpg *= 2
                continue
            if cpg > 1 and cc < 256:
                break
            real_cpg = (gs + cc - 1) // cc
            nch = G * real_cpg
            if nch > slots:
                break
            cpc = max(1, min(slots // nch, Ro))
            if 2 <= nch <= 8 and query:
                n = clusters(nch, warps * 32, 200 * 1024)
                if n > 0:
                    cpc = min(cpc, n)
            rows_cta = (Ro + cpc - 1) // cpc
            for ws in (1, 2, 4):
                if tn["wsplit"] and ws != tn["wsplit"]:
                    continue
                sub = align_up((cc + ws - 1) // ws, 128)
                if ws > 1 and (sub < 256 or (ws - 1) * sub >= cc):
                    continue
                nslots = warps // ws
                rounds = (rows_cta + nslots - 1) // nslots
                util = float(rows_cta) * ws / (float(rounds) * warps)
                cost = float(rows_cta) * cc * (1.0 + 0.5 * (1.0 - util)) + 600.0 + 0.35 * cc
                cost += (24.0 if nch <= 8 else 96.0) * rows_cta + (16.0 * rows_cta if ws > 1 else 0.0)
                cost *= 1.0 + 0.01 * ilog2(real_cpg)
                if cost < best_cost:
                    best_cost, best_cpg, best_cc, best_ws = cost, real_cpg, cc, ws
            cpg *= 2
        if not best_cpg:
            best_cc = MAX_CHUNK_COLS
            best_cpg = (gs + MAX_CHUNK_COLS - 1) // MAX_CHUNK_COLS
            best_ws = 1
        chunk_cols, cpg_, nch = best_cc, best_cpg, G * best_cpg
        wsplit = best_ws
        sub_cols = align_up((best_cc + best_ws - 1) // best_ws, 128) if best_ws > 1 else best_cc
        if nch > slots:
            continue
        cpc = max(1, min(slots // nch, Ro))
        cpc_unclamped = cpc
        rows_cta = (Ro + cpc - 1) // cpc
        rows_alloc = rows_cta + rows_cta // 4 + 1
        part_bytes = rows_alloc * nch * nt * v * 4
        cluster = 1 if (2 <= nch <= 8 and part_bytes <= MAX_CLUSTER_PART_BYTES and tn["cluster"] != 0) else 0
        main_rep = main_rep_smem if main_smem else 1

        def carve(stages, res_rep, cluster, rows_alloc):
            off = align_up((2 + warps * stages) * 8, 128)
            off += align_up(nt * (1 + warps) * 4, 128)
            n_all = chunk_cols + S
            sx_stride = align_up(n_all, 32)
            off += align_up(n_all * 2, 128)
            off += align_up(n_all * 4, 128)
            off += align_up(nt * sx_stride * 4, 128)
            if cluster:
                off += align_up(rows_alloc * nch * nt * v * 4, 128)
            if wsplit > 1:
                off += align_up(rows_alloc * wsplit * nt * v * 4, 128)
                off += align_up(rows_alloc * 4, 128)
            off += align_up(res_smem_bytes * res_rep, 128)
            if main_smem:
                off += align_up(main_bytes * main_rep, 128)
            off += align_up((res_smem_bytes if res_rep > 1 else 0) + (main_bytes if main_smem and main_rep > 1 else 0),
                            128)
            off += align_up(warps * stages * stage_bytes, 128)
            return off

        shapes = [(st, rep) for st in ((4, 3, 2) if main_smem else (2,))
                  for rep in ((res_rep_max if res_smem else 0), (1 if res_smem else 0))]

        def place(cluster, rows_alloc):
            for st, rep in shapes:
                if tn["stages"] and st != tn["stages"]:
                    continue
                need = carve(st, rep, cluster, rows_alloc)
                if need <= smem_limit:
                    return st, rep, need
            return None

        placed = place(cluster, rows_alloc)
        if placed is None:
            continue
        stages, res_rep, smem = placed

        # ---- clusters must all be co-resident
        if cluster and query:
            n = clusters(nch, warps * 32, smem)
            if 0 < n < cpc:
                cpc = n
            rows2 = (Ro + cpc - 1) // cpc
            if rows2 > rows_alloc:          # global reduction, row tables carved again for the clamped cpc
                cluster, rows_alloc = 0, rows2
                placed = place(cluster, rows_alloc)
                if placed is None:
                    continue
                stages, res_rep, smem = placed
        grid = nch * cpc
        ws_partials = align_up(nch * nt * Ro * v * 4, 256) if (nch > 1 and not cluster) else 0
        return Plan(threads=warps * 32, grid=grid, nch=nch, cpg=cpg_, chunk_cols=chunk_cols, cpc=cpc, wsplit=wsplit,
                    sub_cols=sub_cols, stages=stages, main_in_smem=int(main_smem), main_rep=main_rep,
                    res_rep=res_rep, cluster=cluster, nt=nt, smem_bytes=smem, ws_partials_bytes=ws_partials,
                    rows_alloc=rows_alloc, cpc_unclamped=cpc_unclamped, has_res=rb > 0, v=v, Ro=Ro)
    raise Refused(NO_LAYOUT)


def multi_plan(descs, tokens, sms=H100_SMS, optin=H100_OPTIN, clusters=None, tune=None):
    """gemv_multi_launch's planning: (plans, grid, smem) of one fused launch, or Refused where the C++ returns
    VPTQ_ERR_UNSUPPORTED (the caller then launches the layers one by one)."""
    n = len(descs)
    if not 1 <= n <= MAX_FUSED or not 1 <= tokens <= 2:
        raise Refused("1..4 layers and 1..2 tokens")
    d0 = descs[0]
    for d in descs:
        if d.v != 8 or d.dtype != d0.dtype or d.I != d0.I or (d.Kr > 0) != (d0.Kr > 0):
            raise Refused("layers must share dtype, in_features, vector_len 8 and residual-ness")
    vol = [float(d.Ro) * d.I for d in descs]
    total = sum(vol)
    big = max(range(n), key=lambda l: (vol[l], -l))     # the first of the largest
    pb = make_plan(descs[big], tokens, sms, optin, clusters, max(8, int(sms * vol[big] / total)), 0, tune)
    cpg, nch = pb.cpg, pb.nch
    avail = sms
    if pb.cluster and clusters is not None:
        nmax = clusters(nch, pb.threads, 200 * 1024)
        if nmax > 0:
            avail = min(avail, nmax * nch)
    share = [max(nch, int(avail * vol[l] / total) // nch * nch) for l in range(n)]
    used = sum(share)
    while used > avail and share[big] > nch:
        share[big] -= nch
        used -= nch
    if used > avail:
        raise Refused("do not fit co-resident CTAs")
    while used + nch <= avail:
        share[big] += nch
        used += nch
    plans = [make_plan(d, tokens, sms, optin, clusters, share[l], cpg, tune) for l, d in enumerate(descs)]
    pb = plans[big]                                     # the members are held to the largest layer's final plan
    for p in plans:
        if (p.nch != pb.nch or p.threads != pb.threads or p.cluster != pb.cluster or p.main_in_smem != pb.main_in_smem
                or (p.res_rep > 0) != (pb.res_rep > 0) or p.nt != pb.nt or p.ws_partials_bytes):
            raise Refused("the layers do not admit one launch configuration")
    if plans[big].nt != tokens:
        raise Refused("no fused kernel for this configuration")
    return plans, sum(p.grid for p in plans), max(p.smem_bytes for p in plans)


# ------------------------------------------------------------------------------------------------------------------
# census: the plan classes the cost model reaches on an H100 (132 SMs, 232448 bytes of shared memory per block), and
# the smallest test shape of each
# ------------------------------------------------------------------------------------------------------------------
def part_bytes(p):
    """bytes of the cluster partial-sum table the plan's rows would need (cluster iff <= 16384 for nch 2..8)"""
    return p.rows_alloc * p.nch * p.nt * p.v * 4


def empty_subrange(d, p):
    """the last chunk of a codebook group is so narrow that a warp sub-range of it holds no column"""
    last = d.gs - (p.cpg - 1) * p.chunk_cols
    return p.wsplit > 1 and last <= (p.wsplit - 1) * p.sub_cols


CLASSES = {
    "warps16": lambda d, p: p.threads == 512,
    "warps8": lambda d, p: p.threads == 256,
    "main_smem_rep8": lambda d, p: p.main_in_smem and p.main_rep == 8,
    "main_smem_rep1": lambda d, p: p.main_in_smem and p.main_rep == 1,
    "main_l2": lambda d, p: not p.main_in_smem,
    "res_none": lambda d, p: not p.has_res,
    "res_rep8": lambda d, p: p.has_res and p.res_rep == 8,
    "res_rep1": lambda d, p: p.has_res and p.res_rep == 1,
    "res_l2": lambda d, p: p.res_l2,
    "stages4": lambda d, p: p.stages == 4,
    "stages3": lambda d, p: p.stages == 3,
    "stages2": lambda d, p: p.stages == 2,
    "nch1": lambda d, p: p.nch == 1 and p.cpc < p.Ro,
    "cluster": lambda d, p: p.cluster == 1,
    "cluster_part_at_limit": lambda d, p: p.cluster == 1 and part_bytes(p) == MAX_CLUSTER_PART_BYTES,
    "global_part_over_limit": lambda d, p: 2 <= p.nch <= 8 and not p.cluster and part_bytes(p) > MAX_CLUSTER_PART_BYTES,
    "global_nch_over_8": lambda d, p: p.nch > 8,
    "cluster_v_not_8": lambda d, p: p.cluster == 1 and p.v != 8,
    "wsplit1": lambda d, p: p.wsplit == 1,
    "wsplit2": lambda d, p: p.wsplit == 2,
    "wsplit4": lambda d, p: p.wsplit == 4,
    "wsplit_empty_subrange": empty_subrange,
    "one_row_per_cta": lambda d, p: p.cpc == p.Ro > 1,
    "rows_per_cta_gt1": lambda d, p: p.cpc < p.Ro,
    "outliers": lambda d, p: d.S > 0,
    **{f"v{v}": (lambda v: lambda d, p: p.v == v)(v) for v in (2, 4, 6, 8, 10, 12, 16)},
}


def _candidates():
    """deterministic test shapes: v = 8 over the axes that move the plan, then every other v on a few shapes"""
    gss = (128, 256, 300, 640, 1000, 1024, 1100, 1536, 2048, 2200, 3000, 4096, 4500, 8192)
    Os = (24, 64, 264, 1000, 2056, 4104, 6528, 12000)
    for K in (16, 256, 4096, 8192, 16384):
        for Kr in (-1, 16, 256, 512, 65536):
            if Kr > 0 and (K.bit_length() - 1) + (Kr.bit_length() - 1) > 32:
                continue
            for G in (1, 2, 4, 8, 16):
                for gs in gss:
                    for S in (0, 16):
                        if S + G * gs > 65535:
                            continue
                        for O in Os:
                            yield Desc(v=8, K=K, Kr=Kr, G=G, gs=gs, O=O, S=S)
    for v in (2, 4, 6, 10, 12, 16):
        for K in (256, 4096):
            for Kr in (-1, 256):
                for G in (1, 2, 4):
                    for gs in (256, 1024, 2048):
                        for O in (64, 264, 1000):
                            yield Desc(v=v, K=K, Kr=Kr, G=G, gs=gs, O=O)


def shape_size(d):
    """what a shape costs a test: the dense fp64 reference and the probes scale with I * O, staging with K and Kr"""
    return (d.I * d.O + 64 * d.v * (d.K + max(d.Kr, 0)), d.v, d.K, d.Kr, d.G, d.gs, d.O, d.S)


_CENSUS = None


def census_models():
    """the co-residency answers a census plan must keep its classes under: no clamp, the recorded H100, and every
    size answering CENSUS_ANSWER_FLOOR of its maximum"""
    lean = {k: int(max_answer(k) * CENSUS_ANSWER_FLOOR + 0.999) for k in range(2, 9)}
    return [None, h100_clusters, table_clusters(lean)]


def census(tokens=1):
    """{class: (Desc, Plan)}: the smallest candidate shape with more than one index row whose plan is in the class
    under every answer model of census_models() (the plan returned: the recorded H100's)"""
    global _CENSUS
    if _CENSUS is None:
        _CENSUS = {}
    if tokens in _CENSUS:
        return _CENSUS[tokens]
    best = {}
    models = census_models()
    for d in sorted(set(_candidates()), key=shape_size):
        if d.Ro < 2:
            continue
        try:
            plans = [make_plan(d, tokens, clusters=m) for m in models]
        except Refused:
            continue
        p = plans[1]
        for name, pred in CLASSES.items():
            if name not in best and all(pred(d, q) for q in plans):
                best[name] = (d, p)
        if len(best) == len(CLASSES):
            break
    _CENSUS[tokens] = best
    return best


# shapes of the tail-pass and fused-launch tests (tests/test_gpu_gemv_plans.py): v = 8, planned for 4 tokens per pass
TAIL_SHAPES = {
    "nch1": Desc(v=8, K=256, Kr=16, G=1, gs=256, O=264),
    "cluster": Desc(v=8, K=256, Kr=16, G=4, gs=512, O=264),
    "global": Desc(v=8, K=256, Kr=16, G=16, gs=128, O=264),
}
# 2-4 v = 8 layers on one x: (members, does the C side take them in one launch)
FUSED_GROUPS = {
    "nch1_qkv": ([Desc(v=8, K=256, Kr=16, G=1, gs=256, O=o) for o in (2048, 512, 512)], True),
    "cluster_qkv": ([Desc(v=8, K=256, Kr=16, G=1, gs=2048, O=o) for o in (2048, 512, 512)], True),
    "cluster_gate_up": ([Desc(v=8, K=256, Kr=16, G=4, gs=512, O=o) for o in (1024, 264)], True),
    "cluster_four": ([Desc(v=8, K=4096, Kr=-1, G=2, gs=1024, O=o) for o in (2048, 1024, 264, 64)], True),
    "global_refused": ([Desc(v=8, K=256, Kr=16, G=16, gs=128, O=o) for o in (1024, 264)], False),
}


# ------------------------------------------------------------------------------------------------------------------
# the library's own planner, reached without a GPU: vptq_b200_workspace_bytes(OP_GEMV)
# ------------------------------------------------------------------------------------------------------------------
def c_desc(d: Desc):
    """a vptq_linear_desc the C ABI accepts for `d`, with fake (aligned, never dereferenced) pointers"""
    from vptq_b200 import native
    c = native.LinearDesc()
    c.struct_size = ctypes.sizeof(native.LinearDesc)
    c.dtype, c.in_features, c.out_features, c.vector_len = d.dtype, d.I, d.O, d.v
    c.num_centroids, c.num_res_centroids, c.num_codebooks, c.group_size = d.K, d.Kr if d.Kr > 0 else -1, d.G, d.gs
    b = ilog2(d.K) + (ilog2(d.Kr) if d.Kr > 0 else 0)
    c.indices = 0x100000
    c.index_stride_row = (d.gs * b + 31) // 32
    c.index_stride_codebook = d.Ro * c.index_stride_row
    c.centroids, c.centroid_stride = 0x200000, align_up(d.K * d.v, 8)
    if d.Kr > 0:
        c.res_centroids, c.res_centroid_stride = 0x300000, align_up(d.Kr * d.v, 8)
    c.outlier_size, c.outlier_vector_len, c.num_outlier_centroids = d.S, (d.v if d.S else -1), (256 if d.S else -1)
    if d.S:
        c.outlier_indices, c.outlier_centroids = 0x400000, 0x500000
    return c


def library_workspaces(cases):
    """[(Desc, tokens)] -> vptq_b200_workspace_bytes(OP_GEMV) of each, in this process (0: refused, error text)"""
    from vptq_b200 import native
    L = native.lib()
    out = []
    for d, tokens in cases:
        c = c_desc(d)
        ws = int(L.vptq_b200_workspace_bytes(ctypes.byref(c), tokens, native.OP_GEMV))
        out.append((ws, "" if ws else native.last_error()))
    return out


def library_workspaces_without_device(cases):
    """library_workspaces in a child process that sees no CUDA device, so that the library plans for the H100
    geometry it assumes on a CPU-only host (no occupancy query), whatever this machine has"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join(
        [root, os.path.join(root, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "_gemv_plan"]
    payload = json.dumps([[dataclasses.astuple(d), t] for d, t in cases])
    r = subprocess.run(args, input=payload, capture_output=True, text=True, env=env, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return [tuple(x) for x in json.loads(r.stdout)]


if __name__ == "__main__":
    cases = [(Desc(*d), t) for d, t in json.load(sys.stdin)]
    json.dump(library_workspaces(cases), sys.stdout)
