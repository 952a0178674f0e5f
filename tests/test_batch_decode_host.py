"""CPU-side tests of the batched list route (include/vptq_b200_batch.h, csrc/gemv_lists_batch.cu): the header's symbol
table, an integer mirror of the kernel's partition (one combo per CTA, independent of the token count), and the
Python routing with the native entry points stubbed.  The GPU side: test_gpu_batch_decode.py."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SM_COUNT, SMEM_OPTIN = 132, 232448   # H100 SXM
WARPS, STAGE_STEPS, RB, MAX_ROWS, MAX_TOK = 16, 8, 32, 65536, 8


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", src)))


def test_batch_header_declares_exactly_its_exports():
    from vptq_b200 import native
    L = native.lib()
    syms = _declared("vptq_b200_batch.h")
    assert syms == sorted(native.BATCH_EXPORTS)
    for s in syms:
        assert hasattr(L, s), s
    others = set()
    for h in ("vptq_b200.h", "vptq_b200_grad.h", "vptq_b200_graph.h"):
        others |= set(_declared(h))
    assert not set(syms) & others
    assert not set(syms) & (set(native.EXPORTS) | set(native.GRAD_EXPORTS) | set(native.GRAPH_EXPORTS))
    assert len(_declared("vptq_b200.h")) == 15 and native.ABI_VERSION == 7
    assert L.vptq_b200_batch_version() == native.BATCH_VERSION
    assert "vptq_b200_batch.h" in open(os.path.join(ROOT, "include", "vptq_b200.h")).read()


def test_batch_entry_points_refuse_bad_arguments_without_a_launch():
    from vptq_b200 import native
    L = native.lib()
    assert L.vptq_b200_quant_gemv_batch_max_tokens(0, None) == 0
    assert L.vptq_b200_quant_gemv_batch(1, None, None, 0, None, None, 2, None, 0, 0, None) == -1
    assert "NULL" in native.last_error()


# ---------------------------------------------------------------- mirror of batch_partition / the kernel's split
def partition(Ro, Q, P=SM_COUNT):
    """CTAs per combo of each fused layer (csrc/gemv_lists_batch.cu: batch_partition), or None (not eligible)"""
    n, B, rows = len(Ro), P // Q, sum(Ro)
    if n > B or rows * MAX_TOK > MAX_ROWS:
        return None
    k = [min(max(1, B * r // rows), r) for r in Ro]
    used = sum(k)
    while used > B:
        v = -1
        for l in range(n):
            if k[l] > 1 and (v < 0 or k[l] * Ro[v] > k[v] * Ro[l]):
                v = l
        k[v] -= 1
        used -= 1
    while used < B:
        v = -1
        for l in range(n):
            if k[l] < Ro[l] and (v < 0 or Ro[l] * k[v] > Ro[v] * k[l]):
                v = l
        if v < 0:
            break
        k[v] += 1
        used += 1
    return k


def kernel_split(Ro, Q, firsts, tokens):
    """Everything a launch of `tokens` tokens is cut into: per CTA (layer, combo, rows [r0, r1), the 16 warps' step
    runs).  `tokens` picks the instance (2, 4 or 8) and nothing else."""
    ntok = 2 if tokens <= 2 else 4 if tokens <= 4 else 8
    assert 1 <= tokens <= ntok
    k = partition(Ro, Q)
    ctas = []
    for l, (ro, kl) in enumerate(zip(Ro, k)):
        first = firsts[l]
        for q in range(kl * Q):
            combo, j = divmod(q, kl)
            r0, r1 = ro * j // kl, ro * (j + 1) // kl
            T0, T1 = first[combo * ro + r0], first[combo * ro + r1]
            runs = [(T0 + (T1 - T0) * w // WARPS, T0 + (T1 - T0) * (w + 1) // WARPS) for w in range(WARPS)]
            ctas.append((l, combo, r0, r1, tuple(runs)))
    return ctas


def carve(TCW, max_nun, max_kr, ntok, limit=SMEM_OPTIN, stages_tried=(3, 2)):
    """shared-memory bytes of instance ntok (batch_carve), 0: nothing fits"""
    al = lambda v: (v + 127) // 128 * 128
    for stages in stages_tried:
        off = al((1 + WARPS * stages) * 8) + al((max_nun + 1) * 4) + al((WARPS + 1) * MAX_TOK * 4 + 16)
        off += al(WARPS * 2 * ntok * 32 + WARPS * 2 * 4) + al((max_nun // RB + 2) * 4) + 65536
        off += al(max_kr * 16 * 8) + al(TCW * ntok * 2) + WARPS * stages * STAGE_STEPS * 128
        if off <= limit:
            return off
    return 0


def _q(I, K=65536):
    from vptq_b200 import lists
    ns, nt, tcw = lists.geometry(I, K)
    return ns * nt, tcw


# Llama-3 8B / 70B decoder linears as fused for decode: (in_features, [out_features of the fused members])
FUSED_SETS = {
    "8b_qkv": (4096, [4096, 1024, 1024]), "8b_o": (4096, [4096]), "8b_gate_up": (4096, [14336, 14336]),
    "8b_down": (14336, [4096]), "70b_qkv": (8192, [8192, 1024, 1024]), "70b_o": (8192, [8192]),
    "70b_gate_up": (8192, [28672, 28672]), "70b_down": (28672, [8192]),
}


@pytest.mark.parametrize("name", sorted(FUSED_SETS))
def test_partition_covers_every_unit_once_inside_one_combo(name):
    I, outs = FUSED_SETS[name]
    Q, TCW = _q(I)
    Ro = [(o + 7) // 8 for o in outs]
    k = partition(Ro, Q)
    assert k is not None and all(1 <= kl <= ro for kl, ro in zip(k, Ro))
    assert sum(k) * Q <= SM_COUNT and sum(k) == SM_COUNT // Q or all(kl == ro for kl, ro in zip(k, Ro))
    rng = np.random.default_rng(len(name))
    firsts = []
    for ro in Ro:   # list lengths: 1..12 steps per unit, skewed
        steps = 1 + rng.zipf(2.0, size=Q * ro).clip(max=11)
        firsts.append(np.concatenate([[0], np.cumsum(steps)]).tolist())
    ctas = kernel_split(Ro, Q, firsts, 8)
    seen = [np.zeros(Q * ro, np.int32) for ro in Ro]
    for l, combo, r0, r1, runs in ctas:
        assert 0 <= combo < Q and 0 <= r0 < r1 <= Ro[l]
        seen[l][combo * Ro[l] + r0:combo * Ro[l] + r1] += 1        # its units lie inside one combo
        first = firsts[l]
        assert runs[0][0] == first[combo * Ro[l] + r0] and runs[-1][1] == first[combo * Ro[l] + r1]
        assert all(a[1] == b[0] for a, b in zip(runs[:-1], runs[1:]))
    for s in seen:
        assert (s == 1).all()
    max_nun = max((ro + kl - 1) // kl for ro, kl in zip(Ro, k))
    for ntok in (2, 4, 8):
        assert carve(TCW, max_nun, 256, ntok) > 0, ntok
    # the one-combo partition leaves SM_COUNT mod Q SMs idle (and more where k hits Ro)
    assert len(ctas) == sum(k) * Q


@pytest.mark.parametrize("name", sorted(FUSED_SETS))
def test_partition_is_the_same_for_every_token_count(name):
    I, outs = FUSED_SETS[name]
    Q, _ = _q(I)
    Ro = [(o + 7) // 8 for o in outs]
    rng = np.random.default_rng(3)
    firsts = [np.concatenate([[0], np.cumsum(1 + rng.integers(0, 9, size=Q * ro))]).tolist() for ro in Ro]
    ref = kernel_split(Ro, Q, firsts, 1)
    for tokens in range(2, 9):
        assert kernel_split(Ro, Q, firsts, tokens) == ref, tokens


def test_eligibility_limits():
    assert partition([8193], 32) is None                      # rows x 8 tokens past 65536
    assert partition([28672 // 8] * 2, 32) == [2, 2]          # 70B gate + up: 57344 row-tokens, 4 combo copies
    assert partition([512, 512], 132) is None                 # n * Q > SM count
    assert partition([512], 132) == [1]
    assert partition([4096 // 8, 128, 128], 16) == [5, 2, 1]  # 8B q/k/v: 128 of 132 SMs


def _plan(I, outs, K=65536, Kr=256):
    """(Q, k, the carve of NTOK = 2, 4, 8, the same with 3 ring stages only) of a fused set, as the kernel plans it"""
    from vptq_b200 import lists
    ns, nt, tcw = lists.geometry(I, K)
    Q, Ro = ns * nt, [(o + 7) // 8 for o in outs]
    k = partition(Ro, Q)
    if k is None:
        return Q, None, None, None
    mn = max((r + kl - 1) // kl for r, kl in zip(Ro, k))
    return (Q, k, [carve(tcw, mn, Kr, n) for n in (2, 4, 8)],
            [carve(tcw, mn, Kr, n, stages_tried=(3,)) for n in (2, 4, 8)])


# the cut-off shapes of tests/test_gpu_batch_envelope.py, each on its intended side
def test_cutoff_ring_stages():
    """I = 12288, two 20480-output layers: NTOK = 8 needs the 2-stage ring, NTOK = 2 and 4 keep 3 stages; the 70B
    gate+up pair keeps 3 stages at NTOK = 8 (2432 bytes to spare)"""
    Q, k, both, three = _plan(12288, [20480, 20480])
    assert Q == 48 and k == [1, 1]
    assert three[0] == both[0] > 0 and three[1] == both[1] > 0
    assert three[2] == 0 and both[2] == 216704
    Q, k, both, three = _plan(8192, [28672, 28672])
    assert Q == 32 and k == [2, 2] and three == both and SMEM_OPTIN - both[2] == 2432


def test_cutoff_last_layout_that_fits():
    """I = 20480 (Q = 80), Kr = 256: out = 51192 fits with 0 bytes to spare, out = 51200 does not fit"""
    Q, k, both, _ = _plan(20480, [51192])
    assert Q == 80 and k == [1] and both[2] == SMEM_OPTIN
    Q, k, both, _ = _plan(20480, [51200])
    assert both[2] == 0 and both[0] > 0 and both[1] > 0      # batch_max_tokens asks for NTOK = 8: 0


def test_cutoff_workspace_rows():
    """sum Ro x 8 = 65536 accepted (one layer, and 4 fused layers), 65544 refused"""
    assert _plan(4096, [65536])[1] == [8]
    assert _plan(4096, [16384] * 4)[1] == [2, 2, 2, 2]
    assert _plan(4096, [65544])[1] is None
    assert partition([65536 // 8], 16) is not None and partition([65544 // 8], 16) is None


def test_cutoff_partition_regimes():
    """n = B; n > B (three layers at I = 12288); B = 1 (Q = 128); k = Ro; Ro = 1; ragged multi-tile widths"""
    assert _plan(14336, [4096, 4096])[:2] == (64, [1, 1])
    assert SM_COUNT // 48 == 2 and _plan(12288, [4096, 1024, 1024])[1] is None
    assert all(_plan(12288, [o])[1] is not None for o in (4096, 1024))
    assert _plan(32768, [4096])[:2] == (128, [1])
    assert _plan(1024, [264], K=8192)[:2] == (2, [33])
    assert _plan(1024, [8])[:2] == (16, [1])
    from vptq_b200 import lists
    assert lists.geometry(4100, 65536) == (16, 2, 2056) and 4100 - 2056 == 2044
    assert lists.geometry(9004, 65536) == (16, 3, 3008) and 9004 % 8 != 0
    # a valid codebook is a power of two (NS in {2, 4, 8, 16}) and NT <= 16: NS x NT never equals 132
    assert not [(ns, nt) for ns in (2, 4, 8, 16) for nt in range(1, 17) if ns * nt == SM_COUNT]
    for I, outs in FUSED_SETS.values():                       # every full-size set also fits at NTOK = 8
        assert _plan(I, outs)[2][2] > 0


# ---------------------------------------------------------------- python routing with native stubbed
class _Desc:
    def __init__(self, lists=True):
        self.lists_stream = 1 if lists else 0


def _stub(monkeypatch, max_tokens=8):
    from vptq_b200 import native
    calls = []
    monkeypatch.setattr(native, "quant_gemv", lambda d, x, y, flags=0: calls.append(("gemv", x.shape[0])))
    monkeypatch.setattr(native, "quant_gemm", lambda d, x, y, flags=0: calls.append(("gemm", x.shape[0])))
    monkeypatch.setattr(native, "quant_gemv_batch", lambda d, x, y, flags=0: calls.append(("batch", x.shape[0])))

    def bmt(d):
        calls.append(("max", None))
        return max_tokens
    monkeypatch.setattr(native, "batch_max_tokens", bmt)
    return calls


def _aligned(tokens, I=64):
    buf = torch.zeros(tokens * I + 16, dtype=torch.float16)
    off = (-buf.data_ptr() % 16) // 2
    return buf[off:off + tokens * I].view(tokens, I)


def test_opted_out_calls_never_reach_the_batched_entry_points(monkeypatch):
    from vptq_b200 import ops
    calls = _stub(monkeypatch)
    for tokens in range(1, 12):
        ops._forward(_Desc(), _aligned(tokens), 32)
        ops._forward(_Desc(), _aligned(tokens), 32, False)
    assert calls and all(c[0] in ("gemv", "gemm") for c in calls)
    assert [c for c in calls if c[0] == "gemv"] == [("gemv", t) for t in (1, 1, 2, 2)]


def test_opted_in_routing(monkeypatch):
    from vptq_b200 import ops
    calls = _stub(monkeypatch)
    route = {}
    for tokens in range(1, 12):
        calls.clear()
        ops._forward(_Desc(), _aligned(tokens), 32, True)
        route[tokens] = [c[0] for c in calls if c[0] != "max"]
    assert route == {1: ["gemv"], **{t: ["batch"] for t in range(2, 9)}, 9: ["gemm"], 10: ["gemm"], 11: ["gemm"]}
    calls.clear()
    ops._forward(_Desc(lists=False), _aligned(4), 32, True)       # no index lists: as without the opt-in
    assert calls == [("gemm", 4)]
    calls = _stub(monkeypatch, max_tokens=0)                      # not eligible
    ops._forward(_Desc(), _aligned(2), 32, True)
    assert [c for c in calls if c[0] != "max"] == [("gemv", 2)]


def test_module_passes_the_flag(monkeypatch):
    from vptq_b200 import VQuantLinear, ops
    seen = []
    monkeypatch.setattr(ops, "quant_gemm", lambda x, **kw: seen.append(kw["_batched_decode"]))
    m = VQuantLinear(64, 32, vector_lens=[-1, 8], num_centroids=[-1, 256], num_res_centroids=[-1, -1], group_num=1,
                     group_size=64, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                     dtype=torch.float16, enable_proxy_error=False)
    x = torch.zeros(4, 64, dtype=torch.float16)
    m(x)
    assert m.set_batched_decode(True) is m
    m(x)
    m.set_batched_decode(False)
    m(x)
    assert seen == [False, True, False]


def test_set_batched_decode_reaches_fused_members():
    import vptq_b200
    from vptq_b200 import VQuantLinear
    from vptq_b200.fuse import FusedGroup, FusedMember

    def lin():
        return VQuantLinear(64, 32, vector_lens=[-1, 8], num_centroids=[-1, 256], num_res_centroids=[-1, -1],
                            group_num=1, group_size=64, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                            dtype=torch.float16, enable_proxy_error=False)
    a, b, c = lin(), lin(), lin()
    g = FusedGroup([a, b])
    model = torch.nn.Sequential(FusedMember(a, g, 0), FusedMember(b, g, 1), c)
    assert vptq_b200.set_batched_decode(model) == 3
    assert a._batched_decode and b._batched_decode and c._batched_decode
    assert vptq_b200.set_batched_decode(model, False) == 3
    assert not (a._batched_decode or b._batched_decode or c._batched_decode)
