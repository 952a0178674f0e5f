"""CPU-side tests of the vector-length-16 list route (include/vptq_b200_lists16.h, csrc/gemv_lists16.cu): the v = 16
lists against the oracle, the C host builder against the torch builder, dealing, the header's symbol table, refusals
before any launch, an integer mirror of the kernel's partition, shared-memory carve and token limit, and the Python
routing with the native entry points stubbed.  The GPU side: test_gpu_lists16.py."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import vptq_oracle as vo
from vptq_b200 import lists

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SM_COUNT, SMEM_OPTIN = 132, 232448   # H100 SXM
WARPS, STAGE_STEPS, RB, MAX_ROW_TOKENS, MAX_TOK, V = 16, 8, 32, 32768, 4, 16

CASES = [
    dict(I=1024, O=264, K=65536, Kr=256),   # v16-k65536-256, small, ragged last index row
    dict(I=512, O=64, K=16384, Kr=16),
    dict(I=768, O=40, K=32768, Kr=-1),
    dict(I=9000, O=48, K=8192, Kr=256),     # three column tiles
    dict(I=1004, O=100, K=65536, Kr=2),     # in_features not a multiple of 8
]


def _layer(c, perm=True, seed=11):
    return vo.make_layer(c["I"], c["O"], vector_len=16, num_centroids=c["K"], num_res_centroids=c["Kr"], dtype="fp16",
                         seed=seed, enable_perm=perm)


def _perm_t(L):
    return None if L.perm is None else torch.from_numpy(np.asarray(L.perm).astype(np.uint16).astype(np.int64))


def _build(L, c, deal=None):
    return lists.build_lists(torch.from_numpy(np.ascontiguousarray(L.indices)), num_centroids=c["K"],
                             num_res_centroids=c["Kr"], in_features=c["I"], out_features=c["O"], perm=_perm_t(L),
                             deal=deal, vector_len=16)


def _eval(L, c, stream, tab, x):
    xf = vo.to_f32(x, "fp16").astype(np.float64).reshape(-1)
    sc = vo.to_f32(L.weight_scale, "fp16").astype(np.float64)
    wb = vo.to_f32(L.weight_bias, "fp16").astype(np.float64)
    C = torch.from_numpy(vo.to_f32(L.centroids, "fp16"))
    R = None if c["Kr"] <= 0 else torch.from_numpy(vo.to_f32(L.res_centroids, "fp16"))
    y = lists.emulate(stream, tab, num_centroids=c["K"], num_res_centroids=c["Kr"], in_features=c["I"],
                      out_features=c["O"], centroids=C, res_centroids=R, xs=torch.from_numpy(xf * sc),
                      vector_len=16).numpy()
    return y[:c["O"]] + float((xf * wb).sum())


@pytest.mark.parametrize("c", CASES)
@pytest.mark.parametrize("perm", [True, False])
def test_v16_lists_reproduce_the_oracle(c, perm):
    L = _layer(c, perm)
    stream, tab, tcw = _build(L, c)
    NS, NT, TCW = lists.geometry(c["I"], c["K"])
    assert tcw == TCW and tab.shape[0] == NS * NT * ((c["O"] + 15) // 16) + 1
    x = vo.make_x(1, c["I"], "fp16")
    y_star = vo.quant_gemm(x, L).astype(np.float64).reshape(-1)
    assert np.max(np.abs(_eval(L, c, stream, tab, x) - y_star)) <= 1e-5 * max(1.0, np.max(np.abs(y_star)))


def test_v8_default_is_unchanged_and_other_lengths_are_refused():
    L = vo.make_layer(512, 64, vector_len=8, num_centroids=8192, num_res_centroids=4, seed=3)
    ind = torch.from_numpy(np.ascontiguousarray(L.indices))
    kw = dict(num_centroids=8192, num_res_centroids=4, in_features=512, out_features=64, perm=_perm_t(L), deal=True)
    a, b = lists.build_lists(ind, **kw), lists.build_lists(ind, vector_len=8, **kw)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]
    with pytest.raises(ValueError):
        lists.build_lists(ind, vector_len=12, **kw)
    base = dict(num_centroids=65536, num_res_centroids=256, num_codebooks=1, outlier_size=0, in_features=8192)
    assert lists.eligible(vector_len=8, **base) and not lists.eligible(vector_len=16, **base)
    assert lists.eligible(vector_len=16, list_vector_len=16, **base)
    assert not lists.eligible(vector_len=8, list_vector_len=16, **base)
    for bad in (dict(num_res_centroids=512), dict(num_centroids=4096), dict(num_codebooks=2), dict(outlier_size=64)):
        assert not lists.eligible(vector_len=16, list_vector_len=16, **{**base, **bad}), bad


def _c_build(L, c, perm=True):
    from vptq_b200 import native
    lib = native.lib()
    ind = np.ascontiguousarray(L.indices[0])
    NS, NT, _ = lists.geometry(c["I"], c["K"])
    tab_c = np.zeros(NS * NT * ((c["O"] + 15) // 16) + 1, dtype=np.uint32)
    steps, tcw = ctypes.c_size_t(0), ctypes.c_int32(0)
    pp = np.ascontiguousarray(np.asarray(L.perm).astype(np.uint16)) if (perm and L.perm is not None) else None
    args = (ind.ctypes.data, ind.shape[1], c["O"], c["I"], c["K"], c["Kr"], None if pp is None else pp.ctypes.data)
    assert lib.vptq_b200_lists16_build_host(*args, None, 0, tab_c.ctypes.data, ctypes.byref(steps),
                                            ctypes.byref(tcw)) == 0, native.last_error()
    out = np.zeros(steps.value * 32, dtype=np.uint32)
    assert lib.vptq_b200_lists16_build_host(*args, out.ctypes.data, out.nbytes, tab_c.ctypes.data, ctypes.byref(steps),
                                            ctypes.byref(tcw)) == 0, native.last_error()
    assert lib.vptq_b200_lists_deal_host(out.ctypes.data, tab_c.ctypes.data, len(tab_c) - 1, 0) == 0
    return out, tab_c, steps.value, tcw.value, (args, ind, pp)


def test_c_host_builder_is_byte_identical_fuzzed():
    """vptq_b200_lists16_build_host + vptq_b200_lists_deal_host == the torch builder, and the lists still evaluate to
    the oracle's sums"""
    from vptq_b200 import native
    rng = np.random.default_rng(4242)
    for trial in range(14):
        c = dict(K=int(rng.choice([8192, 16384, 32768, 65536])), Kr=int(rng.choice([-1, 2, 64, 256])),
                 I=int(rng.integers(33, 700)), O=int(rng.integers(1, 120)))
        perm = bool(trial % 3)
        L = _layer(c, perm, seed=200 + trial)
        stream, tab, tcw = _build(L, c)
        out, tab_c, steps, tcw_c, (args, *_keep) = _c_build(L, c, perm)
        assert steps == stream.shape[0] and tcw_c == tcw, c
        assert np.array_equal(tab_c.astype(np.int64), tab.numpy().astype(np.int64) & 0xFFFFFFFF), c
        assert np.array_equal(out, stream.numpy().reshape(-1).view(np.uint32)), c
        x = vo.make_x(1, c["I"], "fp16", seed=trial)
        y_star = vo.quant_gemm(x, L).astype(np.float64).reshape(-1)
        assert np.max(np.abs(_eval(L, c, stream, tab, x) - y_star)) <= 1e-5 * max(1.0, np.max(np.abs(y_star))), c
    st, tc = ctypes.c_size_t(0), ctypes.c_int32(0)        # too small a buffer is refused, not overrun
    assert native.lib().vptq_b200_lists16_build_host(*args, out.ctypes.data, 16, tab_c.ctypes.data, ctypes.byref(st),
                                                     ctypes.byref(tc)) == -3


def test_host_builder_rejects_what_the_kernel_does_not_cover():
    from vptq_b200 import native
    lib = native.lib()
    ind = np.zeros((4, 64), dtype=np.int32)
    tab = np.zeros(64, dtype=np.uint32)
    st, tc = ctypes.c_size_t(0), ctypes.c_int32(0)
    for K, Kr in ((4096, -1), (65536, 512), (12288, -1)):
        assert lib.vptq_b200_lists16_build_host(ind.ctypes.data, 64, 32, 64, K, Kr, None, None, 0, tab.ctypes.data,
                                                ctypes.byref(st), ctypes.byref(tc)) == -2, (K, Kr)
    assert lib.vptq_b200_lists16_build_host(None, 64, 32, 64, 65536, 256, None, None, 0, tab.ctypes.data,
                                            ctypes.byref(st), ctypes.byref(tc)) == -1


@pytest.mark.parametrize("c", CASES[:3])
def test_dealing_only_reorders_inside_lists(c):
    L = _layer(c)
    raw, tab, _ = _build(L, c, deal=False)
    dealt, tab2, _ = _build(L, c, deal=True)
    assert torch.equal(tab, tab2)
    r, d = raw.numpy().reshape(-1).view(np.uint32), dealt.numpy().reshape(-1).view(np.uint32)
    t = tab.numpy().astype(np.int64) & 0xFFFFFFFF
    first, end, tail = t[:-1] & lists.STEP_MASK, t[1:] & lists.STEP_MASK, t[:-1] >> 26
    a, b, e = first * 32, (end - 1) * 32 + tail, end * 32
    for u in range(len(a)):
        assert np.array_equal(np.sort(r[a[u]:b[u]]), np.sort(d[a[u]:b[u]])), u
        assert not d[b[u]:e[u]].any(), u


# ---------------------------------------------------------------- the header
def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", src)))


def test_header_declares_exactly_its_exports():
    from vptq_b200 import native
    L = native.lib()
    syms = _declared("vptq_b200_lists16.h")
    assert syms == sorted(native.LISTS16_EXPORTS)
    for s in syms:
        assert hasattr(L, s), s
    others = set()
    for h in ("vptq_b200.h", "vptq_b200_grad.h", "vptq_b200_graph.h", "vptq_b200_batch.h", "vptq_b200_lists_dense.h"):
        others |= set(_declared(h))
    assert not set(syms) & others
    assert len(_declared("vptq_b200.h")) == 15 and native.ABI_VERSION == 7 and L.vptq_b200_abi_version() == 7
    assert L.vptq_b200_lists16_version() == native.LISTS16_VERSION
    assert "vptq_b200_lists16.h" in open(os.path.join(ROOT, "include", "vptq_b200.h")).read()
    src = open(os.path.join(ROOT, "include", "vptq_b200_lists16.h")).read()
    m = re.search(r"#define VPTQ_B200_LISTS16_WORKSPACE_BYTES \(\(size_t\)(\d+) \* (\d+) \+ \(size_t\)(\d+) \* (\d+)\)", src)
    assert m and int(m[1]) * int(m[2]) + int(m[3]) * int(m[4]) == native.LISTS16_WORKSPACE_BYTES


def test_entry_points_refuse_bad_arguments_without_a_launch():
    from vptq_b200 import native
    L = native.lib()
    assert L.vptq_b200_quant_gemv_lists16_max_tokens(0, None) == 0
    assert L.vptq_b200_quant_gemv_lists16_max_tokens(5, None) == 0
    assert L.vptq_b200_quant_gemv_lists16(1, None, None, 0, None, None, 2, None, 0, 0, None) == -1
    assert "NULL" in native.last_error()
    # unknown flags are refused before any descriptor or device is looked at
    d = native.LinearDesc()
    arr = native._desc_array([d])
    y = (ctypes.c_void_p * 1)(16)
    s = (ctypes.c_int64 * 1)(64)
    assert L.vptq_b200_quant_gemv_lists16(1, arr, 16, 64, y, s, 1, 16, 1 << 30, 4, None) == -1
    assert "flags" in native.last_error()
    assert L.vptq_b200_quant_gemv_lists16(1, arr, 16, 64, y, s, 1, 16, 1 << 30, 0, None) == -1   # struct_size 0
    assert L.vptq_b200_quant_gemv_lists16_max_tokens(1, arr) == 0


# ---------------------------------------------------------------- mirror of lists16_partition / carve / max tokens
def partition(Ro, Q, P=SM_COUNT):
    """CTAs per combo of each fused layer (csrc/gemv_lists16.cu: lists16_partition), or None (not eligible)"""
    n, B, rows = len(Ro), P // Q, sum(Ro)
    if n > B or rows > MAX_ROW_TOKENS:
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


def carve(TCW, max_nun, max_kr, ntok, limit=SMEM_OPTIN):
    """(shared-memory bytes, residual replication, ring stages) of instance ntok (lists16_carve); (0, 0, 0): no fit"""
    al = lambda v: (v + 127) // 128 * 128
    for rep in (8, 4, 2, 1):
        for stages in (3, 2):
            off = al(WARPS * stages * 8) + al((max_nun + 1) * 4) + al((WARPS + 1) * MAX_TOK * 4 + 16)
            off += al(WARPS * 2 * ntok * V * 4 + WARPS * 2 * 4) + al((max_nun // RB + 2) * 4) + 2 * 65536
            off += 2 * al(max_kr * 16 * rep) + al(TCW * ntok * 2) + WARPS * stages * STAGE_STEPS * 128
            if off <= limit:
                return off, rep, stages
    return 0, 0, 0


def max_tokens(I, outs, K=65536, Kr=256):
    """the largest instance (4, 2, 1) whose rows x tokens fit the accumulators and whose layout fits; 0: none"""
    ns, nt, tcw = lists.geometry(I, K)
    Q, Ro = ns * nt, [(o + 15) // 16 for o in outs]
    k = partition(Ro, Q)
    if k is None:
        return 0
    mn = max((r + kl - 1) // kl for r, kl in zip(Ro, k))
    for ntok in (4, 2, 1):
        if sum(Ro) * ntok <= MAX_ROW_TOKENS and carve(tcw, mn, Kr, ntok)[0]:
            return ntok
    return 0


def kernel_split(Ro, Q, firsts):
    """per CTA (layer, combo, rows [r0, r1), the 16 warps' step runs); no token count enters it"""
    k = partition(Ro, Q)
    ctas = []
    for l, (ro, kl) in enumerate(zip(Ro, k)):
        first = firsts[l]
        for q in range(kl * Q):
            combo, j = divmod(q, kl)
            r0, r1 = ro * j // kl, ro * (j + 1) // kl
            T0, T1 = first[combo * ro + r0], first[combo * ro + r1]
            ctas.append((l, combo, r0, r1, tuple((T0 + (T1 - T0) * w // WARPS, T0 + (T1 - T0) * (w + 1) // WARPS)
                                                 for w in range(WARPS))))
    return ctas


# Llama-3-70B (= Nemotron-70B), Mistral-Large-123B and Llama-3.1-405B linears as fused for decode
SETS = {
    "70b_qkv": (8192, [8192, 1024, 1024]), "70b_o": (8192, [8192]), "70b_gate_up": (8192, [28672, 28672]),
    "70b_down": (28672, [8192]), "mistral_q": (12288, [12288]), "mistral_kv": (12288, [1024, 1024]),
    "mistral_o": (12288, [12288]), "mistral_gate_up": (12288, [28672, 28672]), "mistral_down": (28672, [12288]),
    "405b_q": (16384, [16384]), "405b_kv": (16384, [1024, 1024]), "405b_o": (16384, [16384]),
    "405b_gate_up": (16384, [53248, 53248]),
}


@pytest.mark.parametrize("name", sorted(SETS))
def test_partition_covers_every_unit_once_and_four_tokens_fit(name):
    I, outs = SETS[name]
    ns, nt, _ = lists.geometry(I, 65536)
    Q, Ro = ns * nt, [(o + 15) // 16 for o in outs]
    k = partition(Ro, Q)
    assert k is not None and all(1 <= kl <= ro for kl, ro in zip(k, Ro))
    assert sum(k) * Q <= SM_COUNT
    rng = np.random.default_rng(len(name))
    firsts = [np.concatenate([[0], np.cumsum(1 + rng.zipf(2.0, size=Q * ro).clip(max=11))]).tolist() for ro in Ro]
    seen = [np.zeros(Q * ro, np.int32) for ro in Ro]
    for l, combo, r0, r1, runs in kernel_split(Ro, Q, firsts):
        seen[l][combo * Ro[l] + r0:combo * Ro[l] + r1] += 1
        assert runs[0][0] == firsts[l][combo * Ro[l] + r0] and runs[-1][1] == firsts[l][combo * Ro[l] + r1]
        assert all(a[1] == b[0] for a, b in zip(runs[:-1], runs[1:]))
    assert all((s == 1).all() for s in seen)
    assert max_tokens(I, outs) == 4


def test_limits_and_the_max_tokens_rule():
    # 405B gate + up fused: 6656 index rows; 4 tokens use 26624 of the 32768 row-token accumulators, 8 would not fit
    assert partition([3328, 3328], 64) == [1, 1] and 6656 * 4 <= MAX_ROW_TOKENS < 6656 * 8
    # the residual table's replication shrinks as the x' tile grows; NTOK = 4 needs the 2-stage ring at TCW = 4096
    assert carve(4096, 256, 256, 1)[1:] == (4, 3) and carve(4096, 256, 256, 2)[1:] == (4, 2)
    assert carve(4096, 256, 256, 4)[1:] == (2, 2)
    assert carve(4096, 256, 0, 4)[1:] == (8, 3)                     # (no residual table)
    assert carve(4096, 3328, 256, 4)[1:] == (1, 2)                  # 405B gate / up: the table costs 13 KiB
    # the token count falls back 4 -> 2 -> 1 on the row-token limit
    assert max_tokens(4096, [131072]) == 4 and max_tokens(4096, [262144]) == 2 and max_tokens(4096, [524288]) == 1
    assert max_tokens(4096, [524304]) == 0
    # not eligible: more combos than SMs (405B down), too many layers for the combo copies (405B and Mistral q/k/v)
    assert max_tokens(53248, [16384]) == 0
    assert max_tokens(16384, [16384, 1024, 1024]) == 0 and max_tokens(12288, [12288, 1024, 1024]) == 0
    assert not lists.launchable(53248, 65536, SM_COUNT) and lists.launchable(28672, 65536, SM_COUNT)


def _plan(I, outs, Kr=256):
    """(carve of each instance 1, 2, 4, max_tokens) of the fused layers `outs` at in_features I"""
    ns, nt, tcw = lists.geometry(I, 65536)
    Ro = [(o + 15) // 16 for o in outs]
    k = partition(Ro, ns * nt)
    mn = max((r + kl - 1) // kl for r, kl in zip(Ro, k))
    return {n: carve(tcw, mn, Kr, n) for n in (1, 2, 4)}, max_tokens(I, outs, Kr=Kr)


def test_cut_off_shapes_of_the_gpu_envelope():
    """every shape tests/test_gpu_lists16_envelope.py runs at a cut-off (tests/_lists16.py), on its side of it"""
    import _lists16 as l16
    assert (SM_COUNT, SMEM_OPTIN) == (l16.SM_COUNT, l16.SMEM_OPTIN)
    # one shape per (replication, stages) the carve chooses, at the instance of its token count
    for (rep, stages), (I, O, Kr, tokens) in l16.CARVE.items():
        c, mt = _plan(I, [O], Kr)
        assert c[4 if tokens > 2 else tokens][1:] == (rep, stages) and mt == 4, (rep, stages)
    assert _plan(4096, [1024], 0)[0] == {1: (191616, 8, 3), 2: (201856, 8, 3), 4: (222336, 8, 3)}
    assert _plan(4096, [1024], 64)[0][4] == (222208, 8, 2)
    assert _plan(4096, [1024])[0] == {1: (224384, 4, 3), 2: (218112, 4, 2), 4: (222208, 2, 2)}
    # the carve never chooses 3 stages below replication 4 for Kr <= 256 (dropping a stage frees at least as much)
    for Kr in (0, 2, 64, 128, 256):
        for tcw in (1024, 2056, 3008, 4096):
            for mn in (1, 8, 257, 1024, 3328, 4511, 4512, 8192):
                for ntok in (1, 2, 4):
                    assert carve(tcw, mn, Kr, ntok)[1:] not in ((2, 3), (1, 3))
    # the exact fit: I = 32768 (Q = 128, B = 1), out = 72176 fills the opt-in at NTOK = 4 with replication 1;
    # one index row more (72192) does not fit at 4 tokens and takes 2 (replication 2 there)
    assert partition([l16.EXACT_FIT[1] // 16], 128) == [1] and lists.geometry(32768, 65536)[:2] == (16, 8)
    c, mt = _plan(*l16.EXACT_FIT[:1], [l16.EXACT_FIT[1]])
    assert c[4] == (232448, 1, 2) and mt == 4
    assert carve(4096, 4511, 256, 4, limit=SMEM_OPTIN - 1) == (0, 0, 0)
    c, mt = _plan(*l16.PAST_FIT[:1], [l16.PAST_FIT[1]])
    assert c[4] == (0, 0, 0) and c[2] == (220288, 2, 2) and mt == 2
    assert carve(4096, 4512, 256, 4, limit=SMEM_OPTIN + 128) == (SMEM_OPTIN + 128, 1, 2)
    # the row-token limit at I = 4096 (Q = 16, B = 8): 32768 [row][token] accumulators of 16 outputs
    for O, want in l16.ROW_TOKENS.items():
        assert max_tokens(4096, [O]) == want, O
        rows = (O + 15) // 16
        assert rows * want <= MAX_ROW_TOKENS and (want == 4 or rows * max(2 * want, 1) > MAX_ROW_TOKENS), O
    assert (524288 // 16) * 1 == MAX_ROW_TOKENS                     # 1 token: the head exactly full
    assert _plan(4096, [524288])[0][1][0] > 0                        # (the 1-token layout fits)
    # the fused 405B q/k/v: three layers, B = 2; each member alone takes 4 tokens
    I, outs = l16.QKV_405B
    assert lists.geometry(I, 65536)[:2] == (16, 4) and partition([o // 16 for o in outs], 64) is None
    assert max_tokens(I, outs) == 0 and all(max_tokens(I, [o]) == 4 for o in outs)
    # partition extremes: B = 1 at I = 32768; one row per CTA at I = 4096, out = 128; Ro = 1
    assert partition([256], 128) == [1] and partition([8], 16) == [8] and partition([1], 16) == [1]
    runs = kernel_split([8], 16, [[s for s in range(0, 16 * 8 + 1)]])         # (1-step units: 15 warps idle)
    assert all(sum(b > a for a, b in w) == 1 for *_, w in runs)
    runs = kernel_split([8], 16, [[0] + [128 * (i + 1) for i in range(16 * 8)]])   # 128-step units: all 16 busy
    assert all(all(b - a == 8 for a, b in w) for *_, w in runs)


def test_partition_does_not_depend_on_the_token_count():
    """the kernel's split takes no token argument at all: the mirror above has none, and neither has
    lists16_partition (only the shared-memory carve and the accumulator offsets see the instance)"""
    src = open(os.path.join(ROOT, "vptq_b200", "csrc", "gemv_lists16.cu")).read()
    sig = re.search(r"int lists16_partition\(([^)]*)\)", src)[1]
    assert "tok" not in sig and "ntok" not in src[src.index("int lists16_partition("):src.index("size_t lists16_carve(")]


# ---------------------------------------------------------------- python routing with native stubbed
def _lin(v=16, I=64):
    from vptq_b200 import VQuantLinear
    return VQuantLinear(I, 32, vector_lens=[-1, v], num_centroids=[-1, 256], num_res_centroids=[-1, -1], group_num=1,
                        group_size=I, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                        dtype=torch.float16, enable_proxy_error=False)


def test_module_passes_the_list_decode_opt_in_and_drops_a_descriptor_without_lists(monkeypatch):
    from vptq_b200 import ops
    seen = []
    monkeypatch.setattr(ops, "quant_gemm", lambda x, **kw: seen.append(kw["_opt_ins"].list_decode))
    m = _lin()
    x = torch.zeros(2, 64, dtype=torch.float16)
    m(x)
    assert m.set_list_decode(True) is m
    m(x)
    m.set_list_decode(False)
    m(x)
    assert seen == [False, True, False]

    class _D:
        lists_stream = 0
    for v, dropped in ((16, True), (8, False)):
        m = _lin(v)
        m._desc_cache, m._desc_key = [_D(), None], ("key",)
        m.set_list_decode(True)
        assert (m._desc_cache == []) == dropped and (m._desc_key is None) == dropped, v


def test_set_list_decode_reaches_every_fused_member_and_fuse_takes_v16_groups():
    import vptq_b200
    from vptq_b200.fuse import FusedGroup, FusedMember, _eligible
    a, b, c = _lin(), _lin(), _lin()
    g = FusedGroup([a, b])
    model = torch.nn.Sequential(FusedMember(a, g, 0), FusedMember(b, g, 1), c)
    assert vptq_b200.set_list_decode(model) == 3
    assert a._opt_ins.list_decode and b._opt_ins.list_decode and c._opt_ins.list_decode
    assert vptq_b200.set_list_decode(model, False) == 3
    assert not (a._opt_ins.list_decode or b._opt_ins.list_decode or c._opt_ins.list_decode)
    assert _eligible([_lin(16), _lin(16)]) and _eligible([_lin(8), _lin(8)])
    assert not _eligible([_lin(16), _lin(8)]) and not _eligible([_lin(4), _lin(4)])


def test_v16_group_without_the_opt_in_is_never_fused(monkeypatch):
    from vptq_b200 import native
    from vptq_b200.fuse import FusedGroup
    g = FusedGroup([_lin(), _lin()])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(native, "lists16_max_tokens", lambda d: pytest.fail("queried without the opt-in"))
    with torch.no_grad():
        for tokens in (1, 2, 4):
            assert g.outputs(torch.zeros(tokens, 64, dtype=torch.float16), 0) is None
