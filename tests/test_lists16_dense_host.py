"""Host-side checks of the dense weight from vector-length-16 index lists (csrc/lists_dense.cu at V = 16, C interface
include/vptq_b200_lists_dense.h) and of decode-only v = 16 modules (set_list_decode + set_lists_prefill +
prepare(drop_packed=True)).

* an integer mirror of what the kernel relies on, on v = 16 lists (index rows of 16 outputs) built by the torch
  builder, dealt and undealt: for every (index row, tile) the NS units hold every feature of the tile exactly once
  with the (main, residual) index of its packed field, and the padding entries are exactly the masked ones;
* the entry points with v = 16 descriptors and fake device addresses: workspace bytes, refusals before any launch;
* the symbol table: still version 1 and four exports;
* the Python routing with the native entry points stubbed, and the refusal matrix of prepare(drop_packed=True).
The GPU side: test_gpu_lists16_dense.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from vptq_b200 import lists
from vptq_b200.pack import pack_index

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZERO = 65536 * 4 + 65536 * 64   # the zero-at-rest head every op leaves untouched

# the shapes of tests/test_lists16_host.py / test_gpu_lists16.py and the Llama-3-70B / Nemotron-70B layers:
# (in_features, out_features, K, Kr, perm)
MIRROR = {
    "k65536_r256_ragged_o": (1024, 264, 65536, 256, True),
    "k16384_r16": (512, 64, 16384, 16, True),
    "k32768_nores_noperm": (768, 40, 32768, -1, False),
    "k8192_three_tiles": (9000, 48, 8192, 256, True),
    "i1004_r2": (1004, 100, 65536, 2, True),
    "ragged_4100_r256": (4100, 264, 65536, 256, True),
    "70b_q_o": (8192, 8192, 65536, 256, True),
    "70b_k_v": (8192, 1024, 65536, 256, True),
    "70b_gate_up": (8192, 28672, 65536, 256, True),
    "70b_down": (28672, 8192, 65536, 256, True),
}


def _fields(I, O, K, Kr, perm, seed):
    g = torch.Generator().manual_seed(seed)
    Ro = (O + 15) // 16
    idx = torch.randint(0, K, (1, Ro, I), generator=g)
    ridx = torch.randint(0, Kr, (1, Ro, I), generator=g) if Kr > 0 else None
    packed = pack_index(idx, K.bit_length() - 1, ridx, Kr.bit_length() - 1 if Kr > 0 else 0)
    p = torch.randperm(I, generator=g).to(torch.int32).to(torch.int16) if perm else None
    return packed, idx[0], None if ridx is None else ridx[0], p


@pytest.mark.parametrize("deal", [False, True])
@pytest.mark.parametrize("name", sorted(MIRROR))
def test_integer_mirror_every_feature_once_padding_masked(name, deal):
    I, O, K, Kr, perm = MIRROR[name]
    packed, idx, ridx, p = _fields(I, O, K, Kr, perm, seed=len(name))
    stream, tab, tcw = lists.build_lists(packed, num_centroids=K, num_res_centroids=Kr, in_features=I,
                                         out_features=O, perm=p, deal=deal, vector_len=16)
    ns, nt, tcw_g = lists.geometry(I, K)
    assert tcw == tcw_g and tcw <= 4096 and tcw % 8 == 0       # the shared tile: 2 planes of tcw x 16 bytes
    ro = (O + 15) // 16
    stream = stream.numpy().view(np.uint32)
    tab = tab.numpy().view(np.uint32)
    U = ns * nt * ro
    assert tab.shape[0] == U + 1
    first, valid_last, end = tab[:U] & ((1 << 26) - 1), tab[:U] >> 26, tab[1:] & ((1 << 26) - 1)
    nsteps = (end - first).astype(np.int64)
    assert (nsteps >= 1).all() and (valid_last <= 32).all() and int(end[-1]) == stream.shape[0]
    assert (first[1:] == end[:-1]).all()
    step_unit = np.repeat(np.arange(U), nsteps)
    step_local = np.arange(stream.shape[0]) - np.repeat(first.astype(np.int64), nsteps)
    lane = np.arange(32)[None, :]
    # the kernel's mask: every lane of a non-final step, lanes < valid count of the final step
    live = (step_local[:, None] < nsteps[step_unit][:, None] - 1) | (lane < valid_last[step_unit][:, None])
    assert not stream[~live].any()                       # padding entries: zero words, masked by the count
    u = np.broadcast_to(step_unit[:, None], stream.shape)[live]
    e = stream[live].astype(np.int64)
    r, combo = u % ro, u // ro
    s, t = combo % ns, combo // ns
    col = (e >> 12) & 4095
    f = t * tcw + col
    assert (col < tcw).all() and (f < I).all()
    # every (index row, feature) exactly once: the NS units of (r, t) partition the tile's features
    key = r * I + f
    assert key.size == ro * I and np.unique(key).size == ro * I
    inv = np.arange(I) if p is None else np.argsort(p.numpy().view(np.uint16).astype(np.int64))
    c = inv[f]
    assert np.array_equal((e & 4095) + 4096 * s, idx.numpy()[r, c])
    want_r = ridx.numpy()[r, c] if ridx is not None else np.zeros_like(e)
    assert np.array_equal(e >> 24, want_r)


# ---------------------------------------------------------------- entry points, fake device addresses
def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    # Llama-3-70B gate/up at v = 16, decode-only: lists, no packed words (fake, never dereferenced: every call below
    # is refused before anything is launched)
    base = dict(dtype=0, in_features=8192, out_features=28672, vector_len=16, num_centroids=65536,
                num_res_centroids=256, num_codebooks=1, group_size=8192, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=None, index_stride_codebook=0, index_stride_row=6144,
                centroids=0x20000, centroid_stride=65536 * 16, res_centroids=0x30000, res_centroid_stride=4096,
                lists_stream=0x40000, lists_tab=0x50000, lists_tile_cols=4096)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


def _align(n, a=1024):
    return (n + a - 1) // a * a


def test_symbols_are_unchanged():
    from test_lists_dense_host import _declared
    from vptq_b200 import native
    assert _declared("vptq_b200_lists_dense.h") == sorted(native.LISTS_DENSE_EXPORTS)
    assert len(native.LISTS_DENSE_EXPORTS) == 4 and native.LISTS_DENSE_VERSION == 1
    assert "#define VPTQ_B200_LISTS_DENSE_VERSION 1" in open(os.path.join(ROOT, "include",
                                                                          "vptq_b200_lists_dense.h")).read()
    assert native.lib().vptq_b200_lists_dense_version() == 1
    assert native.LISTS16_VERSION == 1 and len(native.LISTS16_EXPORTS) == 4


def test_workspace_bytes_v16():
    from vptq_b200 import native
    ws = native.lib().vptq_b200_lists_dense_workspace_bytes
    for tokens in (1, 3, 8192):
        # forward: W [28672][8192] + staged x; transposed: the input-gradient GEMM's layout, as at v = 8
        assert ws(ctypes.byref(_desc()), tokens, 0) == ZERO + 28672 * 8192 * 2 + _align(tokens * 8192 * 2)
        assert ws(ctypes.byref(_desc()), tokens, native.FLAG_TRANSPOSE) == \
            ZERO + 8192 * 28672 * 2 + _align(tokens * 28672 * 2)
    # ragged: O % 16 != 0, I % 8 != 0 (tile width of the lists geometry)
    I, O = 4100, 264
    ragged = _desc(in_features=I, out_features=O, group_size=I, lists_tile_cols=lists.geometry(I, 65536)[2])
    assert ws(ctypes.byref(ragged), 5, 0) == ZERO + _align(O * 4160 * 2) + _align(5 * 4160 * 2)
    assert ws(ctypes.byref(ragged), 5, native.FLAG_TRANSPOSE) == ZERO + _align(I * 320 * 2) + _align(5 * 320 * 2)


def test_refusals_before_any_launch_v16():
    from vptq_b200 import native
    L = native.lib()
    T = native.FLAG_TRANSPOSE
    gemm, deq, wsb = L.vptq_b200_lists_quant_gemm, L.vptq_b200_lists_dequant, L.vptq_b200_lists_dense_workspace_bytes
    d = _desc()
    ws = 1 << 40
    # descriptors the v = 16 lists do not cover: refused with a message naming both families
    for bad in (_desc(lists_tile_cols=2048),                                  # not the lists geometry's tile width
                _desc(num_res_centroids=1024, res_centroid_stride=1024 * 16),  # Kr > 256
                _desc(vector_len=12, centroid_stride=65536 * 12, res_centroid_stride=256 * 12),
                _desc(num_centroids=4096, centroid_stride=4096 * 16),         # one slice
                _desc(num_codebooks=2, group_size=4096),
                _desc(lists_stream=0x40008)):                                 # lists_stream not 16-byte aligned
        for flags in (0, T):
            assert gemm(ctypes.byref(bad), 0x1000, 28672, 0x2000, 28672, 8, 0x3000, ws, flags, None) == -2
            assert "vector_len 8 or 16" in native.last_error()
            assert deq(ctypes.byref(bad), 0x1000, 28672, flags, None) == -2
            assert wsb(ctypes.byref(bad), 8, flags) == 0
    # no lists at all
    full = _desc(lists_stream=None, lists_tab=None, indices=0x10000, index_stride_row=6144)
    assert deq(ctypes.byref(full), 0x1000, 8192, 0, None) == -2 and "no index lists" in native.last_error()
    # dequant: ld < columns, ld % 8, misaligned or NULL w, unknown flags
    for ld, flags in ((8191, 0), (8196, 0), (28671, T), (28676, T), (8192, T)):
        assert deq(ctypes.byref(d), 0x1000, ld, flags, None) == -1, (ld, flags)
        assert "ld" in native.last_error()
    assert deq(ctypes.byref(d), 0x1008, 8192, 0, None) == -1
    assert deq(ctypes.byref(d), None, 8192, 0, None) == -1
    assert deq(ctypes.byref(d), 0x1000, 8192, native.FLAG_PDL, None) == -1
    # GEMM: tokens < 1, short strides (swapped for the transposed call), NULL x / y, unknown flags
    assert gemm(ctypes.byref(d), 0x1000, 8192, 0x2000, 28672, 0, 0x3000, ws, 0, None) == -1
    for xs, ys, flags in ((8191, 28672, 0), (8192, 28671, 0), (8192, 28672, T), (28672, 8191, T)):
        assert gemm(ctypes.byref(d), 0x1000, xs, 0x2000, ys, 8, 0x3000, ws, flags, None) == -1, (xs, ys, flags)
        assert "stride" in native.last_error()
    assert gemm(ctypes.byref(d), None, 8192, 0x2000, 28672, 8, 0x3000, ws, 0, None) == -1
    assert gemm(ctypes.byref(d), 0x1000, 8192, None, 28672, 8, 0x3000, ws, 0, None) == -1
    assert gemm(ctypes.byref(d), 0x1000, 8192, 0x2000, 28672, 8, 0x3000, ws, 8, None) == -1
    assert "unknown flags" in native.last_error()
    if not torch.cuda.is_available():
        # well-formed arguments reach the device check, which fails on a host without an H100
        assert gemm(ctypes.byref(d), 0x1000, 8192, 0x2000, 28672, 8, 0x3000, ws, 0, None) < 0
        assert deq(ctypes.byref(d), 0x1000, 8192, 0, None) < 0


# ---------------------------------------------------------------- python routing with native stubbed
class _Desc:
    def __init__(self, indices=0):
        self.lists_stream = 1
        self.vector_len = 16
        self.indices = indices     # 0: decode-only


def _stub(monkeypatch, max_tokens=4):
    from vptq_b200 import native
    calls = []

    def rec(name):
        return lambda d, x, y, flags=0: calls.append((name, x.shape[0], x.data_ptr() % 16, x.clone(), flags))
    for name in ("quant_gemv", "quant_gemm", "quant_gemv_batch", "quant_gemv_lists16", "lists_quant_gemm",
                 "quant_gemm_dgrad"):
        monkeypatch.setattr(native, name, rec(name))
    monkeypatch.setattr(native, "batch_max_tokens", lambda d: 0)   # v = 16: the batched kernel takes nothing
    monkeypatch.setattr(native, "lists16_max_tokens", lambda d: max_tokens)
    return calls


def _rows(tokens, I=64, off=0):
    buf = torch.arange(tokens * I + 32, dtype=torch.float16)
    o = (-buf.data_ptr() % 16) // 2 + off
    return buf[o:o + tokens * I].view(tokens, I)


@pytest.mark.parametrize("batched", [False, True])
def test_decode_only_v16_routes_only_to_list_entry_points(monkeypatch, batched):
    from vptq_b200 import ops
    for max_tokens in (4, 2, 1):
        calls = _stub(monkeypatch, max_tokens)
        for tokens in list(range(1, 10)) + [2048]:
            for off in (0, 1):
                calls.clear()
                ops._forward(_Desc(), _rows(tokens, off=off), 32, batched, True, True)
                want = "quant_gemv_lists16" if tokens <= max_tokens else "lists_quant_gemm"
                assert [c[0] for c in calls] == [want], (max_tokens, tokens, off)
                if want == "quant_gemv_lists16":     # a misaligned x runs on an aligned copy of the same values
                    assert calls[0][2] == 0 and torch.equal(calls[0][3], _rows(tokens, off=off))


def test_full_v16_module_keeps_todays_routes(monkeypatch):
    """with the packed words, a misaligned x is still left to the generic kernel (no copy)"""
    from vptq_b200 import ops
    calls = _stub(monkeypatch)
    ops._forward(_Desc(indices=1), _rows(1, off=1), 32, False, True, True)
    assert [c[0] for c in calls] == ["quant_gemv"]
    calls.clear()
    ops._forward(_Desc(indices=1), _rows(9), 32, False, True, True)
    assert [c[0] for c in calls] == ["quant_gemm"]


def test_input_gradient_of_decode_only_v16_reads_the_lists(monkeypatch):
    from vptq_b200 import native, ops
    calls = _stub(monkeypatch)

    class _Ctx:
        lists_prefill = True
        needs_input_grad = (True, True)
    d = _Desc()
    d.in_features = 64
    dy = torch.ones(5, 32, dtype=torch.float16)
    dx, db = ops._input_grads(_Ctx(), d, dy)
    assert [(c[0], c[4]) for c in calls] == [("lists_quant_gemm", native.FLAG_TRANSPOSE)]
    assert dx.shape == (5, 64) and torch.equal(db, torch.full((32,), 5.0, dtype=torch.float16))


# ---------------------------------------------------------------- prepare(drop_packed=True) refusal matrix
def _cpu_make_desc(monkeypatch, max_tokens=4, built=True):
    """native.make_desc on CPU tensors: the builder, the SM count and the token limit stubbed"""
    from vptq_b200 import native
    monkeypatch.setattr(native, "require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(native, "_sm_count", lambda dev: 132)
    monkeypatch.setattr(native, "lists16_max_tokens", lambda d: max_tokens)
    fake = (torch.zeros(4, 32, dtype=torch.int32), torch.zeros(9, dtype=torch.int32), 4096)
    monkeypatch.setattr(lists, "build_lists", lambda *a, **k: fake)
    monkeypatch.setattr(lists, "launchable", lambda *a, **k: built)


def _make(vector_len=16, Kr=256, **kw):
    from vptq_b200 import native
    I, O = 8192, 1024
    return native.make_desc(
        dtype=torch.float16, in_features=I, out_features=O, vector_len=vector_len, num_centroids=65536,
        num_res_centroids=Kr, num_codebooks=1, group_size=I, outlier_size=0, outlier_vector_len=-1,
        num_outlier_centroids=-1, indices=torch.zeros(1, O // vector_len, 3 * I // 4, dtype=torch.int32),
        centroids=torch.zeros(1, 65536 * vector_len, dtype=torch.float16),
        res_centroids=torch.zeros(1, Kr * vector_len, dtype=torch.float16), outlier_indices=None,
        outlier_centroids=None, perm=None, weight_scale=None, weight_bias=None, bias=None, drop_packed=True, **kw)


@pytest.mark.parametrize("list_decode", [False, True])
@pytest.mark.parametrize("lists_prefill", [False, True])
@pytest.mark.parametrize("layer", ["eligible", "kr1024", "not_launchable", "no_token_count"])
def test_drop_packed_refusal_matrix(monkeypatch, list_decode, lists_prefill, layer):
    _cpu_make_desc(monkeypatch, max_tokens=0 if layer == "no_token_count" else 4, built=layer != "not_launchable")
    kw = dict(lists=False, lists16=list_decode, lists_prefill=lists_prefill)
    has_lists = list_decode and layer != "kr1024" and layer != "not_launchable"
    if layer == "eligible" and list_decode and lists_prefill:
        d = _make(**kw)
        assert not d.indices and d.lists_stream
        return
    with pytest.raises(RuntimeError) as e:
        _make(Kr=1024 if layer == "kr1024" else 256, **kw)
    if has_lists and not lists_prefill:
        assert "vector_len 8 only" in str(e.value)
    else:
        assert "no index lists" in str(e.value)


def test_v8_drop_packed_needs_no_v16_opt_in(monkeypatch):
    _cpu_make_desc(monkeypatch)
    assert not _make(vector_len=8, lists=True).indices


def _lin(I=64):
    from vptq_b200 import VQuantLinear
    return VQuantLinear(I, 32, vector_lens=[-1, 16], num_centroids=[-1, 256], num_res_centroids=[-1, -1], group_num=1,
                        group_size=I, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                        dtype=torch.float16, enable_proxy_error=False)


@pytest.mark.parametrize("list_decode", [False, True])
@pytest.mark.parametrize("lists_prefill", [False, True])
def test_module_hands_both_opt_ins_to_the_descriptor_and_keeps_indices_on_refusal(monkeypatch, list_decode,
                                                                                   lists_prefill):
    from vptq_b200 import native
    seen = []

    def refuse(**kw):
        seen.append((kw["drop_packed"], kw["lists16"], kw["lists_prefill"]))
        raise RuntimeError("drop_packed: refused")
    monkeypatch.setattr(native, "require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(native, "make_desc", refuse)
    m = _lin().set_list_decode(list_decode).set_lists_prefill(lists_prefill)
    n = m.indices.numel()
    with pytest.raises(RuntimeError, match="refused"):
        m.prepare(drop_packed=True)
    assert seen == [(True, list_decode, lists_prefill)] and m.indices.numel() == n
    assert not m._decode_only()


def test_decode_only_v16_module_keeps_its_opt_ins():
    m = _lin().set_list_decode().set_lists_prefill()
    m._drop_packed, m.indices.data = True, torch.empty(0, dtype=torch.int32)   # as prepare(drop_packed=True) leaves it
    for off in (m.set_list_decode, m.set_lists_prefill):
        with pytest.raises(RuntimeError, match="decode-only"):
            off(False)
    assert m._list_decode and m._lists_prefill
    assert m.set_list_decode(True) is m and m.set_lists_prefill(True) is m   # turning them on again is harmless
    with pytest.raises(RuntimeError, match="decode-only"):
        m.set_quant_grad(True)
    with pytest.raises(RuntimeError, match="decode-only"):
        m.prepare(rebuild=True)
    with pytest.raises(RuntimeError, match="decode-only"):   # the checkpoint would lack the packed words
        m.state_dict()
    with pytest.raises(RuntimeError, match="decode-only"):   # also as a member of a model
        torch.nn.Sequential(m).state_dict()


def test_decode_only_v8_module_state_dict_is_unchanged():
    from vptq_b200 import VQuantLinear
    m = VQuantLinear(64, 32, vector_lens=[-1, 8], num_centroids=[-1, 256], num_res_centroids=[-1, -1], group_num=1,
                     group_size=64, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                     dtype=torch.float16, enable_proxy_error=False)
    m._drop_packed, m.indices.data = True, torch.empty(0, dtype=torch.int32)
    assert m.state_dict()["indices"].numel() == 0


def test_fused_group_keeps_decode_only_descriptors_but_not_across_dtypes(monkeypatch):
    """a decode-only member's descriptor no longer follows `indices`, so a fused call does not re-prepare it; another
    dtype still goes through the member's prepare (whose forward refuses a mismatched x)"""
    from vptq_b200.fuse import FusedGroup
    a, b = _lin(), _lin()
    prepared = []
    for m in (a, b):
        m._desc_cache = ["desc", None]
        m._desc_key = m._cache_key(m._tensors(), torch.float16, torch.device("cpu"))
        m._drop_packed, m.indices.data = True, torch.empty(0, dtype=torch.int32)   # the key's `indices` slot changed
        monkeypatch.setattr(m, "prepare", lambda dtype, m=m: prepared.append((m, dtype)))
    g = FusedGroup([a, b])
    assert g._descs(torch.zeros(1, 64, dtype=torch.float16)) == ["desc", "desc"] and prepared == []
    g._descs(torch.zeros(1, 64, dtype=torch.bfloat16))
    assert prepared == [(a, torch.bfloat16), (b, torch.bfloat16)]
