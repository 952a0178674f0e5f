"""CPU-side tests of the state kept between calls: the descriptor and packed-word cache keys (inference tensors,
res_indices), prepare(rebuild=True)'s refusal, the activation key of fused groups, and the workspace bookkeeping
(growth, capture-private buffers, release) driven with fake buffers.  The GPU side: test_gpu_lifecycle.py."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

UNPACKED = dict(vector_lens=[-1, 8], num_centroids=[-1, 256], num_res_centroids=[-1, 16], group_num=1,
                group_size=64, outlier_size=0, indices_as_float=False, enable_norm=True, enable_perm=True,
                is_indice_packed=False, bias=True, dtype=torch.float16, enable_proxy_error=False)


def _unpacked(seed=0):
    from vptq_b200 import VQuantLinear
    m = VQuantLinear(64, 32, **UNPACKED)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.indices.copy_(torch.randint(0, 256, m.indices.shape, generator=g).to(torch.int16))
        m.res_indices.copy_(torch.randint(0, 16, m.res_indices.shape, generator=g).to(torch.int16))
    return m


def _key(m):
    return m._cache_key(m._tensors(), torch.float16, torch.device("cpu"))


# ---------------------------------------------------------------- cache keys
def test_cache_keys_of_inference_tensors():
    """A module built inside inference mode holds inference tensors: reading their _version raises, so the keys must
    not.  They stay stable from call to call."""
    from vptq_b200 import VQuantLinear
    with torch.inference_mode():
        m = VQuantLinear(64, 32, **UNPACKED)
        m.indices.zero_()
        m.res_indices.zero_()
    assert m.indices.is_inference() and m.centroids.weight.is_inference()
    with pytest.raises(RuntimeError):
        m.indices._version          # the torch behaviour the keys work around
    for mode in (torch.inference_mode, torch.no_grad):
        with mode():
            assert _key(m) == _key(m)
            p = m._packed_indices()
            assert m._packed_indices() is p


def test_cache_keys_of_ordinary_tensors_under_inference_mode():
    """Ordinary parameters keep their version counters inside inference mode: an in-place update there is seen."""
    m = _unpacked()
    k0 = _key(m)
    with torch.inference_mode():
        assert _key(m) == k0
        m.centroids.weight.mul_(2)
        assert _key(m) != k0


def test_res_indices_is_in_both_keys():
    """An in-place update of res_indices alone (unpacked checkpoint) changes the descriptor key and repacks the
    words: they carry the residual field."""
    from vptq_b200.pack import pack_index
    m = _unpacked()
    k0, p0 = _key(m), m._packed_indices().clone()
    assert torch.equal(p0, pack_index(m.indices, 8, m.res_indices, 4))
    with torch.no_grad():
        m.res_indices.copy_((m.res_indices + 1) % 16)
    assert _key(m) != k0
    p1 = m._packed_indices()
    assert not torch.equal(p1, p0)
    assert torch.equal(p1, pack_index(m.indices, 8, m.res_indices, 4))
    # a res_indices change is not a floating-point update: the descriptor (and its lists) must be rebuilt
    m._desc_cache, m._desc_key = [object(), None], k0
    assert not m._refresh_in_place(_key(m))


def test_keys_miss_data_writes():
    """`.data.copy_` does not bump the version counter (why prepare(rebuild=True) exists)."""
    m = _unpacked()
    k0 = _key(m)
    m.indices.data.copy_((m.indices.data + 1) % 256)
    assert _key(m) == k0


def test_rebuild_drops_the_caches_and_refuses_decode_only_modules():
    m = _unpacked()
    m._packed_indices()
    packed = m._packed
    m._desc_cache, m._desc_key = [object(), None], _key(m)
    with pytest.raises(RuntimeError, match="CUDA"):      # the rebuild itself runs a forward: CUDA only
        m.prepare(rebuild=True)
    assert m._desc_cache == [] and m._packed is not packed    # dropped although the keys had not changed
    from vptq_b200 import VQuantLinear
    d = VQuantLinear(64, 32, **dict(UNPACKED, is_indice_packed=True))
    d._drop_packed, d.indices.data = True, torch.empty(0, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="decode-only"):
        d.prepare(rebuild=True)


def test_activation_key_of_inference_tensors():
    from vptq_b200.fuse import activation_key
    x = torch.zeros(1, 8)
    k = activation_key(x)
    x.add_(1)
    assert activation_key(x) != k             # an in-place write between members is seen
    with torch.inference_mode():
        xi = torch.zeros(1, 8)
        assert activation_key(xi) == activation_key(xi)


# ---------------------------------------------------------------- workspace bookkeeping
class Buf:
    """A fake workspace: only numel() is read."""

    def __init__(self, n, tag):
        self.n, self.tag = n, tag

    def numel(self):
        return self.n


class Pool:
    def __init__(self):
        self.current, self.retired, self.captured, self.made = {}, [], {}, []

    def get(self, key, nbytes, capture_id=0):
        from vptq_b200.native import pick_workspace

        def alloc(n):
            b = Buf(n, capture_id)
            self.made.append(b)
            return b
        return pick_workspace(key, nbytes, capture_id, alloc, self.current, self.retired, self.captured)

    def alive(self):
        return list(self.current.values()) + self.retired + list(self.captured.values())


def test_workspace_growth_retires_and_doubles():
    p, k = Pool(), (0, 7)
    a = p.get(k, 4 << 20)
    assert p.get(k, 1000) is a and p.get(k, 4 << 20) is a
    b = p.get(k, (4 << 20) + 1)
    assert b is not a and b.numel() >= 2 * a.numel() and p.retired == [a] and p.current[k] is b
    c = p.get(k, 100 << 20)
    assert c.numel() == 100 << 20 and p.retired == [a, b]
    for n in (c.numel() + 1, 3 * c.numel(), 3 * c.numel() + 5):
        p.get(k, n)
    largest = max(x.numel() for x in p.alive())
    assert sum(x.numel() for x in p.retired) < largest     # everything retired stays below the largest buffer
    assert all(any(x is y for y in p.alive()) for x in p.made)   # nothing a graph may hold was dropped


def test_workspace_minimum_and_streams_apart():
    p = Pool()
    a, b = p.get((0, 1), 10), p.get((0, 2), 10)
    assert a is not b and a.numel() == b.numel() == 1 << 20
    assert p.get((1, 1), 10) is not a


def test_capture_buffers_are_private():
    p, k = Pool(), (0, 3)
    # a capture on a stream without an eager buffer gets its own, even for a tiny request
    c1 = p.get(k, 100, capture_id=11)
    assert k not in p.current and p.get(k, 100, capture_id=11) is c1
    c2 = p.get(k, 100, capture_id=12)
    assert c2 is not c1
    e = p.get(k, 100)                          # eager calls never see a capture's buffer
    assert e is not c1 and e is not c2 and p.current[k] is e
    # a later capture that fits the eager buffer shares it (it is zero at rest)
    assert p.get(k, 100, capture_id=13) is e
    # growth inside a capture: private to it, the eager buffer stays current and alive
    g = p.get(k, 64 << 20, capture_id=13)
    assert g is not e and p.current[k] is e and p.captured[k + (13,)] is g
    g2 = p.get(k, 200 << 20, capture_id=13)
    assert g2.numel() == 200 << 20 and g in p.retired and p.captured[k + (13,)] is g2
    # growth outside capture leaves every capture's buffer alone
    e2 = p.get(k, 300 << 20)
    assert e in p.retired and p.captured[k + (11,)] is c1 and p.captured[k + (12,)] is c2
    assert e2 is not g2 and p.get(k, 300 << 20) is e2


def test_release_workspaces_drops_everything(monkeypatch):
    from vptq_b200 import native
    cur, ret, cap = {(0, 1): Buf(1 << 20, 0)}, [Buf(1 << 20, 0)], {(0, 1, 5): Buf(1 << 20, 5)}
    monkeypatch.setattr(native, "_workspaces", cur)
    monkeypatch.setattr(native, "_retired", ret)
    monkeypatch.setattr(native, "_captured", cap)
    native.release_workspaces()
    assert cur == {} and ret == [] and cap == {}


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    return sorted(set(re.findall(r"VPTQ_B200_API[^;(]*?(vptq_b200_\w+)\s*\(", src)))


def test_graph_header_symbols_are_exported_and_apart_from_the_other_headers():
    """include/vptq_b200_graph.h declares exactly GRAPH_EXPORTS, the library exports them, and neither the inference
    nor the gradient header declares them (their symbol sets stay as they were)."""
    from vptq_b200 import native
    L = native.lib()
    syms = _declared("vptq_b200_graph.h")
    assert syms == sorted(native.GRAPH_EXPORTS) == ["vptq_b200_stream_capture_id"]
    for s in syms:
        assert hasattr(L, s), s
    assert not set(syms) & (set(_declared("vptq_b200.h")) | set(_declared("vptq_b200_grad.h")))
    assert not set(syms) & (set(native.EXPORTS) | set(native.GRAD_EXPORTS))
    assert "vptq_b200_graph.h" in open(os.path.join(ROOT, "include", "vptq_b200.h")).read()


def test_stream_capture_id_export():
    """It validates its output pointer before touching CUDA."""
    from vptq_b200 import native
    L = native.lib()
    assert L.vptq_b200_stream_capture_id(None, None) == -1
    assert "NULL id" in native.last_error()
    if not torch.cuda.is_available():
        cid = ctypes.c_uint64(123)
        assert L.vptq_b200_stream_capture_id(None, ctypes.byref(cid)) < 0    # no device: an error, not "capturing"
