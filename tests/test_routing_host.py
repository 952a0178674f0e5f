"""Which kernel takes each call: the routing table of VQuantLinear, its input gradient and fused groups (CPU).

Every launcher and max-token query of `native` is stubbed, so this runs without a GPU.  The expected routes are
written out here as the rules, independently of the code under test:

One call, the first rule that holds wins (T tokens, A: x starts on 16 bytes, P: the descriptor still has its packed
words, L: it has index lists; B, LP, LD: set_batched_decode, set_lists_prefill, set_list_decode):
  1. T == 0: no launch
  2. LD, v = 16, L, A or not P, T <= lists16_max_tokens: the v = 16 list kernel (a misaligned x runs on a copy)
  3. B, T >= 2, L, A, T <= batch_max_tokens: the batched list kernel
  4. LP, T >= 2, not P: the GEMM from the lists
  5. T < 3: the GEMV;  6. otherwise the GEMM
A max-token query runs exactly when every other condition of its rule holds.

Input gradient: not P and LP -> the transposed GEMM from the lists; not P without LP -> refused; else the dgrad GEMM.

Fused group (grad mode off, dense rows on the GPU): the same rules with B and LD = every member opted in and
"LP and not P" = some decode-only member opted in to LP; x is never copied.  A v = 8 group launches GEMV or batched
routes as one, a v = 16 group only the v = 16 list kernel; every other route leaves each member to its own forward.
"""
from __future__ import annotations

import itertools

import pytest
import torch

I, O = 64, 32
TOKENS = list(range(0, 11)) + [2048]
MAX = (0, 1, 2, 4, 8)


class _Desc:
    def __init__(self, v, lists, packed):
        self.vector_len, self.lists_stream, self.indices, self.in_features = v, int(lists), int(packed), I


def _module(v, packed, B, LP, LD):
    """A VQuantLinear whose kept descriptor is a _Desc (the parameters' cache key is current)."""
    from vptq_b200 import VQuantLinear
    m = VQuantLinear(I, O, vector_lens=[-1, v], num_centroids=[-1, 256], num_res_centroids=[-1, -1], group_num=1,
                     group_size=I, outlier_size=0, indices_as_float=False, is_indice_packed=True, bias=True,
                     dtype=torch.float16, enable_proxy_error=False)
    m.set_batched_decode(B).set_lists_prefill(LP).set_list_decode(LD)
    d = _Desc(v, True, packed)
    if not packed:                       # as prepare(drop_packed=True) leaves a module
        m._drop_packed, m.indices.data = True, torch.empty(0, dtype=torch.int32)
    m._desc_cache = [d, None]
    m._desc_key = m._cache_key(m._tensors(), torch.float16, torch.device("cpu"))
    return m, d


class _Native:
    """Records every launch and max-token query; the answers of the queries are set per case."""

    def __init__(self, monkeypatch):
        from vptq_b200 import native
        self.calls, self.queries, self.m16, self.mb = [], [], 0, 0
        monkeypatch.setattr(native, "require_cuda", lambda *a, **k: None)
        for name in ("quant_gemv", "quant_gemm", "quant_gemv_batch", "quant_gemv_lists16", "lists_quant_gemm",
                     "quant_gemm_dgrad"):
            monkeypatch.setattr(native, name, self._launch(name))
        monkeypatch.setattr(native, "batch_max_tokens", self._query("batch", lambda d: d.lists_stream, "mb"))
        monkeypatch.setattr(native, "lists16_max_tokens",
                            self._query("lists16", lambda d: d.lists_stream and d.vector_len == 16, "m16"))
        rec = self

        class Fused:
            def __init__(self, descs, ys):
                self.descs, self.ys = descs, ys

            def __call__(self, x2d, flags=0):
                rec.calls.append((type(self).__name__, len(self.descs), x2d.shape[0]))
        for name in ("FusedGemv", "FusedGemvBatch", "FusedGemvLists16"):
            monkeypatch.setattr(native, name, type(name, (Fused,), {}))

    def _launch(self, name):
        def f(d, x, y, flags=0):
            self.calls.append((name, x.shape[0], x.data_ptr() % 16, x.clone(), flags))
        return f

    def _query(self, kind, ok, attr):
        def f(descs):
            descs = list(descs) if isinstance(descs, (list, tuple)) else [descs]
            self.queries.append((kind, len(descs)))
            return getattr(self, attr) if all(ok(d) for d in descs) else 0   # as native: 0 without lists
        return f


def _x(tokens, aligned):
    buf = torch.arange(tokens * I + 32, dtype=torch.float16)
    o = (-buf.data_ptr() % 16) // 2 + (0 if aligned else 1)
    return buf[o:o + tokens * I].view(tokens, I)


def _expect(v, L, P, A, B, LP, LD, T, m16, mb):
    """(route, max-token queries) of one call by the rules of the module docstring."""
    if T == 0:
        return None, []
    q = []
    if LD and v == 16 and L and (A or not P):
        q.append(("lists16", 1))
        if T <= m16:
            return "quant_gemv_lists16", q
    if B and T >= 2 and L and A:
        q.append(("batch", 1))
        if T <= mb:
            return "quant_gemv_batch", q
    if LP and T >= 2 and not P:
        return "lists_quant_gemm", q
    return ("quant_gemv" if T < 3 else "quant_gemm"), q


@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("packed", [True, False])
@pytest.mark.parametrize("B,LP,LD", list(itertools.product([False, True], repeat=3)))
def test_one_call(monkeypatch, v, packed, B, LP, LD):
    nat = _Native(monkeypatch)
    m, d = _module(v, packed, B, LP, LD)
    for L, A, T, m16, mb in itertools.product([True, False], [True, False], TOKENS, MAX, MAX):
        d.lists_stream = int(L)
        nat.m16, nat.mb = m16, mb
        nat.calls.clear()
        nat.queries.clear()
        x = _x(T, A)
        with torch.no_grad():
            y = m(x)
        want, queries = _expect(v, L, packed, A, B, LP, LD, T, m16, mb)
        case = (L, A, T, m16, mb)
        assert y.shape == (T, O), case
        assert [c[0] for c in nat.calls] == ([want] if want else []), case
        assert nat.queries == queries, case
        if want:
            assert nat.calls[0][1] == T and nat.calls[0][4] == 0, case
            if want == "quant_gemv_lists16":     # a misaligned decode-only call runs on an aligned copy of x
                assert nat.calls[0][2] == 0 and torch.equal(nat.calls[0][3], x), case
            else:
                assert nat.calls[0][2] == (0 if A else 2), case


@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("packed", [True, False])
@pytest.mark.parametrize("LP", [False, True])
def test_input_gradient(monkeypatch, v, packed, LP):
    from vptq_b200 import native
    nat = _Native(monkeypatch)
    nat.m16 = nat.mb = 8
    m, _ = _module(v, packed, True, LP, True)
    for T in (0, 1, 2, 5):
        nat.calls.clear()
        x = _x(T, True).clone().requires_grad_(True)
        y = m(x)
        nat.calls.clear()
        if not packed and not LP:
            with pytest.raises(RuntimeError, match="decode-only"):
                y.backward(torch.ones_like(y))
            continue
        y.backward(torch.ones_like(y))
        assert x.grad.shape == (T, I) and torch.equal(m.bias.grad, torch.full((O,), float(T), dtype=torch.float16))
        m.bias.grad = None
        want = ("lists_quant_gemm", native.FLAG_TRANSPOSE) if not packed else ("quant_gemm_dgrad", 0)
        assert [(c[0], c[4]) for c in nat.calls] == ([want] if T else []), T


# member kinds of a fused group: (packed, B, LP, LD)
KINDS = [(True, False, False, False), (True, True, True, True), (False, True, True, True), (False, False, True, False)]


def _groups():
    for n in (1, 2, 3):
        kinds = itertools.product([True, False], repeat=4) if n == 1 else itertools.product(KINDS, repeat=n)
        for k in kinds:
            yield (k,) if n == 1 else k


def _expect_group(v, kinds, L, A, T, m16, mb):
    """(launcher or None, the max-token queries allowed) of a fused group's call."""
    B = all(k[1] for k in kinds)
    LD = all(k[3] for k in kinds)
    lists_decode_only = any(k[2] and not k[0] for k in kinds)
    allowed = set()
    if T == 0:
        return None, allowed
    if LD and v == 16 and A:
        allowed.add("lists16")
    if B and T >= 2 and A:
        allowed.add("batch")
    if LD and v == 16 and L and A and T <= m16:
        route = "FusedGemvLists16"
    elif B and T >= 2 and L and A and T <= mb:
        route = "FusedGemvBatch"
    elif lists_decode_only and T >= 2:
        route = None
    elif T < 3:
        route = "FusedGemv"
    else:
        route = None
    fusable = ("FusedGemvLists16",) if v == 16 else ("FusedGemv", "FusedGemvBatch")
    return (route if route in fusable else None), allowed


@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("L", [True, False])
def test_fused_group(monkeypatch, v, L):
    from vptq_b200.fuse import FusedGroup
    nat = _Native(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    modules = {}
    for k in itertools.product([True, False], repeat=4):
        modules[k] = _module(v, *k)
        modules[k][1].lists_stream = int(L)
    xs = {(T, A): _x(T, A) for T in TOKENS for A in (True, False)}
    for kinds in _groups():
        layers = [modules[k][0] for k in kinds]
        for (T, A), (m16, mb) in itertools.product(xs, zip(MAX, (0, 8, 2, 8, 4))):
            nat.m16, nat.mb = m16, mb
            nat.calls.clear()
            nat.queries.clear()
            g = FusedGroup(layers)
            with torch.no_grad():
                out = g.outputs(xs[T, A], 0)
            want, allowed = _expect_group(v, kinds, L, A, T, m16, mb)
            case = (kinds, T, A, m16, mb)
            assert (out is None) == (want is None), case
            assert [c[0] for c in nat.calls] == ([want] if want else []), case
            if want:
                assert nat.calls[0][1:] == (len(kinds), T) and out.shape == (T, O * len(kinds)), case
                if len(kinds) > 1:     # the next member takes its slice of the same launch
                    assert g.outputs(xs[T, A], 1) is out and len(nat.calls) == 1, case
            assert {q for q, n in nat.queries} <= allowed and all(n == len(kinds) for _, n in nat.queries), case


def test_grad_mode_and_layout_leave_each_member_its_own_forward(monkeypatch):
    from vptq_b200.fuse import FusedGroup
    nat = _Native(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    layers = [_module(8, True, False, False, False)[0] for _ in range(2)]
    g = FusedGroup(layers)
    x = _x(1, True)
    assert g.outputs(x.clone().requires_grad_(True), 0) is None          # autograd records each member
    layers[0].set_quant_grad(True)
    layers[0].centroids.weight.requires_grad_(True)
    assert g.outputs(x, 0) is None                                       # some member needs quantizer gradients
    layers[0].set_quant_grad(False)
    with torch.no_grad():
        assert g.outputs(torch.zeros(I, dtype=torch.float16).expand(2, I), 0) is None     # rows overlap
        assert g.outputs(torch.zeros(2, 2 * I, dtype=torch.float16)[:, ::2], 0) is None   # columns not dense
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: False))
        assert g.outputs(x, 0) is None                                   # not on the GPU
    assert nat.calls == [] and nat.queries == []
