"""The state that lives between calls, checked against fp64 and against fresh modules.

Every other GPU test builds a module, calls it once or replays one graph, and compares.  Here the same modules are
called again after what real deployments do between calls:
  A. workspace lifetime: graphs captured and then replayed after the stream's workspace grew (eagerly or inside a
     later capture), the torch-docs capture pattern (warm-up on a side stream, capture on torch's capture stream),
     one memory pool shared by several graphs, every op on one workspace, two streams at once;
  B. weight updates: in-place updates and optimizer steps before graph replay, reloads, moves, permutations,
     unpacked checkpoints' res_indices, and writes through `.data` (prepare(rebuild=True));
  C. torch.inference_mode(): every route, fused groups, modules built and prepared inside it.
Whatever can be compared bit for bit is compared with the same call on a freshly built module; everything is also
compared with the fp64 oracle at TOL.  The host-side liveness checks (weakref) of A1 and A4 come before any replay.
"""
import copy
import gc
import random
import weakref

import numpy as np
import pytest
import torch
import torch.nn as nn

import vptq_oracle as vo
from _gpu import make_module, x_to_t
from _probe import fp64_bias, fp64_weight, launched_kernels, ran
from _util import TOL

pytestmark = pytest.mark.gpu

ZERO = 65536 * 4 + 65536 * 64          # the workspace's zero-at-rest head (DESIGN.md section 1)

CONFIGS = {
    "lists": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True),
    "lists_bf16": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True,
                       dtype="bf16"),
    "generic": dict(in_features=1000 + 128, out_features=250, vector_len=4, num_centroids=4096, num_res_centroids=16,
                    num_codebooks=2, outlier_size=128, outlier_vector_len=4, num_outlier_centroids=256, bias=True),
    "prep": dict(in_features=1004, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True),
    "q": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, seed=11),
    "k": dict(in_features=1024, out_features=128, num_centroids=65536, num_res_centroids=256, seed=12),
    "v": dict(in_features=1024, out_features=136, num_centroids=65536, num_res_centroids=256, bias=True, seed=13),
    "other": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, bias=True, seed=99),
    "other_q": dict(in_features=1024, out_features=264, num_centroids=65536, num_res_centroids=256, seed=98),
}
_LAYERS = {}


def layer(name):
    if name not in _LAYERS:
        _LAYERS[name] = vo.make_layer(**{"vector_len": 8, "seed": 4242, **CONFIGS[name]})
    return _LAYERS[name]


def xs(L, tokens, seed=1):
    return x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=seed), L)


KERNELS = {
    "lists": lambda n: ran(n, "gemv_lists_kernel") and not ran(n, "gemv_kernel"),
    "fused": lambda n: sum(ran([k], "gemv_lists_kernel") for k in n) == 1 and not ran(n, "gemv_kernel"),
    "generic": lambda n: ran(n, "gemv_kernel") and not ran(n, "gemv_lists_kernel"),
    "direct": lambda n: ran(n, "dequant_o8_kernel") and ran(n, "gemm_tn_wgmma") and not ran(n, "prefill_prep_x"),
    "prep": lambda n: ran(n, "prefill_prep_x") and ran(n, "gemm_tn_wgmma") and not ran(n, "dequant_o8_kernel"),
    "batch": lambda n: sum(ran([k], "gemv_lists_batch_kernel") for k in n) == 1 and not ran(n, "gemv_lists_kernel")
    and not ran(n, "gemv_kernel") and not ran(n, "gemm_tn_wgmma"),
}


def assert_route(kind, fn):
    names = launched_kernels(fn)
    assert KERNELS[kind](names), (kind, names)


def close64(L, x, y):
    """y against x W64^T + bias in fp64, at TOL."""
    ref = x.double() @ fp64_weight(L).T
    b = fp64_bias(L)
    if b is not None:
        ref = ref + b
    err = float((y.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
    assert err <= TOL[L.dtype], err


def close64_w(L, w):
    ref = fp64_weight(L)
    err = float((w.double() - ref).abs().max() / ref.abs().max())
    assert err <= TOL[L.dtype], err


def np16(t, L):
    t = t.detach().cpu().contiguous()
    return t.numpy() if L.dtype == "fp16" else t.view(torch.int16).numpy().view(np.uint16)


def layer_of(m, L):
    """The oracle Layer of module m's current tensors (L gives the configuration)."""
    L2 = copy.copy(L)
    L2.indices = m.indices.detach().cpu().numpy().reshape(np.shape(L.indices))
    L2.centroids = np16(m.centroids.weight, L).reshape(np.shape(L.centroids))
    if L.res_bits:
        L2.res_centroids = np16(m.res_centroids.weight, L).reshape(np.shape(L.res_centroids))
    if L.perm is not None:
        L2.perm = m.perm.detach().cpu().numpy().view(np.uint16).reshape(np.shape(L.perm))
    if L.weight_scale is not None:
        L2.weight_scale, L2.weight_bias = np16(m.weight_scale, L), np16(m.weight_bias, L)
    if L.bias is not None:
        L2.bias = np16(m.bias, L)
    return L2


def fresh_of(m, L):
    """A new module holding copies of m's current tensors."""
    f = make_module(L)
    f.load_state_dict(m.state_dict())
    return f


def heads_at_rest():
    """Every workspace the library holds -- current, retired, private to a capture -- is zero in its head."""
    from vptq_b200 import native
    torch.cuda.synchronize()
    bufs = list(native._workspaces.values()) + list(native._retired) + list(native._captured.values())
    assert bufs
    for b in bufs:
        assert int(b[:min(ZERO, b.numel())].count_nonzero()) == 0


@pytest.fixture(autouse=True)
def _own_workspaces():
    """torch's stream pool recycles handles, so workspace keys alias across tests: start and end with none."""
    from vptq_b200 import native
    torch.cuda.synchronize()
    gc.collect()
    native.release_workspaces()
    yield
    torch.cuda.synchronize()
    gc.collect()
    native.release_workspaces()


def same(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def ws_key(stream):
    return (torch.cuda.current_device(), stream.cuda_stream)


class QKV(nn.Module):
    def __init__(self, dtype_layers=("q", "k", "v")):
        super().__init__()
        self.q_proj, self.k_proj, self.v_proj = (make_module(layer(n)) for n in dtype_layers)

    def forward(self, x):
        return torch.cat([self.q_proj(x), self.k_proj(x), self.v_proj(x)], dim=-1)


def fresh_qkv(layers):
    """A new fused q/k/v group holding copies of `layers`' tensors: fused launches are compared with fused launches
    (the fused generic GEMV need not round like three separate ones)."""
    from vptq_b200 import fuse
    f = QKV()
    for name, l in zip(("q_proj", "k_proj", "v_proj"), layers):
        getattr(f, name).load_state_dict(l.state_dict())
    fuse(f)
    return f


def qkv_oracle_check(x, y):
    a = 0
    for n in ("q", "k", "v"):
        L = layer(n)
        close64(L, x, y[:, a:a + L.out_features])
        a += L.out_features


# ================================================================================================ A. workspaces
def test_a1_graphs_survive_eager_workspace_growth():
    from vptq_b200 import native
    L, Lp = layer("lists"), layer("prep")
    m, mp, qkv = make_module(L), make_module(Lp), [make_module(layer(n)) for n in "qkv"]
    for mm in (m, mp, *qkv):
        mm.prepare()
    x1, x2 = xs(L, 1), xs(L, 2, seed=2)
    ysf = [torch.empty(1, l.out_features, dtype=torch.float16, device="cuda") for l in qkv]
    fused = native.FusedGemv([l._desc_cache[0] for l in qkv], ysf)
    assert_route("lists", lambda: m(x1))
    assert_route("generic", lambda: m(x2))
    assert_route("fused", lambda: fused(x1))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        e1, e2 = m(x1), m(x2)                      # warm-up: the stream's eager workspace
        fused(x1)
        ef = torch.cat(ysf, 1).clone()
        g1, g2, gf = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1, stream=s):
            y1 = m(x1)
        with torch.cuda.graph(g2, stream=s):
            y2 = m(x2)
        with torch.cuda.graph(gf, stream=s):
            fused(x1)
        old = native._workspaces[ws_key(s)]
        size, old_ref = old.numel(), weakref.ref(old)
        del old
        for mm, LL in ((mp, Lp), (m, L)):                # prefills on the same stream: the workspace grows
            for t in (300, 8192):
                x = xs(LL, t, seed=t)
                close64(LL, x, mm(x))
        assert native._workspaces[ws_key(s)] is not old_ref(), "the prefills did not grow the workspace"
    assert old_ref() is not None, "workspace of the captured graphs was freed when the stream's workspace grew"
    assert_route("direct", lambda: m(xs(L, 300)))
    assert_route("prep", lambda: mp(xs(Lp, 300)))
    filler = torch.full((size,), 0xA5, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(s):
        for _ in range(10):
            g1.replay()
            g2.replay()
            gf.replay()
    torch.cuda.synchronize()
    assert same(y1, e1) and same(y2, e2) and same(torch.cat(ysf, 1), ef)
    assert bool((filler == 0xA5).all()), "a replay wrote into memory the allocator had handed out again"
    close64(L, x1, y1)
    close64(L, x2, y2)
    heads_at_rest()


def test_a2_torch_docs_capture_pattern():
    """Warm up on a side stream, capture with torch.cuda.graph(g) (torch's own capture stream, which has no
    workspace yet), replay the last graph first, then the others, interleaved with eager calls."""
    from vptq_b200 import native
    L, Lg = layer("lists"), layer("generic")
    m, mg = make_module(L), make_module(Lg)
    x1, x2, xg = xs(L, 1), xs(L, 2, seed=2), xs(Lg, 1, seed=3)
    assert_route("generic", lambda: mg(xg))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        e1, e2, eg = m(x1), m(x2), mg(xg)
    torch.cuda.current_stream().wait_stream(s)
    graphs = []
    with torch.no_grad():
        for fn in (lambda: m(x1), lambda: m(x2), lambda: mg(xg)):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                y = fn()
            graphs.append((g, y))
    cap = torch.cuda.graphs.graph.default_capture_stream
    assert ws_key(cap) not in native._workspaces, "a buffer zeroed inside one capture was left for everyone"
    expect = (e1, e2, eg)
    for i in (2, 0, 1):
        graphs[i][0].replay()
        torch.cuda.synchronize()
        assert same(graphs[i][1], expect[i]), i
    with torch.no_grad():
        for rep in range(3):
            for i in (1, 2, 0):
                graphs[i][0].replay()
                assert same(m(x1), e1) and same(mg(xg), eg)
                torch.cuda.synchronize()
                assert same(graphs[i][1], expect[i]), (rep, i)
    close64(Lg, xg, graphs[2][1])
    heads_at_rest()


def test_a3_shared_pool_largest_first():
    from vptq_b200 import fuse
    L = layer("lists")
    m, qkv = make_module(L), QKV()
    fuse(qkv)
    x64, x2, x1 = xs(L, 64, seed=64), xs(L, 2, seed=2), xs(L, 1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    fns = [lambda: m(x64), lambda: qkv(x1), lambda: m(x2), lambda: m(x1)]
    with torch.cuda.stream(s), torch.no_grad():
        expect = [fn().clone() for fn in fns]
        graphs, pool = [], None
        for fn in fns:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s, pool=pool):
                y = fn()
            pool = pool if pool is not None else g.pool()
            graphs.append((g, y))
    rng = random.Random(3)
    order = [3, 2, 1, 0] + [rng.randrange(4) for _ in range(24)]
    with torch.cuda.stream(s):
        for i in order:
            graphs[i][0].replay()
            s.synchronize()
            assert same(graphs[i][1], expect[i]), i
    close64(L, x64, graphs[0][1])
    qkv_oracle_check(x1, graphs[1][1])
    heads_at_rest()


def test_a4_graph_survives_growth_during_a_later_capture():
    from vptq_b200 import native
    L, Lp = layer("lists"), layer("prep")
    m, mp = make_module(L), make_module(Lp)
    x1, xp = xs(L, 1), xs(Lp, 300, seed=300)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        e1 = m(x1)
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1, stream=s):
            y1 = m(x1)
        ws = native._workspaces[ws_key(s)]
        mp.prepare()
        assert native.workspace_bytes(mp._desc_cache[0], 300, native.OP_GEMM) > ws.numel()
        ref = weakref.ref(ws)
        del ws
        gp = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gp, stream=s):
            yp = mp(xp)
    assert ref() is not None and native._workspaces[ws_key(s)] is ref(), \
        "the decode graph's workspace was replaced by one allocated inside a later capture"
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(10):
            gp.replay()
            g1.replay()
    torch.cuda.synchronize()
    assert same(y1, e1)
    with torch.no_grad():
        assert same(yp, mp(xp))
    close64(Lp, xp, yp)
    heads_at_rest()


def _ops():
    """Every op of the library on the layers of this file, as closures returning fresh outputs."""
    from vptq_b200 import native
    L, Lg, Lp = layer("lists"), layer("generic"), layer("prep")
    m, mg, mp, qkv = make_module(L), make_module(Lg), make_module(Lp), [make_module(layer(n)) for n in "qkv"]
    for mm in (m, mg, mp, *qkv):
        mm.prepare()
    d = m._desc_cache[0]
    x1, x2, x300, xg, xp = xs(L, 1), xs(L, 2, seed=2), xs(L, 300, seed=5), xs(Lg, 1, seed=3), xs(Lp, 300, seed=6)
    dy = x_to_t(vo.make_x(300, L.out_features, L.dtype, seed=7), L)
    dw = x_to_t(vo.make_x(L.out_features, L.in_features, L.dtype, seed=8), L)

    def grads():
        return {"centroids": torch.zeros_like(m.centroids.weight), "res_centroids": torch.zeros_like(m.res_centroids.weight),
                "weight_scale": torch.zeros_like(m.weight_scale), "weight_bias": torch.zeros_like(m.weight_bias)}

    def fused():
        ys = [torch.empty(1, l.out_features, dtype=torch.float16, device="cuda") for l in qkv]
        native.FusedGemv([l._desc_cache[0] for l in qkv], ys)(x1)
        return torch.cat(ys, 1)

    def dgrad():
        dx = torch.empty(300, L.in_features, dtype=torch.float16, device="cuda")
        native.quant_gemm_dgrad(d, dy, dx)
        return dx

    def wgrad(flags):
        def f():
            g = grads()
            native.quant_gemm_wgrad(d, x300, dy, g, flags)
            return torch.cat([t.reshape(-1) for t in g.values()])
        return f

    def dequant_backward():
        g = grads()
        native.dequant_backward(d, dw, g)
        return torch.cat([t.reshape(-1) for t in g.values()])

    return {"lists": lambda: m(x1), "generic": lambda: mg(xg), "fused": fused, "direct": lambda: m(x300),
            "prep": lambda: mp(xp), "dequant": m.dequant, "dgrad": dgrad, "wgrad": wgrad(0),
            "wgrad_generic": wgrad(native.GRAD_FLAG_GENERIC), "dequant_backward": dequant_backward}


def test_a5_every_op_on_one_workspace():
    from vptq_b200 import native
    ops = _ops()
    alone = {}
    for name, fn in ops.items():                  # each op alone, on a stream of its own
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            alone[name] = fn()
        s.synchronize()
    L = layer("lists")
    close64(L, xs(L, 1), alone["lists"])
    close64(L, xs(L, 300, seed=5), alone["direct"])
    close64_w(L, alone["dequant"])
    names = list(ops) * 2
    random.Random(5).shuffle(names)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for name in names:
            y = ops[name]()
            s.synchronize()
            ws = native._workspaces[ws_key(s)]
            assert int(ws[:ZERO].count_nonzero()) == 0, name
            assert same(y, alone[name]), name
    heads_at_rest()


@pytest.mark.parametrize("pair", [("lists", "generic"), ("lists", "lists"), ("lists", "prep")])
def test_a6_two_streams_at_once(pair):
    mods = {n: make_module(layer(n)) for n in set(pair)}
    tokens = {"lists": 1, "generic": 1, "prep": 300}
    xin = {n: xs(layer(n), tokens[n], seed=9) for n in pair}
    with torch.no_grad():
        serial = {n: mods[n](xin[n]) for n in pair}
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    outs = [[], []]
    with torch.no_grad():
        for _ in range(50):
            for k, (s, n) in enumerate(zip(streams, pair)):
                with torch.cuda.stream(s):
                    outs[k].append(mods[n](xin[n]))
    torch.cuda.synchronize()
    for k, n in enumerate(pair):
        for i, y in enumerate(outs[k]):
            assert same(y, serial[n]), (n, k, i)
    for n in set(pair):
        close64(layer(n), xin[n], serial[n])
    heads_at_rest()


# ================================================================================================ B. weight updates
def _check_all_routes(m, L, fresh, tag=""):
    """1 token (lists), 2 tokens, 300 tokens and dequant() of m bit-identical to `fresh` and close to fp64."""
    L2 = layer_of(fresh, L)
    with torch.no_grad():
        for t in (1, 2, 300):
            x = xs(L, t, seed=20 + t)
            y = m(x)
            assert same(y, fresh(x)), (tag, t)
            close64(L2, x, y)
        w = m.dequant()
        assert same(w, fresh.dequant()), tag
        close64_w(L2, w)


@pytest.mark.parametrize("update", ["mul", "adam"])
def test_b1_graphs_after_in_place_updates(update):
    L, Lp = layer("lists"), layer("prep")
    m, mp = make_module(L), make_module(Lp)
    m.prepare()
    mp.prepare()
    desc, stream = m._desc_cache[0], m._desc_cache[0].lists_stream
    assert stream
    inputs = [(m, xs(L, 1)), (m, xs(L, 2, seed=2)), (m, xs(L, 300, seed=3)), (mp, xs(Lp, 300, seed=4))]
    assert_route("lists", lambda: m(inputs[0][1]))
    assert_route("direct", lambda: m(inputs[2][1]))
    assert_route("prep", lambda: mp(inputs[3][1]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graphs = []
    with torch.cuda.stream(s), torch.no_grad():
        for mm, x in inputs:
            mm(x)
        for mm, x in inputs:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                y = mm(x)
            graphs.append((g, y))
    torch.cuda.current_stream().wait_stream(s)
    for mm in (m, mp):
        params = [mm.centroids.weight, mm.res_centroids.weight, mm.weight_scale, mm.weight_bias, mm.bias]
        if update == "mul":
            with torch.no_grad():
                for k, p in enumerate(params):
                    p.mul_(1.0 + 0.125 * (k + 1))
        else:
            mm.set_quant_grad(True)
            for p in params:
                p.requires_grad_(True)
            opt = torch.optim.Adam(params, lr=1e-3, eps=1e-4)
            x = xs(L if mm is m else Lp, 64, seed=30)
            mm(x).float().square().mean().backward()
            opt.step()
            mm.set_quant_grad(False)
        mm.prepare()
    assert m._desc_cache[0] is desc and m._desc_cache[0].lists_stream == stream
    fresh = {id(m): fresh_of(m, L), id(mp): fresh_of(mp, Lp)}
    with torch.cuda.stream(s):
        for g, _ in graphs:
            g.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        for (mm, x), (_, y) in zip(inputs, graphs):
            assert same(y, fresh[id(mm)](x)), (mm.in_features, x.shape[0])
            close64(layer_of(mm, L if mm is m else Lp), x, y)
    _check_all_routes(m, L, fresh[id(m)], update)
    heads_at_rest()


def _run_everything(m, L):
    with torch.no_grad():
        for t in (1, 2, 300):
            m(xs(L, t, seed=20 + t))
        m.dequant()


@pytest.mark.parametrize("change", ["copy_indices", "permute_perm", "load_state_dict", "init_parameters",
                                    "cpu_round_trip"])
def test_b2_eager_after_changes(change):
    L, Lo = layer("lists"), layer("other")
    m, other = make_module(L), make_module(Lo)
    _run_everything(m, L)
    with torch.no_grad():
        if change == "copy_indices":
            m.indices.copy_(other.indices)
        elif change == "permute_perm":
            p = torch.randperm(L.in_features, generator=torch.Generator().manual_seed(1)).cuda()
            m.perm.copy_(m.perm[p])
        elif change == "load_state_dict":
            m.load_state_dict(other.state_dict())
        elif change == "init_parameters":
            idx, ridx = vo.unpack_index(Lo.indices, Lo.index_bits, Lo.group_size, Lo.res_bits)
            cent = vo.to_f32(Lo.centroids, Lo.dtype).reshape(1, -1)
            resc = vo.to_f32(Lo.res_centroids, Lo.dtype).reshape(1, -1)
            m.init_parameters(
                {0: None, 1: torch.from_numpy(cent[0]).half()}, {0: None, 1: torch.from_numpy(idx[0])},
                res_centroids={0: None, 1: torch.from_numpy(resc[0]).half()}, res_indices={0: None, 1: torch.from_numpy(ridx[0])},
                weight_scale=other.weight_scale.detach().clone(), weight_bias=other.weight_bias.detach().clone(),
                perm=other.perm.detach().view(torch.uint16).to(torch.int64))
            m.bias.copy_(other.bias)
        else:
            m.to("cpu")
            m.to("cuda")
    _check_all_routes(m, L, fresh_of(m, L), change)


def test_b2_load_state_dict_through_fuse():
    from vptq_b200 import fuse
    p = QKV()
    fuse(p)
    x1 = xs(layer("q"), 1)
    with torch.no_grad():
        p(x1)
    sd = {**{"q_proj." + k: v for k, v in make_module(layer("other_q")).state_dict().items()},
          **{"k_proj." + k: v for k, v in p.k_proj.layer.state_dict().items()},
          **{"v_proj." + k: v for k, v in p.v_proj.layer.state_dict().items()}}
    p.load_state_dict(sd)
    ref = make_module(layer("other_q"))
    fresh = fresh_qkv([ref, p.k_proj.layer, p.v_proj.layer])
    with torch.no_grad():
        y = p(x1)                                    # rebuilds q_proj's descriptor and lists
        assert_route("fused", lambda: p(x1))
        assert same(y, fresh(x1))
        x2 = xs(layer("q"), 2, seed=2)
        assert same(p(x2), fresh(x2))
        x = xs(layer("q"), 300, seed=300)
        assert same(p.q_proj(x), ref(x))
    close64(layer("other_q"), x1, y[:, :264])


def _unpacked(L):
    from vptq_b200 import VQuantLinear
    mu = VQuantLinear(L.in_features, L.out_features, vector_lens=[-1, 8], num_centroids=[-1, L.num_centroids],
                      num_res_centroids=[-1, L.num_res_centroids], group_num=1, group_size=L.group_size,
                      outlier_size=0, indices_as_float=False, enable_norm=True, enable_perm=True,
                      is_indice_packed=False, bias=True, device="cuda", dtype=torch.float16, enable_proxy_error=False)
    mp = make_module(L)
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    with torch.no_grad():
        mu.indices.data = torch.from_numpy(idx.astype(np.uint16)).view(torch.int16).cuda()
        mu.res_indices.data = torch.from_numpy(ridx.astype(np.uint16)).view(torch.int16).cuda()
        for n in ("weight_scale", "weight_bias", "bias"):
            getattr(mu, n).data = getattr(mp, n).data.clone()
        mu.centroids.weight.data = mp.centroids.weight.data.clone()
        mu.res_centroids.weight.data = mp.res_centroids.weight.data.clone()
        mu.perm.data = torch.from_numpy(np.asarray(L.perm).astype(np.uint16).astype(np.int64)).cuda()
    return mu.eval()


def test_b2_unpacked_res_indices_update():
    from vptq_b200.pack import pack_index
    L = layer("lists")
    mu = _unpacked(L)
    _run_everything(mu, L)
    with torch.no_grad():
        r = mu.res_indices.view(torch.uint16).to(torch.int64)
        mu.res_indices.copy_(((r * 7 + 3) % L.num_res_centroids).to(torch.uint16).view(torch.int16))
    fresh = make_module(L)
    with torch.no_grad():
        fresh.indices.data = pack_index(mu.indices, L.index_bits, mu.res_indices, L.res_bits)
    _check_all_routes(mu, L, fresh, "res_indices")


def test_b3_data_writes_need_rebuild():
    L, Lo = layer("lists"), layer("other")
    m, other = make_module(L), make_module(Lo)
    _run_everything(m, L)
    m.indices.data.copy_(other.indices.data)
    m.weight_scale.data.copy_(other.weight_scale.data)
    stale = m(xs(L, 1, seed=21)).clone()
    m.prepare(rebuild=True)
    fresh = fresh_of(m, L)
    with torch.no_grad():
        assert not same(stale, fresh(xs(L, 1, seed=21))), "the write was visible without a rebuild"
    _check_all_routes(m, L, fresh, "rebuild")
    assert m._desc_cache[0].lists_stream


# ================================================================================================ C. inference mode
@pytest.mark.parametrize("name", ["lists", "lists_bf16", "generic", "prep"])
def test_c1_inference_mode_equals_no_grad(name):
    L = layer(name)
    m = make_module(L)
    inputs = [xs(L, t, seed=40 + t) for t in (1, 2, 300)]
    with torch.no_grad():
        ref = [m(x) for x in inputs] + [m.dequant()]
    with torch.inference_mode():
        got = [m(x) for x in inputs] + [m.dequant()]
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(inputs[0])
            with torch.cuda.graph(g, stream=s):
                yg = m(inputs[0])
            g.replay()
        torch.cuda.synchronize()
    for a, b in zip(got, ref):
        assert same(a, b)
    assert same(yg, ref[0])
    for x, y in zip(inputs, got):
        close64(L, x, y)
    heads_at_rest()


def test_c1_c2_fused_group_under_inference_mode():
    from vptq_b200 import fuse
    p = QKV()
    groups = fuse(p)
    assert len(groups) == 1
    x = xs(layer("q"), 1)
    with torch.no_grad():
        ref = p(x)
        ref2 = p(xs(layer("q"), 2, seed=2))
    with torch.inference_mode():
        xi = x.clone()
        assert xi.is_inference()
        assert_route("fused", lambda: p(xi))
        y = p(xi)
        y2 = p(xs(layer("q"), 2, seed=2))
    assert same(y, ref) and same(y2, ref2)
    qkv_oracle_check(x, y)


def test_c3_model_built_inside_inference_mode():
    L = layer("lists")
    with torch.inference_mode():
        m = make_module(L)
        assert m.centroids.weight.is_inference() and m.indices.is_inference()
        got = {t: m(xs(L, t, seed=50 + t)) for t in (1, 2, 300)}
        w = m.dequant()
        assert_route("lists", lambda: m(xs(L, 1)))
    ref = make_module(L)
    with torch.no_grad():
        for t, y in got.items():
            x = xs(L, t, seed=50 + t)
            assert same(y, ref(x)) and same(m(x), y), t
            close64(L, x, y)
        assert same(w, ref.dequant())
    close64_w(L, w)


def test_c4_prepared_in_inference_mode_then_trained():
    import vptq_b200
    p = QKV()
    with torch.inference_mode():
        vptq_b200.fuse(p)
        p(xs(layer("q"), 1))
    layers = [p.q_proj.layer, p.k_proj.layer, p.v_proj.layer]
    descs = [l._desc_cache[0] for l in layers]
    assert all(d.lists_stream for d in descs)
    vptq_b200.set_quant_grad(p, True)
    params = [t for l in layers for t in (l.centroids.weight, l.res_centroids.weight, l.weight_scale)]
    for l in layers:
        l.weight_bias.requires_grad_(False)
    opt = torch.optim.Adam(params, lr=1e-4, eps=1e-4)
    x = xs(layer("q"), 64, seed=60)
    target = torch.randn(64, 528, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 0.1
    x1, x300 = xs(layer("q"), 1, seed=61), xs(layer("q"), 300, seed=62)
    losses = []
    for step in range(3):
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(p(x).float(), target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
        with torch.no_grad():
            assert same(p(x1), fresh_qkv(layers)(x1)), step
            for k, (l, n) in enumerate(zip(layers, "qkv")):
                fresh = fresh_of(l, layer(n))
                assert same(l(x1), fresh(x1)), (step, n)
                assert same(l(x300), fresh(x300)), (step, n)
                assert l._desc_cache[0] is descs[k], (step, n)
    assert losses[-1] < losses[0], losses


# ================================================================================================ batched decode
def batched(L):
    return make_module(L).set_batched_decode(True)


def test_batch_graphs_across_growth_capture_streams_and_a_second_stream():
    """A1 + A2 + A6 for the batched route: a graph captured on a side stream survives eager workspace growth; a graph
    captured on torch's capture stream (a workspace private to the capture) replays last-captured first; a batched
    stream and a single-token list stream run at once"""
    from vptq_b200 import native
    L, Lp = layer("lists"), layer("prep")
    m, mp, m1 = batched(L), make_module(Lp), make_module(L)
    x5, x8, x1 = xs(L, 5, seed=5), xs(L, 8, seed=8), xs(L, 1, seed=1)
    assert_route("batch", lambda: m(x5))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        e5, e8 = m(x5), m(x8)
        g5 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g5, stream=s):
            y5 = m(x5)
        old = weakref.ref(native._workspaces[ws_key(s)])
        for t in (300, 8192):
            x = xs(Lp, t, seed=t)
            close64(Lp, x, mp(x))
        assert native._workspaces[ws_key(s)] is not old()
    assert old() is not None
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        g8 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g8):
            y8 = m(x8)
    assert ws_key(torch.cuda.graphs.graph.default_capture_stream) not in native._workspaces
    with torch.no_grad():
        for rep in range(3):
            g8.replay()
            with torch.cuda.stream(s):
                g5.replay()
            assert same(m(x5), e5)
            torch.cuda.synchronize()
            assert same(y8, e8) and same(y5, e5), rep
        serial1 = m1(x1)
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        for st in streams:
            st.wait_stream(torch.cuda.current_stream())
        outs = [[], []]
        for _ in range(30):
            with torch.cuda.stream(streams[0]):
                outs[0].append(m(x8))
            with torch.cuda.stream(streams[1]):
                outs[1].append(m1(x1))
    torch.cuda.synchronize()
    assert all(same(y, e8) for y in outs[0]) and all(same(y, serial1) for y in outs[1])
    close64(L, x5, e5)
    close64(L, x8, e8)
    heads_at_rest()


def test_batch_on_the_shared_workspace():
    """A5: the batched route interleaved with every other op on one stream's workspace, each result the bits of the
    op alone"""
    from vptq_b200 import native
    ops = _ops()
    L = layer("lists")
    mb = batched(L)
    x5 = xs(L, 5, seed=55)
    ops["batch"] = lambda: mb(x5)
    alone = {}
    for name, fn in ops.items():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            alone[name] = fn()
        s.synchronize()
    close64(L, x5, alone["batch"])
    names = list(ops) + ["batch"] * 4
    random.Random(6).shuffle(names)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for name in names:
            y = ops[name]()
            s.synchronize()
            assert int(native._workspaces[ws_key(s)][:ZERO].count_nonzero()) == 0, name
            assert same(y, alone[name]), name
    heads_at_rest()


@pytest.mark.parametrize("update", ["mul", "adam"])
def test_batch_graph_after_in_place_updates(update):
    """B1: mul_ or an Adam step on every float tensor (weight_scale / weight_bias are read in original order by this
    kernel), prepare(), then replay: the bits of a fresh module with batched decode on"""
    L = layer("lists")
    m = batched(L)
    m.prepare()
    x = xs(L, 6, seed=6)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        m(x)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            y = m(x)
    torch.cuda.current_stream().wait_stream(s)
    params = [m.centroids.weight, m.res_centroids.weight, m.weight_scale, m.weight_bias, m.bias]
    if update == "mul":
        with torch.no_grad():
            for k, p in enumerate(params):
                p.mul_(1.0 + 0.125 * (k + 1))
    else:
        m.set_quant_grad(True)
        for p in params:
            p.requires_grad_(True)
        opt = torch.optim.Adam(params, lr=1e-3, eps=1e-4)
        m(xs(L, 64, seed=30)).float().square().mean().backward()
        opt.step()
        m.set_quant_grad(False)
    m.prepare()
    fresh = fresh_of(m, L).set_batched_decode(True)
    with torch.cuda.stream(s):
        g.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        assert_route("batch", lambda: fresh(x))
        assert same(y, fresh(x))
        for t in (2, 5, 8):
            xt = xs(L, t, seed=70 + t)
            assert same(m(xt), fresh(xt)), t
    close64(layer_of(m, L), x, y)
    heads_at_rest()


@pytest.mark.parametrize("change", ["copy_indices", "permute_perm", "load_state_dict"])
def test_batch_eager_after_changes(change):
    """B2 for the batched route"""
    L, Lo = layer("lists"), layer("other")
    m, other = batched(L), make_module(Lo)
    with torch.no_grad():
        m(xs(L, 5))
        if change == "copy_indices":
            m.indices.copy_(other.indices)
        elif change == "permute_perm":
            p = torch.randperm(L.in_features, generator=torch.Generator().manual_seed(1)).cuda()
            m.perm.copy_(m.perm[p])
        else:
            m.load_state_dict(other.state_dict())
        fresh = fresh_of(m, L).set_batched_decode(True)
        for t in (2, 5, 8):
            x = xs(L, t, seed=80 + t)
            assert_route("batch", lambda: m(x))
            y = m(x)
            assert same(y, fresh(x)), (change, t)
            close64(layer_of(m, L), x, y)
    heads_at_rest()


def test_batch_load_state_dict_through_fuse():
    import vptq_b200
    p = QKV()
    vptq_b200.fuse(p)
    vptq_b200.set_batched_decode(p)
    x5 = xs(layer("q"), 5, seed=5)
    with torch.no_grad():
        p(x5)
    sd = {**{"q_proj." + k: v for k, v in make_module(layer("other_q")).state_dict().items()},
          **{"k_proj." + k: v for k, v in p.k_proj.layer.state_dict().items()},
          **{"v_proj." + k: v for k, v in p.v_proj.layer.state_dict().items()}}
    p.load_state_dict(sd)
    fresh = fresh_qkv([make_module(layer("other_q")), p.k_proj.layer, p.v_proj.layer])
    vptq_b200.set_batched_decode(fresh)
    with torch.no_grad():
        y = p(x5)                                    # rebuilds q_proj's descriptor and lists
        assert_route("batch", lambda: p(x5))
        assert same(y, fresh(x5))
    close64(layer("other_q"), x5, y[:, :264])
    heads_at_rest()


def test_batch_under_inference_mode():
    """C1 / C2: a module and a fused group under torch.inference_mode(), a graph included, equal to no_grad"""
    import vptq_b200
    L = layer("lists_bf16")
    m = batched(L)
    p = QKV()
    vptq_b200.fuse(p)
    vptq_b200.set_batched_decode(p)
    x, xq = xs(L, 7, seed=7), xs(layer("q"), 4, seed=4)
    with torch.no_grad():
        ref, refq = m(x), p(xq)
    with torch.inference_mode():
        xi, xqi = x.clone(), xq.clone()
        assert_route("batch", lambda: m(xi))
        assert_route("batch", lambda: p(xqi))
        got, gotq = m(xi), p(xqi)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(xi)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                yg = m(xi)
            g.replay()
        torch.cuda.synchronize()
    assert same(got, ref) and same(yg, ref) and same(gotq, refq)
    close64(L, x, got)
    qkv_oracle_check(xq, gotq)
    heads_at_rest()


# ------------------------------------------------------------------------------------------------ PDL chain
def test_batch_pdl_chain_of_a_llama_decoder_layer():
    """Llama-3-8B decoder layer of batched launches, each with programmatic dependent launch and reading the previous
    launch's output view directly: q/k/v -> o (on the q slice) -> gate/up -> down (on the gate slice) -> the next
    q/k/v.  Eager and as one CUDA graph, every stage the bits of the same launches run one at a time without PDL,
    and within the bar on the x it consumed"""
    from _batch import GpuLayer, assert_close, kernel_star, q_of
    from vptq_b200 import native
    qkv = [GpuLayer(4096, o, seed=90 + k) for k, o in enumerate((4096, 1024, 1024))]
    o_proj = [GpuLayer(4096, 4096, seed=93)]
    gate_up = [GpuLayer(4096, 14336, seed=94 + k) for k in range(2)]
    down = [GpuLayer(14336, 4096, seed=96)]
    qkv2 = [GpuLayer(4096, o, seed=97 + k) for k, o in enumerate((4096, 1024, 1024))]
    stages = [qkv, o_proj, gate_up, down, qkv2]
    for tokens in (2, 5, 8):
        x0 = torch.randn(tokens, 4096, device="cuda", generator=torch.Generator(device="cuda").manual_seed(tokens))
        x0 = (0.5 * x0).half()
        outs = [torch.empty(tokens, sum(l.O for l in st), dtype=torch.float16, device="cuda") for st in stages]

        def views(k):
            a, v = 0, []
            for l in stages[k]:
                v.append(outs[k][:, a:a + l.O])
                a += l.O
            return v
        srcs = [x0, outs[0][:, :4096], outs[1], outs[2][:, :14336], outs[3]]
        launches = [native.FusedGemvBatch([l.desc for l in st], views(k)) for k, st in enumerate(stages)]

        def chain(flags):
            for fb, src in zip(launches, srcs):
                fb(src, flags)

        ref = []
        for fb, src, out in zip(launches, srcs, outs):          # one at a time, no PDL
            fb(src, 0)
            torch.cuda.synchronize()
            ref.append(out.clone())
        for o in outs:
            o.fill_(float("nan"))
        chain(native.FLAG_PDL)
        torch.cuda.synchronize()
        assert all(same(o, r) for o, r in zip(outs, ref)), tokens
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain(native.FLAG_PDL)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                chain(native.FLAG_PDL)
        for o in outs:
            o.fill_(float("nan"))
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        for k, (o, r) in enumerate(zip(outs, ref)):
            assert same(o, r), (tokens, k)
        for k, st in enumerate(stages):
            src = x0 if k == 0 else [None, ref[0][:, :4096], ref[1], ref[2][:, :14336], ref[3]][k]
            a = 0
            for l in st:
                rows = l.sample(16, seed=k)
                Ls, cols, keep = l.oracle(rows)
                idx = torch.from_numpy(np.nonzero(keep)[0]).cuda()
                ys = ref[k][:, a:a + l.O][:, torch.from_numpy(cols[keep]).cuda()]
                assert_close(ys, kernel_star(Ls, src)[:, idx], l.dtype, q_of(l.I, l.K))
                a += l.O
        del g
    heads_at_rest()
