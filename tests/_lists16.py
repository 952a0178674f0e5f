"""Helpers for the GPU tests of the vector-length-16 list kernel (csrc/gemv_lists16.cu): descriptors, one launch,
layers generated on the GPU at sizes whose fp64 weight would not fit (checked on a seeded sample of index rows), and
the shapes that sit at the kernel's cut-offs (asserted against the integer mirror in tests/test_lists16_host.py)."""
import numpy as np
import torch

import vptq_oracle as vo

KERNEL = "gemv_lists16_kernel"
SMEM_OPTIN, SM_COUNT = 232448, 132   # H100 SXM: the cut-off shapes below are where they are for this device

# (residual replication, ring stages) of the shared-memory carve -> (in_features, out_features, Kr, tokens): one
# shape each that the carve places there.  (2, 3) and (1, 3) are never chosen for Kr <= 256: dropping a stage frees
# 16 KiB, at least what halving the replication from 4 to 2 (or from 2 to 1) frees, and the carve tries it first.
CARVE = {(8, 3): (4096, 1024, 0, 4), (8, 2): (4096, 1024, 64, 4), (4, 3): (4096, 1024, 256, 1),
         (4, 2): (4096, 1024, 256, 2), (2, 2): (4096, 1024, 256, 4), (1, 2): (32768, 72176, 256, 4)}
EXACT_FIT = (32768, 72176)          # Q = 128, one CTA per combo: 232448 bytes at NTOK = 4 (replication 1, 2 stages)
PAST_FIT = (32768, 72192)           # one index row more: NTOK = 4 does not fit, 2 does
# row-token limit at I = 4096 (32768 [row][token] accumulators of 16 outputs): out_features -> largest token count
ROW_TOKENS = {131072: 4, 262144: 2, 524288: 1, 524304: 0}
QKV_405B = (16384, [16384, 1024, 1024])   # Q = 64, B = 2 < 3 layers: refused as one group


def desc_t(t, dtype, I, O, K, Kr, lists16=True):
    """descriptor of a v = 16 layer (its tensors hang off it as `_tensors`), with or without the v = 16 lists"""
    from vptq_b200 import native
    d = native.make_desc(dtype=torch.float16 if dtype == "fp16" else torch.bfloat16, in_features=I, out_features=O,
                         vector_len=16, num_centroids=K, num_res_centroids=Kr, num_codebooks=1, group_size=I,
                         outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1, outlier_indices=None,
                         outlier_centroids=None, lists16=lists16, **t)
    d._tensors = t
    return d


def tensors_of(L):
    from _gpu import to_t
    return dict(indices=to_t(L.indices, L, "i32"), centroids=to_t(L.centroids, L),
                res_centroids=to_t(L.res_centroids, L) if L.res_bits else None,
                perm=to_t(L.perm, L, "u16") if L.perm is not None else None,
                weight_scale=to_t(L.weight_scale, L) if L.weight_scale is not None else None,
                weight_bias=to_t(L.weight_bias, L) if L.weight_bias is not None else None,
                bias=to_t(L.bias, L) if L.bias is not None else None)


def desc_of(L, lists16=True):
    """list-carrying v = 16 descriptor of the oracle layer L"""
    d = desc_t(tensors_of(L), L.dtype, L.in_features, L.out_features, L.num_centroids, L.num_res_centroids, lists16)
    assert bool(d.lists_stream) == lists16
    return d


def run(descs, x, ys=None, flags=0):
    """one vptq_b200_quant_gemv_lists16 launch; outputs NaN-filled unless given"""
    from vptq_b200 import native
    single = not isinstance(descs, (list, tuple))
    descs = [descs] if single else list(descs)
    if ys is None:
        ys = [torch.full((x.shape[0], d.out_features), float("nan"), dtype=x.dtype, device=x.device) for d in descs]
    native.FusedGemvLists16(descs, ys)(x, flags)
    return ys[0] if single else ys


def only_kernel(fn, launches=None):
    """fn launches the v = 16 list kernel and nothing else (`launches` of it, when given)"""
    from _probe import launched_kernels, ran
    names = launched_kernels(fn)
    assert names and all(ran([n], KERNEL) for n in names), names
    assert launches is None or len(names) == launches, names


def repack(L, idx=None, ridx=None):
    """copy of the oracle layer L with index fields idx / ridx ([1, Ro, I]; None: unchanged)"""
    import _extreme as ex
    L = ex.copy_layer(L)
    i0, r0 = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    idx = i0 if idx is None else idx
    ridx = r0 if ridx is None else ridx
    L.indices = vo.pack_index(idx, L.index_bits, ridx if L.res_bits else None, L.res_bits)
    L.meta["idx"] = idx
    if L.res_bits:
        L.meta["ridx"] = ridx
    return L


def module_of(G):
    """VQuantLinear holding a GpuLayer16's tensors (eval mode, list decode off)"""
    from vptq_b200 import VQuantLinear
    t = G.t
    m = VQuantLinear(G.I, G.O, vector_lens=[-1, 16], num_centroids=[-1, G.K], num_res_centroids=[-1, G.Kr],
                     group_num=1, group_size=G.I, outlier_size=0, indices_as_float=False, is_indice_packed=True,
                     enable_norm=t["weight_scale"] is not None, enable_perm=t["perm"] is not None,
                     bias=t["bias"] is not None, device="cuda", dtype=t["centroids"].dtype, enable_proxy_error=False)
    with torch.no_grad():
        m.indices.data = t["indices"]
        m.centroids.weight.data = t["centroids"].reshape(1, -1)
        if G.Kr > 0:
            m.res_centroids.weight.data = t["res_centroids"].reshape(1, -1)
        if t["perm"] is not None:
            m.perm.data = t["perm"]
        if t["weight_scale"] is not None:
            m.weight_scale.data, m.weight_bias.data = t["weight_scale"], t["weight_bias"]
        if t["bias"] is not None:
            m.bias.data = t["bias"]
    return m.eval()


# ------------------------------------------------------------------------------------------------------------------
# layers built on the GPU, checked on a sample of index rows
# ------------------------------------------------------------------------------------------------------------------
class GpuLayer16:
    """A seeded v = 16 layer (one group) generated and packed on the GPU, with its v = 16 list descriptor;
    `check` compares outputs on a sample of index rows with the oracle of those rows.  `all_ones`: every index field
    K - 1 and every residual field Kr - 1."""

    def __init__(self, I, O, *, K=65536, Kr=256, dtype="fp16", seed=0, lists16=True, perm=True, norm=True, bias=False,
                 all_ones=False):
        from vptq_b200.pack import pack_index
        self.I, self.O, self.K, self.Kr, self.dtype = I, O, K, Kr, dtype
        self.Ro = (O + 15) // 16
        dt = torch.float16 if dtype == "fp16" else torch.bfloat16
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
        if all_ones:
            idx = torch.full((1, self.Ro, I), K - 1, dtype=torch.int64, device="cuda")
            ridx = torch.full((1, self.Ro, I), Kr - 1, dtype=torch.int64, device="cuda") if Kr > 0 else None
        else:
            idx = torch.randint(0, K, (1, self.Ro, I), device="cuda", generator=g)
            ridx = torch.randint(0, Kr, (1, self.Ro, I), device="cuda", generator=g) if Kr > 0 else None
        t = dict(indices=pack_index(idx, K.bit_length() - 1, ridx, Kr.bit_length() - 1 if Kr > 0 else 0))
        del idx, ridx
        t["centroids"] = (0.02 * rnd(1, K * 16)).to(dt)
        t["res_centroids"] = (0.005 * rnd(1, Kr * 16)).to(dt) if Kr > 0 else None
        t["perm"] = torch.randperm(I, device="cuda", generator=g).to(torch.int32).to(torch.int16) if perm else None
        t["weight_scale"] = (1.0 + 0.1 * rnd(I)).to(dt) if norm else None
        t["weight_bias"] = (0.01 * rnd(I)).to(dt) if norm else None
        t["bias"] = (0.1 * rnd(O)).to(dt) if bias else None
        self.t = t
        self.desc = desc_t(t, dtype, I, O, K, Kr if Kr > 0 else -1, lists16)

    def sample(self, n, seed=0):
        """sorted seeded sample of n index rows (all rows when there are at most n), always the last one"""
        if self.Ro <= n:
            return np.arange(self.Ro)
        rows = np.random.default_rng(seed).choice(self.Ro - 1, size=n - 1, replace=False)
        return np.sort(np.append(rows, self.Ro - 1))

    def oracle(self, rows):
        """(oracle Layer of index rows `rows`, the output columns of the full layer they hold, which of those are
        real outputs: the last index row may be padding past out_features)"""
        from _batch import _np16
        t, dt = self.t, self.dtype
        rows = np.asarray(rows)
        cols = (rows[:, None] * 16 + np.arange(16)[None, :]).reshape(-1)
        keep = cols < self.O
        L = vo.Layer(dtype=dt, in_features=self.I, out_features=len(rows) * 16, vector_len=16, num_centroids=self.K,
                     num_res_centroids=self.Kr if self.Kr > 0 else -1, num_codebooks=1, group_size=self.I)
        L.indices = t["indices"][:, torch.from_numpy(rows).cuda()].cpu().numpy()
        L.centroids = _np16(t["centroids"], dt)
        if self.Kr > 0:
            L.res_centroids = _np16(t["res_centroids"], dt)
        if t["perm"] is not None:
            L.perm = t["perm"].cpu().numpy().view(np.uint16)
        if t["weight_scale"] is not None:
            L.weight_scale, L.weight_bias = _np16(t["weight_scale"], dt), _np16(t["weight_bias"], dt)
        if t["bias"] is not None:
            b = np.zeros(len(cols), dtype=np.float32)
            b[keep] = t["bias"].float().cpu().numpy()[cols[keep]]
            L.bias = _np16(torch.from_numpy(b).to(torch.float16 if dt == "fp16" else torch.bfloat16), dt)
        return L, cols, keep

    def check(self, x, y, n=48, seed=0, rows=None):
        """y [tokens, O] within the bar of the kernel's arithmetic on sampled rows, twice that of the exact product"""
        from _batch import assert_close, kernel_star, q_of
        import _extreme as ex
        L, cols, keep = self.oracle(self.sample(n, seed) if rows is None else rows)
        k = torch.from_numpy(np.nonzero(keep)[0]).cuda()
        ys = y[:, torch.from_numpy(cols[keep]).cuda()]
        q = q_of(self.I, self.K)
        assert torch.isfinite(ys).all()
        assert_close(ys, kernel_star(L, x)[:, k], self.dtype, q)
        assert_close(ys, ex.y_star(L, x)[:, k], self.dtype, q, factor=2.0)

    def probe(self, features, rows):
        """one-hot probes x = e_f (f in `features`, up to 4 per launch, each token count 1..4) through one launch
        each: the outputs of index rows `rows` equal the list kernel's arithmetic to the last bit"""
        from _probe import probe_expect
        L, cols, keep = self.oracle(rows)
        dt = self.t["centroids"].dtype
        expect = torch.from_numpy(probe_expect(L, "lists")).to("cuda").to(dt)[:, torch.from_numpy(keep).cuda()]
        cols = torch.from_numpy(cols[keep]).cuda()
        features = list(features)
        for a in range(0, len(features), 4):
            f = features[a:a + 4]
            x = torch.zeros(4, self.I, dtype=dt, device="cuda")
            x[torch.arange(len(f)), torch.tensor(f, device="cuda")] = 1.0
            x = x[:len(f)]
            y = run(self.desc, x)
            torch.cuda.synchronize()
            want = expect[torch.tensor(f, device="cuda")]
            assert torch.equal(y[:, cols].view(torch.int16), want.view(torch.int16)), (self.I, self.O, f)
