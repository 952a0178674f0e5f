"""Helpers for the GPU tests of the batched list kernel (csrc/gemv_lists_batch.cu): descriptors, one launch, the
fp64 evaluation of the kernel's arithmetic and its bar, and layers built on the GPU at sizes whose fp64 weight
would not fit (checked on a seeded sample of index rows)."""
import numpy as np
import torch

import vptq_oracle as vo
from _util import TOL

BATCH = "gemv_lists_batch_kernel"
ZERO_HEAD = 65536 * 4 + 65536 * 64   # kZeroRegionBytes: the workspace head kernels leave zeroed


def desc_of(L):
    """list-carrying descriptor of the oracle layer L (its tensors hang off it as `_tensors`)"""
    from _gpu import to_t
    t = dict(indices=to_t(L.indices, L, "i32"), centroids=to_t(L.centroids, L),
             res_centroids=to_t(L.res_centroids, L) if L.res_bits else None,
             perm=to_t(L.perm, L, "u16") if L.perm is not None else None,
             weight_scale=to_t(L.weight_scale, L) if L.weight_scale is not None else None,
             weight_bias=to_t(L.weight_bias, L) if L.weight_bias is not None else None,
             bias=to_t(L.bias, L) if L.bias is not None else None)
    return desc_from_tensors(t, L.dtype, L.in_features, L.out_features, L.num_centroids, L.num_res_centroids)


def desc_from_tensors(t, dtype, I, O, K, Kr, lists=True):
    from vptq_b200 import native
    d = native.make_desc(dtype=torch.float16 if dtype == "fp16" else torch.bfloat16, in_features=I, out_features=O,
                         vector_len=8, num_centroids=K, num_res_centroids=Kr, num_codebooks=1, group_size=I,
                         outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1, outlier_indices=None,
                         outlier_centroids=None, lists=lists, **t)
    d._tensors = t
    assert bool(d.lists_stream) == lists
    return d


def q_of(I, K):
    from vptq_b200.lists import geometry
    ns, nt, _ = geometry(I, K)
    return ns * nt


def batch(descs, x, ys=None, flags=0):
    """one vptq_b200_quant_gemv_batch launch; outputs NaN-filled unless given"""
    from vptq_b200 import native
    single = not isinstance(descs, (list, tuple))
    descs = [descs] if single else list(descs)
    if ys is None:
        ys = [torch.full((x.shape[0], d.out_features), float("nan"), dtype=x.dtype, device=x.device) for d in descs]
    native.FusedGemvBatch(descs, ys)(x, flags)
    return ys[0] if single else ys


def kernel_star(L, x):
    """fp64 evaluation of the kernel's arithmetic: rn16(x * s) . (C + R)^T [C + R rounded to fp16 for fp16 layers]
    + x . wbias + bias, as element-wise products (inf * 0 = NaN, like the kernel)"""
    import _extreme as ex
    P = ex.copy_layer(L)
    dt = torch.float16 if L.dtype == "fp16" else torch.bfloat16
    if P.weight_scale is not None:
        s = torch.from_numpy(vo.to_f32(L.weight_scale, L.dtype)).to(x.device)
        wb = torch.from_numpy(vo.to_f32(L.weight_bias, L.dtype).astype(np.float64)).to(x.device)
        P.weight_scale = ex.encode(np.ones(L.in_features), L.dtype)
        P.weight_bias = ex.encode(np.zeros(L.in_features), L.dtype)
        xq = (x.float() * s).to(dt).double()
    else:
        wb, xq = None, x.double()
    P.bias = None
    W = torch.from_numpy(ex.dense64(P)).to(x.device)             # C + R in fp64 (scale 1, bias 0)
    if L.dtype == "fp16":
        W = W.half().double()                                    # packed fp16 c + r
    y = ex.ew_matmul(xq, W, ex.bias64(L, x.device))
    if wb is not None:
        y = y + ex.ew_matmul(x.double(), wb[None, :])
    return y


def assert_close(y, ystar, dtype, q, factor=1.0):
    """per token t: |y - y*| <= factor (TOL max|y*_t| + Q 2^-31)"""
    for t in range(y.shape[0]):
        bar = factor * (TOL[dtype] * float(ystar[t].abs().max()) + q * 2.0 ** -31)
        err = float((y[t].double() - ystar[t]).abs().max())
        assert err <= bar, (t, err, bar)


def head_zero():
    """every workspace the library holds is zero in its head"""
    from vptq_b200 import native
    torch.cuda.synchronize()
    bufs = list(native._workspaces.values()) + list(native._retired) + list(native._captured.values())
    assert bufs
    for ws in bufs:
        assert int(ws[:min(ZERO_HEAD, ws.numel())].count_nonzero()) == 0


# ------------------------------------------------------------------------------------------------------------------
# layers built on the GPU, checked on a sample of index rows
# ------------------------------------------------------------------------------------------------------------------
def _np16(t, dtype):
    t = t.detach().cpu().contiguous()
    return t.numpy() if dtype == "fp16" else t.view(torch.int16).numpy().view(np.uint16)


class GpuLayer:
    """A seeded layer (v = 8, one group) generated and packed on the GPU, with its list-carrying descriptor.
    `oracle(rows)` is the oracle Layer of index rows `rows` only: the reference for layers too large for a dense
    fp64 weight."""

    def __init__(self, I, O, *, K=65536, Kr=256, dtype="fp16", perm=True, norm=True, bias=False, seed=0):
        from vptq_b200.pack import pack_index
        self.I, self.O, self.K, self.Kr, self.dtype = I, O, K, Kr, dtype
        self.Ro = (O + 7) // 8
        dt = torch.float16 if dtype == "fp16" else torch.bfloat16
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
        idx = torch.randint(0, K, (1, self.Ro, I), device="cuda", generator=g)
        ridx = torch.randint(0, Kr, (1, self.Ro, I), device="cuda", generator=g) if Kr > 0 else None
        t = dict(indices=pack_index(idx, K.bit_length() - 1, ridx, Kr.bit_length() - 1 if Kr > 0 else 0))
        del idx, ridx
        t["centroids"] = (0.02 * rnd(1, K * 8)).to(dt)
        t["res_centroids"] = (0.005 * rnd(1, Kr * 8)).to(dt) if Kr > 0 else None
        t["perm"] = torch.randperm(I, device="cuda", generator=g).to(torch.int32).to(torch.int16) if perm else None
        t["weight_scale"] = (1.0 + 0.1 * rnd(I)).to(dt) if norm else None
        t["weight_bias"] = (0.01 * rnd(I)).to(dt) if norm else None
        t["bias"] = (0.1 * rnd(O)).to(dt) if bias else None
        self.t = t
        self.desc = desc_from_tensors(t, dtype, I, O, K, Kr if Kr > 0 else -1)

    def sample(self, n, seed=0):
        """sorted seeded sample of n index rows (all rows when there are at most n), always the last one"""
        if self.Ro <= n:
            return np.arange(self.Ro)
        rows = np.random.default_rng(seed).choice(self.Ro - 1, size=n - 1, replace=False)
        return np.sort(np.append(rows, self.Ro - 1))

    def oracle(self, rows):
        """(oracle Layer of index rows `rows`, the output columns of the full layer its rows hold, which of those are
        real outputs: the last index row may be padding past out_features)"""
        t, dt = self.t, self.dtype
        rows = np.asarray(rows)
        cols = (rows[:, None] * 8 + np.arange(8)[None, :]).reshape(-1)
        keep = cols < self.O
        L = vo.Layer(dtype=dt, in_features=self.I, out_features=len(rows) * 8, vector_len=8, num_centroids=self.K,
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

    def check(self, x, y, rows, factor_exact=True):
        """y [tokens, O] within the bar of the kernel's arithmetic on `rows`, twice that against the exact product"""
        L, cols, keep = self.oracle(rows)
        kstar = kernel_star(L, x)[:, torch.from_numpy(np.nonzero(keep)[0]).cuda()]
        ys = y[:, torch.from_numpy(cols[keep]).cuda()]
        q = q_of(self.I, self.K)
        assert torch.isfinite(ys).all()
        assert_close(ys, kstar, self.dtype, q)
        if factor_exact:
            import _extreme as ex
            exact = ex.y_star(L, x)[:, torch.from_numpy(np.nonzero(keep)[0]).cuda()]
            assert_close(ys, exact, self.dtype, q, factor=2.0)


def rand_x(tokens, I, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(tokens, I, device="cuda", generator=g).to(torch.float16 if dtype == "fp16" else torch.bfloat16)
