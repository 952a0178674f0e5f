"""Helpers for the envelope tests of the dense weight from the index lists (csrc/lists_dense.cu, its GEMM glue
lists_gemm_launch in csrc/gemm_wgmma.cu, C interface include/vptq_b200_lists_dense.h).

* `deal(...)`: an integer mirror of how lists_dense_kernel deals the steps of one (index row, column tile) CTA to its
  warps -- which warp, iteration and unroll slot take which step of which unit, which slice the kernel's linear search
  over s_first finds, which lanes are masked -- and `deal_stats` / `slot_of` on top of it.  Used by the CPU file on
  lists built on the host and by the GPU file on the lists of every descriptor it checks.
* `writer_weight(...)`: W [O, I] as the writer computes it from the lists (fp32 C + R, one fmaf with scale and
  weight_bias, rounded to the 16-bit type), in numpy.
* `DenseLayer`: a seeded layer of vector length 8 or 16 generated on the GPU (any index pattern), with list-carrying
  descriptors in fp16 and bf16 that share one set of lists, and `check_weight`: the bit bar of W and Wt against the
  packed dequant.
"""
import numpy as np
import torch

import vptq_oracle as vo

DENSE, GEMM, STAGE = "lists_dense_kernel", "gemm_tn_wgmma", "dgrad_stage_dy"
WARPS, UNROLL = 8, 8                  # LD_WARPS, LD_UNROLL of csrc/lists_dense.cu
STEP_MASK = (1 << 26) - 1
SENTINEL = 0x7A5A                     # a finite 16-bit pattern in both types
SM_COUNT = 132                        # H100 SXM: which (NS, in_features) pairs get lists (NS * NT <= SM count)


# ------------------------------------------------------------------------------------------------------------------
# integer mirror of the writer
# ------------------------------------------------------------------------------------------------------------------
def units(tab, NS, NT, Ro):
    """tab (uint32 words) -> (step0, nsteps, valid) of every unit, each [NT, NS, Ro] (unit u = (t NS + s) Ro + r)"""
    tb = np.asarray(tab).astype(np.int64) & 0xFFFFFFFF
    U = NS * NT * Ro
    first = tb & STEP_MASK
    shape = (NT, NS, Ro)
    return first[:U].reshape(shape), (first[1:] - first[:-1]).reshape(shape), (tb[:U] >> 26).reshape(shape)


def deal(tab, NS, NT, Ro):
    """Every step the kernel deals, as flat arrays over all CTAs (r, t):
    r, t, g (step of the CTA's concatenation), warp, it (loop iteration), i (unroll slot), s (slice the kernel's search
    finds), k (step inside that unit), row (stream step it reads), nvalid (lanes the mask lets through), last (k is the
    unit's last step).  Asserts that the search finds the unit each step belongs to."""
    step0, nsteps, valid = units(tab, NS, NT, Ro)
    s_first = np.concatenate([np.zeros((NT, 1, Ro), np.int64), np.cumsum(nsteps, axis=1)], axis=1)  # [NT, NS+1, Ro]
    # one record per step, in unit order: its (t, s, r) and its place inside the unit
    n = nsteps.reshape(-1)
    tt, ss, rr = (a.reshape(-1).repeat(n) for a in np.meshgrid(np.arange(NT), np.arange(NS), np.arange(Ro),
                                                                    indexing="ij"))
    kk = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
    g = s_first[tt, ss, rr] + kk
    # the kernel: s = 0; while (s + 1 < NS && s_first[s + 1] <= g) ++s   (s_first increases: every unit has a step)
    s = np.zeros_like(g)
    for c in range(1, NS):
        s += s_first[tt, c, rr] <= g
    assert np.array_equal(s, ss), "the search over s_first lands in another unit"
    k = g - s_first[tt, s, rr]
    last = k + 1 == nsteps[tt, s, rr]
    nvalid = np.where(last, valid[tt, s, rr], 32)
    return dict(r=rr, t=tt, g=g, warp=g % WARPS, it=g // (WARPS * UNROLL), i=(g // WARPS) % UNROLL, s=s, k=k,
                row=step0[tt, s, rr] + k, nvalid=nvalid, last=last, total=s_first[:, NS, :])


def deal_stats(tab, NS, NT, Ro):
    """The list shapes one layer's lists put in front of the writer: longest unit (steps), number of 1-step empty
    units, and the largest number of units the 8 steps of one warp's iteration come from."""
    _, nsteps, valid = units(tab, NS, NT, Ro)
    d = deal(tab, NS, NT, Ro)
    cta = d["t"] * Ro + d["r"]
    key = (cta * (int(d["it"].max()) + 1) + d["it"]) * WARPS + d["warp"]           # one warp's iteration
    pairs = np.unique(key * NS + d["s"])
    _, crossed = np.unique(pairs // NS, return_counts=True)
    return dict(longest=int(nsteps.max()), empty=int(((nsteps == 1) & (valid == 0)).sum()),
                max_units_per_deal=int(crossed.max()))


def slot_of(col):
    """shared-memory slot (16 bytes) of tile column `col` in a [TCW][8] plane: the writer's XOR swizzle"""
    col = np.asarray(col)
    return col ^ ((col >> 3) & 7)


def read_slot(j, k):
    """slot thread j reads for feature 8 j + k of its 8 consecutive features"""
    return 8 * np.asarray(j) + (np.asarray(k) ^ (np.asarray(j) & 7))


# ------------------------------------------------------------------------------------------------------------------
# the writer's arithmetic
# ------------------------------------------------------------------------------------------------------------------
def writer_weight(L, stream, tab):
    """W [O, I] (float32 values of the layer's 16-bit type) that lists_dense_kernel writes for oracle layer L from its
    lists: c = fp32(C) + fp32(R) rounded to fp32, w = fmaf(c, scale[f], weight_bias[f]) (scale 1, bias 0 without a
    norm), rounded to the 16-bit type.  The fma is evaluated in float64 and asserted exact there before its one
    rounding to fp32."""
    from vptq_b200.lists import geometry
    v, I, O, K, Kr = L.vector_len, L.in_features, L.out_features, L.num_centroids, L.num_res_centroids
    Ro = (O + v - 1) // v
    NS, NT, TCW = geometry(I, K)
    words = np.asarray(stream).reshape(-1, 32).astype(np.int64) & 0xFFFFFFFF
    d = deal(tab, NS, NT, Ro)
    lane = np.arange(32)[None, :]
    live = lane < d["nvalid"][:, None]
    e = words[d["row"]][live]
    r = np.broadcast_to(d["r"][:, None], live.shape)[live]
    f = np.broadcast_to(d["t"][:, None], live.shape)[live] * TCW + ((e >> 12) & 4095)
    s = np.broadcast_to(d["s"][:, None], live.shape)[live]
    C = vo.to_f32(L.centroids, L.dtype).reshape(K, v)[s * 4096 + (e & 4095)]                  # [n, v]
    c = C + vo.to_f32(L.res_centroids, L.dtype).reshape(Kr, v)[e >> 24] if Kr > 0 else C       # fp32 add
    c = c.astype(np.float32)
    if L.weight_scale is not None:
        sc = vo.to_f32(L.weight_scale, L.dtype)[f].astype(np.float64)[:, None]
        wb = vo.to_f32(L.weight_bias, L.dtype)[f].astype(np.float64)[:, None]
        p = c.astype(np.float64) * sc                                                        # exact: 24 + 11 bits
        w64 = p + wb
        assert np.array_equal(w64 - p, np.broadcast_to(wb, w64.shape)) and np.array_equal(w64 - wb, p), \
            "the float64 sum is not exact for this layer"
        c = w64.astype(np.float32)
    W = np.full((Ro * v, I), np.nan, np.float32)
    W[(r[:, None] * v + np.arange(v)[None, :]).reshape(-1), np.repeat(f, v)] = c.reshape(-1)
    return vo.round_to(W[:O], L.dtype)


# ------------------------------------------------------------------------------------------------------------------
# layers generated on the GPU, any index pattern
# ------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int16)


def dt_of(dtype):
    return torch.float16 if dtype == "fp16" else torch.bfloat16


class DenseLayer:
    """A seeded one-group layer of vector length v on the GPU: main indices of `_envelope.pattern` `kind`, residual
    indices uniform or all ones (`res_kind`), Kr <= 0 for no residual codebook.  `desc(dtype)` is its list-carrying
    descriptor with the layer's codebooks in that type; both types share the lists built for the first."""

    def __init__(self, v, I, O, *, K=65536, Kr=256, kind="uniform", res_kind="uniform", perm=True, norm=True,
                 bias=False, seed=0):
        from vptq_b200.pack import pack_index
        from _envelope import pattern
        self.v, self.I, self.O, self.K, self.Kr = v, I, O, K, Kr
        self.Ro = (O + v - 1) // v
        self.perm_np = np.random.default_rng(seed).permutation(I) if perm else None
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
        shape = (1, self.Ro, I)
        if kind == "uniform":
            idx = torch.randint(0, K, shape, device="cuda", generator=g)
        else:
            idx = torch.from_numpy(pattern(kind, K, shape, np.random.default_rng(seed + 1), perm=self.perm_np)).cuda()
        ridx = None
        if Kr > 0:
            ridx = torch.full(shape, Kr - 1, device="cuda") if res_kind == "ones" else \
                torch.randint(0, Kr, shape, device="cuda", generator=g)
        self.packed = pack_index(idx, K.bit_length() - 1, ridx, Kr.bit_length() - 1 if Kr > 0 else 0)
        del idx, ridx
        self.f32 = dict(centroids=0.02 * rnd(1, K * v), res_centroids=0.005 * rnd(1, Kr * v) if Kr > 0 else None,
                        weight_scale=1.0 + 0.1 * rnd(I) if norm else None,
                        weight_bias=0.01 * rnd(I) if norm else None, bias=0.1 * rnd(O) if bias else None)
        self.perm = None if self.perm_np is None else \
            torch.from_numpy(self.perm_np.astype(np.int32)).to(torch.int16).cuda()
        self._descs = {}

    def desc(self, dtype):
        from _lists16 import desc_t
        from _batch import desc_from_tensors
        if dtype in self._descs:
            return self._descs[dtype]
        t = {k: (None if a is None else a.to(dt_of(dtype))) for k, a in self.f32.items()}
        t.update(indices=self.packed, perm=self.perm)
        first = next(iter(self._descs.values()), None)
        Kr = self.Kr if self.Kr > 0 else -1
        if self.v == 8:
            d = desc_from_tensors(t, dtype, self.I, self.O, self.K, Kr, lists=first is None)
        else:
            d = desc_t(t, dtype, self.I, self.O, self.K, Kr, lists16=first is None)
        if first is not None:
            d.lists_stream, d.lists_tab, d.lists_tile_cols = first.lists_stream, first.lists_tab, first.lists_tile_cols
            d._lists_of = first
        assert d.lists_stream, "no lists were built for this layer"
        self._descs[dtype] = d
        return d

    def lists(self):
        """(stream, tab) of the layer's lists as uint32 numpy arrays"""
        d = next(iter(self._descs.values()))
        stream, tab = d._keep[-2:]
        return stream.cpu().numpy().view(np.uint32), tab.cpu().numpy().view(np.uint32)


def packed_w(d, dt):
    from vptq_b200 import native
    w = torch.empty(d.out_features, d.in_features, dtype=dt, device="cuda")
    native.dequant(d, w)
    return w


def assert_route(names, gemm=True):
    """lists_dense_kernel ran (and the GEMM, if `gemm`), no kernel that dequantises the packed words"""
    from _probe import ran
    assert ran(names, DENSE) and ran(names, GEMM) == gemm, names
    assert not any("dequant" in n for n in names), names


def check_weight(d, dt, lds=(0, 8, 16)):
    """The bit bar: W and Wt written from the lists into sentinel-filled buffers at pitch min + extra (extra in
    `lds`) are bit-identical to the packed dequant, their padding columns are zero and nothing past the view changed;
    the input-gradient GEMM on the lists with dY = identity returns what the packed input gradient does."""
    from vptq_b200 import native
    from _probe import launched_kernels
    I, O = d.in_features, d.out_features
    w_ref = _bits(packed_w(d, dt))
    eye = torch.eye(O, dtype=dt, device="cuda")
    dx_p = torch.empty(O, I, dtype=dt, device="cuda")
    native.quant_gemm_dgrad(d, eye, dx_p)
    out = []

    def lists_side():
        out.clear()
        for extra in lds:
            for tr, rows, cols in ((0, O, I), (native.FLAG_TRANSPOSE, I, O)):
                ld = (cols + 7) // 8 * 8 + extra
                buf = torch.full(((rows + 1) * ld + 64,), SENTINEL, dtype=torch.int16, device="cuda")
                native.lists_dequant(d, buf.view(dt), ld, tr)
                out.append((tr, rows, cols, ld, buf))
        dx = torch.empty(O, I, dtype=dt, device="cuda")
        native.lists_quant_gemm(d, eye, dx, native.FLAG_TRANSPOSE)
        out.append(dx)

    assert_route(launched_kernels(lists_side))
    for tr, rows, cols, ld, buf in out[:-1]:
        view = buf[:rows * ld].view(rows, ld)
        want = w_ref.t() if tr else w_ref
        assert torch.equal(view[:, :cols], want), (tr, ld, int((view[:, :cols] != want).sum()))
        assert not view[:, cols:].any(), (tr, ld)
        assert bool((buf[rows * ld:] == SENTINEL).all()), (tr, ld)
    assert torch.equal(_bits(out[-1]), _bits(dx_p))
