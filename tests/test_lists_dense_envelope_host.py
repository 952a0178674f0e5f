"""Host-side envelope of the dense weight from the index lists (csrc/lists_dense.cu): an integer mirror of the writer's
deal on the lists of every index pattern and shape tests/test_gpu_lists_dense_envelope.py runs, the arithmetic its
probe test assumes, and refusals at the edge shapes.

* the deal (tests/_lists_dense.py `deal`): for every (index row, column tile) CTA the kernel's linear search over
  s_first finds the unit each step belongs to, the mask lets through exactly the unit's valid lanes, and with the XOR
  swizzle every feature of the tile goes to one plane slot, written once, which the store phase reads back as that
  feature.  Every (output row, feature) of W and of Wt, zero columns included, is written exactly once at every pitch
  the GPU file uses, and nothing at or past the pitch;
* the probes: W as the writer computes it from the lists is what `_probe.probe_expect(L, "direct")` simulates, so the
  GPU probe test holds lists_quant_gemm to that simulation bit for bit;
* refusals with nothing launched at the new edge shapes (v = 16 with a partial last index row, in_features 65535).
"""
import ctypes

import numpy as np
import pytest
import torch

import _envelope as env
import vptq_oracle as vo
from _lists_dense import deal, deal_stats, read_slot, slot_of, units, writer_weight
from _probe import probe_expect
from vptq_b200 import lists

# the GPU file's shapes: index data at 4096 x 4096 (v = 8) and 4096 x 1024 (v = 16), slices x widths, out_features,
# perm on and off
INDEX = [(v, kind, K) for v in (8, 16) for kind in env.PATTERNS for K in (8192, 65536)]
WIDTHS = (4096, 4100, 9004, 65528, 65535)
NS_I = [(ns, I) for ns in (2, 4, 8, 16) for I in WIDTHS if ns * lists.geometry(I, 4096 * ns)[1] <= 132]
OUTS = {8: (1, 3, 8, 9, 1003, 1004), 16: (8, 9, 15, 16, 17, 1000)}
SKEWED = ("ones", "row_slice", "constant", "ramp")


def _lists(v, I, O, K, kind="uniform", perm=True, seed=0):
    from vptq_b200.pack import pack_index
    Ro = (O + v - 1) // v
    rng = np.random.default_rng(seed)
    p = rng.permutation(I) if perm else None
    idx = env.pattern(kind, K, (1, Ro, I), rng, perm=p)
    ridx = rng.integers(0, 256, size=(1, Ro, I))
    packed = pack_index(torch.from_numpy(idx), K.bit_length() - 1, torch.from_numpy(ridx), 8)
    pt = None if p is None else torch.from_numpy(p.astype(np.int32)).to(torch.int16)
    stream, tab, tcw = lists.build_lists(packed, num_centroids=K, num_res_centroids=256, in_features=I,
                                         out_features=O, perm=pt, deal=True, vector_len=v)
    assert tcw == lists.geometry(I, K)[2]
    return stream.numpy().view(np.uint32).reshape(-1, 32), tab.numpy().view(np.uint32), idx[0], p


def _mirror(v, I, O, K, stream, tab, idx, p):
    """the writer's deal on these lists: every entry lands once, at the slot and output its fields name"""
    NS, NT, TCW = lists.geometry(I, K)
    Ro = (O + v - 1) // v
    d = deal(tab, NS, NT, Ro)
    _, nsteps, valid = units(tab, NS, NT, Ro)
    assert (valid <= 32).all() and (nsteps >= 1).all()
    # the steps of a CTA are dealt round-robin: warp g % 8, 8 in flight per iteration, every step once
    cta = d["t"] * Ro + d["r"]
    assert np.array_equal(np.sort(cta * (1 << 24) + d["g"]),
                          np.sort(np.concatenate([c * (1 << 24) + np.arange(n) for c, n in
                                                  enumerate(d["total"].reshape(-1))])))
    lane = np.arange(32)[None, :]
    live = lane < d["nvalid"][:, None]
    assert not stream[d["row"]][~live].any()                # masked lanes hold padding words only
    e = stream[d["row"]][live].astype(np.int64)
    r = np.broadcast_to(d["r"][:, None], live.shape)[live]
    t = np.broadcast_to(d["t"][:, None], live.shape)[live]
    s = np.broadcast_to(d["s"][:, None], live.shape)[live]
    col = (e >> 12) & 4095
    ncols = np.minimum(TCW, I - t * TCW)
    assert (col < ncols).all()
    # original order: plane slot of (CTA, column), once each; the store phase reads slot read_slot(j, k) as feature
    # 8 j + k of the tile -- the slot that feature's entry wrote
    slot = (r * NT + t) * TCW + slot_of(col)
    assert np.unique(slot).size == slot.size == Ro * I
    c = np.arange(TCW)
    assert np.array_equal(read_slot(c // 8, c % 8), slot_of(c))
    # and the entry carries the packed field of (index row, feature)
    f = t * TCW + col
    inv = np.arange(I) if p is None else np.argsort(p)
    assert np.array_equal((e & 4095) + 4096 * s, idx[r, inv[f]])
    return d


def _stores(v, I, O, TCW, ld, transposed):
    """how many times the store phase writes every element of the [rows][ld] buffer (the entries' features covered,
    from the plane check): W rows o < min(V, O - o0) per index row, zero columns [I, ld) from the last tile's CTAs;
    Wt halves o0 + 8 h below ld per feature, the zero tail from the CTAs of index rows Ro .. ceil(ld / V) - 1"""
    Ro, NT = (O + v - 1) // v, (I + TCW - 1) // TCW
    if transposed:
        n = np.zeros(ld + 16, np.int64)
        for r in range((ld + v - 1) // v):
            for h in range(v // 8):
                if v > 8 and r * v + 8 * h >= ld:
                    break
                n[r * v + 8 * h:r * v + 8 * h + 8] += 1
        return np.broadcast_to(n, (I, ld + 16))
    n = np.zeros((Ro * v, ld + 16), np.int64)
    for r in range(Ro):
        rows = min(v, O - r * v)
        for t in range(NT):
            f0, nc = t * TCW, min(TCW, I - t * TCW)
            n[r * v:r * v + rows, f0:f0 + nc] += 1
            if f0 + nc == I:
                n[r * v:r * v + rows, I:ld] += 1
    return n


def _check_stores(v, I, O, K):
    TCW = lists.geometry(I, K)[2]
    for extra in (0, 8, 16):
        for tr, rows, cols in ((False, O, I), (True, I, O)):
            ld = (cols + 7) // 8 * 8 + extra
            n = _stores(v, I, O, TCW, ld, tr)
            assert (n[:rows, :ld] == 1).all() and not n[:, ld:].any() and not n[rows:].any(), (tr, ld)


@pytest.mark.parametrize("v,kind,K", INDEX)
def test_deal_mirror_on_every_index_pattern(v, kind, K):
    I, O = 4096, 4096 if v == 8 else 1024
    stream, tab, idx, p = _lists(v, I, O, K, kind, seed=K + v)
    _mirror(v, I, O, K, stream, tab, idx, p)
    NS, NT, _ = lists.geometry(I, K)
    st = deal_stats(tab, NS, NT, (O + v - 1) // v)
    if kind in SKEWED:     # one unit of a whole tile's steps next to 1-step empty ones
        assert st["longest"] >= 64 and st["empty"] > 0, st
    if kind == "uniform":
        assert st["empty"] == 0, st


@pytest.mark.parametrize("v", [8, 16])
@pytest.mark.parametrize("ns,I", NS_I)
def test_deal_mirror_across_slices_and_widths(ns, I, v):
    O = 24 if v == 8 else 40
    stream, tab, idx, p = _lists(v, I, O, 4096 * ns, seed=ns * 7 + I)
    _mirror(v, I, O, 4096 * ns, stream, tab, idx, p)
    _check_stores(v, I, O, 4096 * ns)


@pytest.mark.parametrize("perm", [True, False])
@pytest.mark.parametrize("v,O", [(v, o) for v in OUTS for o in OUTS[v]])
def test_deal_mirror_across_out_features(v, O, perm):
    stream, tab, idx, p = _lists(v, 4100, O, 65536, perm=perm, seed=O)
    _mirror(v, 4100, O, 65536, stream, tab, idx, p)
    _check_stores(v, 4100, O, 65536)


def test_ns_i_grid_follows_the_sm_count():
    """at in_features >= 61441 a layer has 16 column tiles, so 16 slices (256 combos) get no lists"""
    assert (16, 65528) not in NS_I and (16, 65535) not in NS_I and (8, 65535) in NS_I
    assert lists.geometry(65535, 65536)[1:] == (16, 4096) and 65535 - 15 * 4096 == 4095


# ---------------------------------------------------------------- the probe test's simulation
PROBE = {8: dict(in_features=1024, out_features=264), 16: dict(in_features=1024, out_features=272)}


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("kind", ["uniform", "zipf_hot0"])
@pytest.mark.parametrize("v", [8, 16])
def test_probe_expect_direct_is_the_writer_arithmetic(v, kind, dtype):
    """y = x . W^T + bias with x = e_f: the fp32 accumulator holds W[o][f] exactly (every other product is zero), the
    epilogue adds the bias in fp32 and rounds once -- rn16(W16 + bias), where W16 is the writer's weight.  That is
    probe_expect's "direct" route; Wt (the transposed writer, same arithmetic) gives it without the bias."""
    L = env.layer_with(kind, vector_len=v, num_centroids=65536, num_res_centroids=256, bias=True, dtype=dtype,
                       seed=300 + v, **PROBE[v])
    stream, tab, _ = lists.build_lists(torch.from_numpy(np.asarray(L.indices, np.int32)), num_centroids=65536,
                                       num_res_centroids=256, in_features=L.in_features, out_features=L.out_features,
                                       perm=torch.from_numpy(np.asarray(L.perm).astype(np.uint16).view(np.int16)),
                                       deal=True, vector_len=v)
    W16 = writer_weight(L, stream.numpy().view(np.uint32), tab.numpy().view(np.uint32))   # [O, I]
    y = vo.round_to(W16 + vo.to_f32(L.bias, dtype)[:, None], dtype)
    expect = probe_expect(L, "direct")                                                     # [I, O]
    assert np.array_equal(y.T.view(np.uint32), expect.view(np.uint32))
    import _extreme as ex
    P = ex.copy_layer(L)
    P.bias = None
    assert np.array_equal(W16.T.view(np.uint32), probe_expect(P, "direct").view(np.uint32))


# ---------------------------------------------------------------- refusals at the edge shapes
def _desc(**over):
    from vptq_b200 import native
    d = native.LinearDesc()
    d.struct_size = ctypes.sizeof(native.LinearDesc)
    # decode-only, fake addresses never dereferenced: every call below is refused before anything is launched
    base = dict(dtype=0, in_features=65535, out_features=9, vector_len=16, num_centroids=32768,
                num_res_centroids=256, num_codebooks=1, group_size=65535, outlier_size=0, outlier_vector_len=-1,
                num_outlier_centroids=-1, indices=None, index_stride_codebook=0, index_stride_row=0,
                centroids=0x20000, centroid_stride=32768 * 16, res_centroids=0x30000, res_centroid_stride=4096,
                lists_stream=0x40000, lists_tab=0x50000, lists_tile_cols=4096)
    base.update(over)
    for k, v in base.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("v,I,O", [(16, 65535, 9), (16, 4100, 17), (8, 65535, 3), (8, 9004, 1)])
def test_refusals_at_edge_shapes(v, I, O):
    from vptq_b200 import native
    L = native.lib()
    T = native.FLAG_TRANSPOSE
    d = _desc(vector_len=v, in_features=I, group_size=I, out_features=O, centroid_stride=32768 * v,
              res_centroid_stride=256 * v, lists_tile_cols=lists.geometry(I, 32768)[2])
    deq, gemm = L.vptq_b200_lists_dequant, L.vptq_b200_lists_quant_gemm
    for flags, cols in ((0, I), (T, O)):
        lo = (cols + 7) // 8 * 8
        for ld in (lo + 4, cols - 1):                                      # ld % 8 != 0, ld < cols
            assert deq(ctypes.byref(d), 0x1000, ld, flags, None) == -1, (flags, ld)
            assert "ld" in native.last_error()
        for w in (0x1002, 0x1008):                                         # w not 16-byte aligned
            assert deq(ctypes.byref(d), w, lo, flags, None) == -1
        xc, yc = (I, O) if flags == 0 else (O, I)
        for xs, ys, tokens in ((xc - 1, yc, 4), (xc, yc - 1, 4), (xc, yc, 0), (xc, yc, -3)):
            assert gemm(ctypes.byref(d), 0x1000, xs, 0x2000, ys, tokens, 0x3000, 1 << 40, flags, None) == -1
            assert "bad x/y/tokens/strides" in native.last_error()
