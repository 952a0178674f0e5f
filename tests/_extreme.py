"""Reference for the extreme-value tests: inf / NaN in any input or layer tensor, and magnitudes far from 1.

* `dense64(L)`: the layer's dense weight [O, I] in float64, from the oracle's own dequant (IEEE arithmetic:
  0 * inf = NaN, inf - inf = NaN).
* `ew_matmul(a, b)`: out[t, n] = sum_k a[t, k] * b[n, k] as an explicit element-wise product and sum in float64,
  in chunks of rows of b.  Not a matmul: BLAS does not promise IEEE behaviour for 0 * inf.
  `y_star(L, x)` = ew_matmul(x, W) + bias, `dgrad_star(L, dy)` = ew_matmul(dy, W^T).
* `isolate(L, main={k: rows}, res={k: rows})`: a copy of L whose main (residual) codebook entry k of group 0 is
  used exactly once in each index row of `rows` and nowhere else.
* `inject(L, site, value, ...)`: a copy of L with one value written into one of its tensors.
* `classify(y)`: every element -> FINITE / POS_INF / NEG_INF / NAN.
"""
import dataclasses

import numpy as np
import torch

import vptq_oracle as vo

FINITE, POS_INF, NEG_INF, NAN = 0, 1, 2, 3
VALUES = {"nan": float("nan"), "+inf": float("inf"), "-inf": float("-inf")}


def classify(y):
    """torch tensor -> int8 tensor of FINITE / POS_INF / NEG_INF / NAN, element-wise"""
    c = torch.zeros(y.shape, dtype=torch.int8, device=y.device)
    c[y == float("inf")] = POS_INF
    c[y == float("-inf")] = NEG_INF
    c[torch.isnan(y)] = NAN
    return c


def encode(a, dtype):
    """float values -> the layer's storage (fp16 array, or uint16 bf16 bit patterns)"""
    a = np.asarray(a, dtype=np.float32)
    return a.astype(np.float16) if dtype == "fp16" else vo.f32_to_bf16_bits(a)


def copy_layer(L):
    """deep copy of the arrays of L (the oracle Layer shares them otherwise)"""
    kw = {f.name: getattr(L, f.name) for f in dataclasses.fields(L)}
    kw = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    kw["meta"] = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in L.meta.items()}
    return vo.Layer(**kw)


def dense64(L):
    """W [O, I] float64 with whatever values L holds"""
    with np.errstate(invalid="ignore", over="ignore"):
        return vo.dequant(L, np.float64)


def bias64(L, device="cuda"):
    return None if L.bias is None else torch.from_numpy(vo.to_f32(L.bias, L.dtype).astype(np.float64)).to(device)


def ew_matmul(a, b, bias=None, budget=1 << 24):
    """a [T, K], b [N, K] (float64 torch, same device) -> [T, N]: sum_k a[t, k] * b[n, k] (+ bias[n]), computed as
    element-wise products and a sum, `budget` products at a time"""
    T, K = a.shape
    N = b.shape[0]
    out = torch.empty(T, N, dtype=torch.float64, device=a.device)
    step = max(1, budget // max(T * K, 1))
    for n0 in range(0, N, step):
        out[:, n0:n0 + step] = (a[:, None, :] * b[None, n0:n0 + step, :]).sum(-1)
    if bias is not None:
        out += bias[None, :]
    return out


def y_star(L, x, W=None):
    """x [T, I] (16-bit torch tensor) -> y* [T, O] float64 on x's device"""
    W = torch.from_numpy(dense64(L)).to(x.device) if W is None else W
    return ew_matmul(x.double(), W, bias64(L, x.device))


def dgrad_star(L, dy, W=None):
    """dy [T, O] (16-bit torch tensor) -> dX* = dy W [T, I] float64 on dy's device"""
    W = torch.from_numpy(dense64(L)).to(dy.device) if W is None else W
    return ew_matmul(dy.double(), W.t().contiguous())


def isolate(L, main=None, res=None):
    """Copy of L in which main-codebook entry k of group 0 (main = {k: rows}) is used exactly once in each index row
    of `rows` and nowhere else; likewise residual entry k (res = {k: rows}).  Every other use of k moves to a
    neighbouring entry that is not isolated.  The row sets must be disjoint."""
    L = copy_layer(L)
    idx, ridx = L.meta["idx"], L.meta.get("ridx")
    G, Ro, gs = idx.shape
    taken = {}
    for arr, spec, n in ((idx, main, L.num_centroids), (ridx, res, max(L.num_res_centroids, 0))):
        if not spec:
            continue
        keys = set(spec)
        for k in keys:
            repl = next(j % n for j in range(k + 1, k + n) if j % n not in keys)
            arr[0][arr[0] == k] = repl
        for k, rows in spec.items():
            for r in rows:
                assert taken.setdefault((arr is ridx, r), k) == k, "row sets must be disjoint"
                arr[0, r, isolated_column(L, r, k)] = k
    L.indices = vo.pack_index(idx, L.index_bits, ridx, L.res_bits)
    return L


def isolated_column(L, r, k):
    """the quantised column (of group 0) at which `isolate` places entry k in index row r"""
    return (r * 7919 + k * 31 + 5) % L.group_size


def feature_of(L, c):
    """original input feature of quantised column c (outlier columns come first, then group 0)"""
    c = c + (L.outlier_size if L.enable_outlier else 0)
    return int(np.asarray(L.perm).astype(np.uint16)[c]) if L.perm is not None else c


def rows_using(L, k, residual=False):
    """{index row: number of uses} of main (residual) entry k of group 0, decoded from the packed words"""
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, L.group_size, L.res_bits)
    a = (ridx if residual else idx)[0]
    rows, counts = np.unique(np.nonzero(a == k)[0], return_counts=True)
    return dict(zip(rows.tolist(), counts.tolist()))


def inject(L, site, value, k=0, e=0, f=0, o=0):
    """Copy of L with `value` written into one element:
      "C" / "R" / "Col": element e of main / residual / outlier codebook entry k (group 0)
      "scale" / "wbias": weight_scale[f] / weight_bias[f];  "bias": bias[o]"""
    L = copy_layer(L)
    v = encode([value], L.dtype)[0]
    if site == "C":
        L.centroids[0, k * L.vector_len + e] = v
    elif site == "R":
        L.res_centroids[0, k * L.vector_len + e] = v
    elif site == "Col":
        L.outlier_centroids[0, k * L.outlier_vector_len + e] = v
    elif site == "scale":
        L.weight_scale[f] = v
    elif site == "wbias":
        L.weight_bias[f] = v
    elif site == "bias":
        L.bias[o] = v
    else:
        raise ValueError(site)
    return L
