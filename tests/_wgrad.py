"""Weight-gradient oracle for the tests: dC, dR, dCol, d weight_scale and d weight_bias of one layer in fp64.

Given G[o][f] = dL/dW[o][f] (W = `vptq_oracle.dequant(L)`, original feature order) the gradients are those of
include/vptq_b200_grad.h:
  dC_g[k][e]   = sum of s_f G[o][f] over the (r, c) of group g with main index k, o = v r + e < O
  dR_g[kr][e]  = the same over residual index kr
  dCol[oi][eo] = the same over outlier columns, vector length vol
  d weight_scale[f] = sum_o G[o][f] Wq[o][f],   d weight_bias[f] = sum_o G[o][f]
For `quant_gemm`, G = dY^T x.  Gradients come back in the shapes of the layer arrays (centroids [G, K*v], ...),
float64; only the tensors the layer has are present.
"""
import copy

import numpy as np

import vptq_oracle as vo


def wq_original_order(L: vo.Layer) -> np.ndarray:
    """Wq [O, I] (C + R, or the outlier codebook) in original feature order, no scale / bias, fp64."""
    Lq = copy.copy(L)
    Lq.weight_scale = Lq.weight_bias = None
    return vo.dequant(Lq, out_dtype=np.float64)


def grads_from_gamma(gamma: np.ndarray, L: vo.Layer) -> dict:
    """gamma [O, I] (float, original feature order) -> {name: gradient}."""
    gamma = np.asarray(gamma, dtype=np.float64)
    O, I, v, G, gs = L.out_features, L.in_features, L.vector_len, L.num_codebooks, L.group_size
    K, Kr = L.num_centroids, L.num_res_centroids
    S = L.outlier_size if L.enable_outlier else 0
    perm = np.arange(I) if L.perm is None else np.asarray(L.perm).astype(np.uint16).astype(np.int64)
    s = np.ones(I) if L.weight_scale is None else vo.to_f32(L.weight_scale, L.dtype).astype(np.float64)
    out = {}
    if L.weight_scale is not None:
        out["weight_bias"] = gamma.sum(0)
        out["weight_scale"] = (gamma * wq_original_order(L)).sum(0)
    sg = gamma[:, perm] * s[perm][None, :]          # s_f G[o][f] in quantised column order c
    idx, ridx = vo.unpack_index(L.indices, L.index_bits, gs, L.res_bits)   # [G, Ro, gs]
    Ro = idx.shape[1]
    pad = np.zeros((Ro * v, I))
    pad[:O] = sg
    dC = np.zeros((G, K, v))
    dR = np.zeros((G, max(Kr, 1), v))
    for g in range(G):
        t = pad[:, S + g * gs:S + (g + 1) * gs].reshape(Ro, v, gs).transpose(0, 2, 1)   # [Ro, gs, v]
        np.add.at(dC[g], idx[g], t)
        if L.res_bits:
            np.add.at(dR[g], ridx[g], t)
    out["centroids"] = dC.reshape(G, K * v)
    if L.res_bits:
        out["res_centroids"] = dR.reshape(G, Kr * v)
    if S:
        vol, Kol = L.outlier_vector_len, L.num_outlier_centroids
        oidx = np.asarray(L.outlier_indices).astype(np.uint16).astype(np.int64).reshape(-1, S)   # [Rol, S]
        Rol = oidx.shape[0]
        po = np.zeros((Rol * vol, S))
        po[:O] = sg[:, :S]
        dCol = np.zeros((Kol, vol))
        np.add.at(dCol, oidx, po.reshape(Rol, vol, S).transpose(0, 2, 1))
        out["outlier_centroids"] = dCol.reshape(1, Kol * vol)
    return out


def gamma_from_x_dy(x: np.ndarray, dy: np.ndarray, L: vo.Layer) -> np.ndarray:
    """G = dY^T x in fp64 from 16-bit x [T, I] and dY [T, O] (fp16 values, or bf16 bit patterns)."""
    xf = vo.to_f32(x, L.dtype).astype(np.float64).reshape(-1, L.in_features)
    dyf = vo.to_f32(dy, L.dtype).astype(np.float64).reshape(-1, L.out_features)
    return dyf.T @ xf


def quant_gemm_wgrad(x: np.ndarray, dy: np.ndarray, L: vo.Layer) -> dict:
    return grads_from_gamma(gamma_from_x_dy(x, dy, L), L)
