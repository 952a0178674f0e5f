"""Input-gradient oracle for the backward tests: dX* = dY @ W on the identical 16-bit tensors, fp64 accumulation.

W is `vptq_oracle.dequant(L)` (the reference's dense weight, [out_features, in_features]), so dX* is the gradient of
`vptq_oracle.quant_gemm` with respect to x -- what autograd through the reference's `dequant` + `F.linear` gives.
"""
import numpy as np

import vptq_oracle as vo


def quant_gemm_dgrad(dy: np.ndarray, L: vo.Layer, acc_dtype=np.float64) -> np.ndarray:
    """dy [..., out_features] (fp16 values, or bf16 bit patterns when L.dtype == 'bf16') -> dX [..., in_features]."""
    W = vo.dequant(L, out_dtype=np.float32).astype(acc_dtype)
    dyf = vo.to_f32(dy, L.dtype).astype(acc_dtype)
    dx = dyf.reshape(-1, L.out_features) @ W
    return dx.reshape(*dy.shape[:-1], L.in_features).astype(np.float32)
