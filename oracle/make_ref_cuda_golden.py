"""Record what the reference's own CUDA kernels return for the cases of tests/test_gpu_vs_ref_cuda.py.

    python oracle/make_ref_cuda_golden.py OUT.npz      (needs a GPU and oracle/_ref/libvptq.so, see build_ref.sh)

The layers, activations and sample positions are regenerated from their seeds, so only the reference outputs are
stored, as raw 16-bit words: y of quant_gemv for 1 and 2 tokens, and a fixed, seeded sample of the dequantised
weight (the full matrices are megabytes).  The file goes to tests/golden/ref_cuda/, and the test compares our kernels with it.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import vptq_oracle as vo  # noqa: E402
from _gpu import from_t, make_module, x_to_t  # noqa: E402
from test_gpu_vs_ref_cuda import (CASES, DEQUANT_CASES, DEQUANT_SEED, GEMV_SEED, ref_tensors, sample_positions,  # noqa: E402
                                   to_bits)


def main(out):
    spec = importlib.util.spec_from_file_location("libvptq", os.path.join(ROOT, "oracle", "_ref", "libvptq.so"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    z = {}
    for name in sorted(CASES):
        L = vo.make_layer(seed=GEMV_SEED, **CASES[name])
        m = make_module(L)
        cent, rcent, ocent = ref_tensors(L, m)
        for tokens in (1, 2):
            x = x_to_t(vo.make_x(tokens, L.in_features, L.dtype, seed=tokens), L)
            y = ref.quant_gemv(x, m.indices, cent, None, rcent, m.outlier_indices, ocent, m.perm, m.weight_scale,
                               m.weight_bias, m.bias, L.in_features, L.out_features)
            z[f"gemv__{name}__t{tokens}"] = to_bits(from_t(y), L.dtype)
    for name in DEQUANT_CASES:
        L = vo.make_layer(seed=DEQUANT_SEED, **CASES[name])
        m = make_module(L)
        cent, rcent, ocent = ref_tensors(L, m)
        inv = torch.argsort(m.perm.view(torch.uint16).to(torch.int64)).to(torch.uint16).view(torch.int16)
        W = from_t(ref.dequant(m.indices, cent, None, rcent, m.outlier_indices, ocent, inv, m.weight_scale,
                               m.weight_bias, L.vector_len, L.in_features, L.out_features))
        z[f"dequant__{name}__shape"] = np.array(W.shape, dtype=np.int64)
        z[f"dequant__{name}__values"] = to_bits(W.reshape(-1)[sample_positions(W.size)], L.dtype)
    torch.cuda.synchronize()
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **z)
    print(f"wrote {out}: {len(z)} arrays")


if __name__ == "__main__":
    main(sys.argv[1])
