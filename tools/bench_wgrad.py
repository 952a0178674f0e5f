"""Weight-gradient timing on the three Llama-3-8B layer shapes (K = 65536, Kr = 256, perm, norm), fp16:

  (a) ours   vptq_b200_quant_gemm_wgrad: dC, dR, d weight_scale, d weight_bias from x and dY, fused route (the GEMM
             epilogue reduces G); also the generic route (VPTQ_GRAD_FLAG_GENERIC: G in the workspace + scatter) and
             the kernel split of both, from the profiler in a separate run
  (b) cublas G = dY^T x alone (torch.matmul), the dense product every route has to form
  (c) torch  a differentiable gather-based dequant written from the formulas of include/vptq_b200_grad.h plus
             F.linear; autograd.grad on the recorded graph (backward only)

    python tools/bench_wgrad.py [--tokens 2048,8192] [--out FILE]

Prints one JSON object with the card name and power limit, read in the same process.  CUDA events, warm-ups.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
import torch

import vptq_oracle as vo
from _gpu import make_module
from vptq_b200 import native


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def torch_route(m, L):
    """Leaves (the layer's codebooks / scale / bias) and a function building W from them with gathers."""
    O, I, v, K, Kr = L.out_features, L.in_features, L.vector_len, L.num_centroids, L.num_res_centroids
    idx = torch.from_numpy(L.meta["idx"][0]).cuda()
    ridx = torch.from_numpy(L.meta["ridx"][0]).cuda()
    inv = torch.argsort(torch.from_numpy(np.asarray(L.perm).astype(np.int64)).cuda())
    leaves = [t.detach().clone().requires_grad_() for t in
              (m.centroids.weight, m.res_centroids.weight, m.weight_scale, m.weight_bias)]
    Ro = idx.shape[0]

    def weight():
        C, R, s, b = leaves
        wq = C.view(K, v)[idx] + R.view(Kr, v)[ridx]                     # [Ro, I, v]
        w = wq.permute(0, 2, 1).reshape(Ro * v, I)[:O]
        return w[:, inv] * s + b

    return leaves, weight


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="2048,8192")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"device": torch.cuda.get_device_name(), "power_limit": power_limit(), "dtype": "fp16", "rows": {}}
    for (i, o) in ((4096, 4096), (4096, 14336), (14336, 4096)):
        L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                          seed=1)
        m = make_module(L)
        m.prepare()
        desc = m._desc_cache[0]
        grads = {"centroids": torch.empty_like(m.centroids.weight),
                 "res_centroids": torch.empty_like(m.res_centroids.weight),
                 "weight_scale": torch.empty_like(m.weight_scale), "weight_bias": torch.empty_like(m.weight_bias)}
        leaves, weight = torch_route(m, L)
        for T in (int(t) for t in a.tokens.split(",")):
            x = torch.randn(T, i, device="cuda").half()
            dy = torch.randn(T, o, device="cuda").half()
            t_a = timeit(lambda: native.quant_gemm_wgrad(desc, x, dy, grads))
            t_gen = timeit(lambda: native.quant_gemm_wgrad(desc, x, dy, grads, flags=native.GRAD_FLAG_GENERIC))

            def split(flags):
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        native.quant_gemm_wgrad(desc, x, dy, grads, flags=flags)
                    torch.cuda.synchronize()
                share = {}
                for e in prof.key_averages():
                    k = next((n for n in ("gemm_tn_wgmma", "wg_scatter", "wg_transpose", "wg_row_stats") if n in e.key),
                             None)
                    if k:
                        share[k] = round(share.get(k, 0.0) + e.device_time_total / 5 / 1000, 4)
                return share
            t_b = timeit(lambda: torch.matmul(dy.t(), x))
            y = torch.nn.functional.linear(x, weight())
            t_c = timeit(lambda: torch.autograd.grad(y, leaves, dy, retain_graph=True))
            del y
            row = dict(a_ours_ms=round(t_a, 4), a_generic_route_ms=round(t_gen, 4), b_cublas_gamma_ms=round(t_b, 4),
                       c_torch_autograd_ms=round(t_c, 4), a_over_b=round(t_a / t_b, 3), a_over_c=round(t_a / t_c, 3),
                       a_kernels_ms=split(0), a_generic_kernels_ms=split(native.GRAD_FLAG_GENERIC),
                       workspace_bytes=native.grad_workspace_bytes(desc, T, native.GRAD_OP_WGRAD),
                       workspace_bytes_generic=native.grad_workspace_bytes(desc, T, native.GRAD_OP_WGRAD_GENERIC))
            out["rows"][f"{o}x{i}/T{T}"] = row
            print(f"{o}x{i} T={T}: {row}", file=sys.stderr, flush=True)
            torch.cuda.empty_cache()
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
