"""Prefill timing: our fused path (prep + dequant + wgmma GEMM) vs torch (cuBLAS) on the same dequantised weight."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch
import vptq_oracle as vo
from _gpu import make_module

def timeit(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

out = {}
for (i, o) in ((4096, 4096), (4096, 14336), (14336, 4096)):
    L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=1)
    m = make_module(L)
    for T in (16, 256, 2048, 8192):
        x = torch.randn(T, i, device="cuda").half()
        t_ours = timeit(lambda: m(x))
        W = m.dequant()
        t_deq = timeit(lambda: m.dequant())
        t_cublas = timeit(lambda: torch.nn.functional.linear(x, W))
        fl = 2.0 * T * i * o
        out[f"{o}x{i}/T{T}"] = dict(ours_ms=round(t_ours, 4), ours_tflops=round(fl / t_ours / 1e9, 1),
                                   ref_style_dequant_ms=round(t_deq, 4), cublas_ms=round(t_cublas, 4),
                                   cublas_tflops=round(fl / t_cublas / 1e9, 1),
                                   dequant_plus_cublas_ms=round(t_deq + t_cublas, 4))
        print(f"{o}x{i} T={T}: {out[f'{o}x{i}/T{T}']}", flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "prefill_bench.json"), "w"), indent=1)
