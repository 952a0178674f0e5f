"""Prefill timing: our fused path (prep + dequant + wgmma GEMM) vs torch (cuBLAS) on the same dequantised weight.
The dgrad leg times the layer's input gradient dX = dY W (transposed dequant + wgmma GEMM) against m.dequant() +
torch.matmul(dY, W).  --legs picks the legs (default: both)."""
import os, sys, json, argparse
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch
import vptq_oracle as vo
from _gpu import make_module
from vptq_b200 import native

ap = argparse.ArgumentParser()
ap.add_argument("--legs", default="fwd,dgrad")
legs = ap.parse_args().legs.split(",")

def timeit(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

out = {"device": torch.cuda.get_device_name()}
for (i, o) in ((4096, 4096), (4096, 14336), (14336, 4096)):
    L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=1)
    m = make_module(L)
    if "fwd" in legs:
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
    if "dgrad" in legs:
        m.prepare()
        desc = m._desc_cache[0]
        for T in (2048, 8192):
            dy = torch.randn(T, o, device="cuda").half()
            dx = torch.empty(T, i, device="cuda", dtype=torch.float16)
            t_ours = timeit(lambda: native.quant_gemm_dgrad(desc, dy, dx))
            # share of the transposed dequant (kernel time from the profiler, run apart from the timed window)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(5): native.quant_gemm_dgrad(desc, dy, dx)
                torch.cuda.synchronize()
            t_tdq = sum(e.device_time_total for e in prof.key_averages() if "dequant_t" in e.key) / 5 / 1000
            W = m.dequant()
            t_deq = timeit(lambda: m.dequant())
            t_cublas = timeit(lambda: torch.matmul(dy, W))
            fl = 2.0 * T * i * o
            out[f"dgrad/{o}x{i}/T{T}"] = dict(ours_ms=round(t_ours, 4), ours_tflops=round(fl / t_ours / 1e9, 1),
                                             ours_transposed_dequant_ms=round(t_tdq, 4), dequant_ms=round(t_deq, 4), cublas_ms=round(t_cublas, 4),
                                             cublas_tflops=round(fl / t_cublas / 1e9, 1),
                                             dequant_plus_cublas_ms=round(t_deq + t_cublas, 4),
                                             ratio_vs_dequant_plus_cublas=round(t_ours / (t_deq + t_cublas), 3))
            print(f"dgrad {o}x{i} T={T}: {out[f'dgrad/{o}x{i}/T{T}']}", flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "prefill_bench.json"), "w"), indent=1)
