"""Prefill and input gradient of decode-only layers from the index lists, against the full layer's packed routes.

    python tools/bench_lists_prefill.py [--tokens 16 128 2048 8192] [--out FILE]

Llama-3-8B layer shapes (4096x4096, 14336x4096 = down, 4096x14336 = gate/up as out x in), K = 65536, Kr = 256,
perm and norm on, fp16, synthetic random indices and codebooks.  Per shape:
  * the dense weight alone: vptq_b200_lists_dequant (from the lists) against vptq_b200_dequant (packed words);
  * the whole op, forward (y = x W^T + bias) and input gradient (dX = dY W): the full module's routes against a
    decode-only copy (prepare(drop_packed=True)) with set_lists_prefill().
CUDA events, mean of 10 calls after 3 warm-up calls.  One JSON line per measurement, plus the GPU's name, power limit
and clocks first.  Needs a GPU: there is no CPU fall-back.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = ((4096, 4096), (4096, 14336), (14336, 4096))   # (in_features, out_features)
K, KR = 65536, 256


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired):
        out = []
    return {"query": q, "gpus": out, "torch_device": torch.cuda.get_device_name(0)}


def timed(fn, warmup=3, iters=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def make_layer(I, O, seed):
    from vptq_b200 import VQuantLinear
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = VQuantLinear(I, O, vector_lens=[-1, 8], num_centroids=[-1, K], num_res_centroids=[-1, KR], group_num=1,
                     group_size=I, outlier_size=0, indices_as_float=False, enable_norm=True, enable_perm=True,
                     is_indice_packed=True, bias=True, device="cuda", dtype=torch.float16, enable_proxy_error=False)
    with torch.no_grad():
        m.indices.data = torch.randint(-2**31, 2**31 - 1, m.indices.shape, generator=g, device="cuda",
                                       dtype=torch.int64).to(torch.int32)
        m.centroids.weight.data = (torch.randn(m.centroids.weight.shape, generator=g, device="cuda") * 0.02).half()
        m.res_centroids.weight.data = (torch.randn(m.res_centroids.weight.shape, generator=g, device="cuda") * 0.002).half()
        m.perm.data = torch.randperm(I, generator=g, device="cuda").to(torch.int16)
        m.weight_scale.data = (1 + 0.1 * torch.randn(I, generator=g, device="cuda")).half()
        m.weight_bias.data = (0.01 * torch.randn(I, generator=g, device="cuda")).half()
        m.bias.data = (0.01 * torch.randn(O, generator=g, device="cuda")).half()
    m.eval()
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, nargs="+", default=[16, 128, 2048, 8192])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lists_prefill needs a GPU")
    from vptq_b200 import native
    lines = [{"gpu": gpu_info()}]
    for I, O in SHAPES:
        full = make_layer(I, O, seed=I + O)
        dec = make_layer(I, O, seed=I + O)
        full.prepare()
        dec.prepare(drop_packed=True)
        dec.set_lists_prefill()
        dfull, ddec = full._desc_cache[0], dec._desc_cache[0]
        w = torch.empty(O, I, dtype=torch.float16, device="cuda")
        w2 = torch.empty(O, I, dtype=torch.float16, device="cuda")
        t_packed = timed(lambda: native.dequant(dfull, w))
        t_lists = timed(lambda: native.lists_dequant(ddec, w2, I))
        same = bool(torch.equal(w.view(torch.int16), w2.view(torch.int16)))
        lines.append({"shape": [O, I], "what": "dense weight", "packed_dequant_ms": round(t_packed, 4),
                      "lists_dequant_ms": round(t_lists, 4), "ratio": round(t_lists / t_packed, 3),
                      "bit_identical": same})
        del w, w2
        for T in a.tokens:
            x = (torch.randn(T, I, device="cuda") * 0.5).half()
            dy = (torch.randn(T, O, device="cuda") * 0.5).half()
            dx = torch.empty(T, I, dtype=torch.float16, device="cuda")
            with torch.no_grad():
                f_full = timed(lambda: full(x))
                f_dec = timed(lambda: dec(x))
                same = bool(torch.equal(full(x).view(torch.int16), dec(x).view(torch.int16)))
            b_full = timed(lambda: native.quant_gemm_dgrad(dfull, dy, dx))
            b_dec = timed(lambda: native.lists_quant_gemm(ddec, dy, dx, native.FLAG_TRANSPOSE))
            lines.append({"shape": [O, I], "tokens": T, "forward_full_ms": round(f_full, 4),
                          "forward_lists_ms": round(f_dec, 4), "forward_ratio": round(f_dec / f_full, 3),
                          "forward_bit_identical": same, "dgrad_full_ms": round(b_full, 4),
                          "dgrad_lists_ms": round(b_dec, 4), "dgrad_ratio": round(b_dec / b_full, 3)})
            del x, dy, dx
        del full, dec
        native.release_workspaces()
        torch.cuda.empty_cache()
    text = "\n".join(json.dumps(l) for l in lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
