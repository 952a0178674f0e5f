"""Generic decode GEMV (gemv_kernel, no index lists) at 2 tokens on the three Llama-3-8B layer shapes (K = 65536,
Kr = 256, perm, norm), fp16: mean time per call over CUDA events, several repeats, so that the spread between repeats
is visible next to the mean.

    python tools/bench_gemv_generic.py [--tokens 2] [--calls 200] [--repeats 5]

Prints one JSON object with the card name and power limit, read in the same process.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch

import vptq_oracle as vo
from _gpu import make_module
from vptq_b200 import native

SHAPES = {"4096x4096": (4096, 4096), "4096x14336": (4096, 14336), "14336x4096": (14336, 4096)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # (no nvidia-smi: the number still stands, without its card)
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=2)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    out = {"card": card(), "tokens": a.tokens, "calls": a.calls, "us_per_call": {}}
    for name, (i, o) in SHAPES.items():
        L = vo.make_layer(in_features=i, out_features=o, vector_len=8, num_centroids=65536, num_res_centroids=256,
                          seed=3)
        L.meta = {}
        m = make_module(L)
        os.environ["VPTQ_B200_LISTS"] = "0"
        m.prepare()
        d = m._desc_cache[0]
        assert not d.lists_stream
        x = torch.randn(a.tokens, i, device="cuda").half()
        y = torch.empty(a.tokens, o, device="cuda", dtype=torch.float16)
        for _ in range(20):
            native.quant_gemv(d, x, y)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.calls):
                native.quant_gemv(d, x, y)
            e1.record()
            torch.cuda.synchronize()
            times.append(round(e0.elapsed_time(e1) * 1e3 / a.calls, 2))
        out["us_per_call"][name] = times
        del m, d
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
