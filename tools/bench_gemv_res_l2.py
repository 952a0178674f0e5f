"""Decode GEMV of a layer whose residual codebook does not fit in shared memory: 4096 x 4096, v = 8, K = Kr = 65536
(b = 32, both codebooks 1 MiB and gathered through L1/L2 by gemv_kernel_res_l2), perm and norm, fp16.  For comparison
the same shape with Kr = 256 (gemv_kernel, residual in shared memory).  Mean time per call over CUDA events, several
repeats, at 1 and 2 tokens.

    python tools/bench_gemv_res_l2.py [--calls 200] [--repeats 5]

Prints one JSON object with the card name and power limit, read in the same process.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import torch

import vptq_oracle as vo
from _gpu import make_module
from bench_gemv_generic import card
from vptq_b200 import native


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    os.environ["VPTQ_B200_LISTS"] = "0"
    out = {"card": card(), "calls": a.calls, "us_per_call": {}}
    for Kr in (65536, 256):
        L = vo.make_layer(in_features=4096, out_features=4096, vector_len=8, num_centroids=65536, num_res_centroids=Kr,
                          seed=3)
        L.meta = {}
        m = make_module(L)
        m.prepare()
        d = m._desc_cache[0]
        assert not d.lists_stream
        for tokens in (1, 2):
            x = torch.randn(tokens, 4096, device="cuda").half()
            y = torch.empty(tokens, 4096, device="cuda", dtype=torch.float16)
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
            out["us_per_call"][f"kr{Kr}_t{tokens}"] = times
        del m, d
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
