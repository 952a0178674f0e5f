"""Decode steps of 1, 2, 4 and 8 tokens on Llama-3-8B v8-k65536-256 (synthetic weights, bench.py's layout): the
default routing against the batched list kernel (include/vptq_b200_batch.h).

    python tools/bench_decode_batch.py [--steps 50] [--warmup 10] [--tokens 1,2,4,8]

Every step is the 7 linears x 32 decoder layers, chained (q/k/v and gate/up fused into one launch each), captured
as one CUDA graph and launched with programmatic dependent launch where the route has it.  Routes:
  default  1 token: the single-token list kernel (vptq_b200_quant_gemv_multi_ws); 2 tokens: the generic GEMV
           (the same entry point); 3+ tokens: the dequant + wgmma GEMM, one launch per linear;
  batched  vptq_b200_quant_gemv_batch, one launch per fused group.
Prints one JSON line: us per step and tokens/s per (route, tokens), us per fused launch of layer 0 (CUDA events, eager
back-to-back launches), and the card, power limit and max SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return dict(card=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # (no nvidia-smi: the card name from torch only)
        import torch
        return dict(card=torch.cuda.get_device_name(0), power_limit=None, max_sm_clock=None, info_error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--tokens", default="1,2,4,8")
    ap.add_argument("--layers", type=int, default=32)
    a = ap.parse_args()

    import torch
    import bench
    from vptq_b200 import native

    torch.cuda.set_device(0)
    dev, dt = torch.device("cuda:0"), torch.float16
    m = dict(bench.LLAMA3_8B, layers=a.layers)
    stack = bench.build_stack(m, bench.QUANT, dev, 0, 1, dt)
    h, kv, f = m["hidden"], m["kv"], m["ffn"]
    pdl = native.FLAG_PDL
    result = dict(tool="bench_decode_batch", model="llama3-8b v8-k65536-256 synthetic", layers=m["layers"],
                  steps=a.steps, warmup=a.warmup, **gpu_info(), routes={})

    def plan(route, T):
        """[(fn, x, outputs)] per decoder layer, x of layer l + 1 = the down output of layer l"""
        x0 = torch.randn(T, h, device=dev).to(dt)
        launches, x = [], x0
        for L in stack:
            qkv = torch.empty(T, h + 2 * kv, dtype=dt, device=dev)
            o = torch.empty(T, h, dtype=dt, device=dev)
            gu = torch.empty(T, 2 * f, dtype=dt, device=dev)
            down = torch.empty(T, h, dtype=dt, device=dev)
            groups = [(["q", "k", "v"], x, [qkv[:, :h], qkv[:, h:h + kv], qkv[:, h + kv:]]),
                      (["o"], qkv[:, :h], [o]), (["gate", "up"], o, [gu[:, :f], gu[:, f:]]),
                      (["down"], gu[:, :f], [down])]
            for names, xin, ys in groups:
                descs = [L[n]["desc"] for n in names]
                if route == "batched":
                    fn = native.FusedGemvBatch(descs, ys)
                    launches.append((lambda fn=fn, xin=xin: fn(xin, pdl), names))
                elif T <= 2:
                    fn = native.FusedGemv(descs, ys)
                    launches.append((lambda fn=fn, xin=xin: fn(xin, pdl), names))
                else:
                    for d, y in zip(descs, ys):
                        launches.append((lambda d=d, y=y, xin=xin: native.quant_gemm(d, xin, y), names))
            x = down
        return launches

    def time_events(fn, n, warm):
        for _ in range(warm):
            fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(n):
            fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) * 1000.0 / n

    for T in [int(t) for t in a.tokens.split(",")]:
        for route in ("default", "batched"):
            if route == "batched" and native.batch_max_tokens([stack[0]["q"]["desc"]]) < T:
                continue
            launches = plan(route, T)
            step = lambda: [fn() for fn, _ in launches]
            step()
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()                                  # workspaces of this stream, outside the capture
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    step()
            torch.cuda.synchronize()
            us = time_events(g.replay, a.steps, a.warmup)
            per_launch = {}
            seen = set()
            for fn, names in launches:
                key = "+".join(names)
                if key in seen:
                    continue
                seen.add(key)
                same = [f2 for f2, n2 in launches[:len(launches) // m["layers"]] if n2 == names]
                per_launch[key] = round(time_events(lambda: [f2() for f2 in same], 200, 20), 2)
            result["routes"][f"{route}_t{T}"] = dict(tokens=T, us_per_step=round(us, 1),
                                                     tokens_per_s=round(T * 1e6 / us, 1), us_per_launch=per_launch)
            del g
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
