"""Decode of vector-length-16 layers (v16-k65536-256, fp16, perm and norm; synthetic weights): the default routing
against the v = 16 list kernel (include/vptq_b200_lists16.h, opt-in VQuantLinear.set_list_decode).

    python tools/bench_decode_v16.py [--steps 20] [--warmup 5] [--tokens 1,2,3,4] [--layers 80]

  * Llama-3-70B stack (the shapes of Llama-3.1-Nemotron-70B): 80 decoder layers x 7 linears, q/k/v and gate/up fused
    into one launch each, chained, one CUDA graph per step, programmatic dependent launch where the route has it.
    The 80 layers hold their own copies of one generated layer's tensors and lists: the same bytes at distinct
    addresses, so no layer is served from another's L2 lines (about 31 GB with the lists).
  * per-launch us of every 70B launch group, and of Llama-3.1-405B q / o, gate+up and down: eager back-to-back
    launches over all copies of that group (80 for 70B, --copies405 for 405B), CUDA events.
Routes: default = 1..2 tokens the generic GEMV (one token per pass), 3+ tokens dequant + wgmma GEMM per linear;
lists16 = vptq_b200_quant_gemv_lists16, one launch per fused group (where it takes the group: else per linear).
Prints one JSON line with the card, power limit and max SM clock read in the same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

K, KR, V = 65536, 256, 16


def make_layer(I, O, dev, gen, dt):
    """tensors of one synthetic v16-k65536-256 layer, packed on the GPU"""
    import torch
    from vptq_b200.pack import pack_index
    Ro = (O + V - 1) // V
    idx = torch.randint(0, K, (1, Ro, I), device=dev, generator=gen)
    ridx = torch.randint(0, KR, (1, Ro, I), device=dev, generator=gen)
    t = dict(indices=pack_index(idx, 16, ridx, 8))
    del idx, ridx
    rnd = lambda *s: torch.randn(*s, device=dev, generator=gen)
    t["centroids"] = (0.02 * rnd(1, K * V)).to(dt)
    t["res_centroids"] = (0.005 * rnd(1, KR * V)).to(dt)
    t["perm"] = torch.randperm(I, device=dev, generator=gen).to(torch.int32).to(torch.int16)
    t["weight_scale"] = (1.0 + 0.1 * rnd(I)).to(dt)
    t["weight_bias"] = (0.01 * rnd(I)).to(dt)
    return t


def descs_of(t, I, O, dt, lists16):
    from vptq_b200 import native
    d = native.make_desc(dtype=dt, in_features=I, out_features=O, vector_len=V, num_centroids=K, num_res_centroids=KR,
                         num_codebooks=1, group_size=I, outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1,
                         outlier_indices=None, outlier_centroids=None, bias=None, lists16=lists16, **t)
    d._t = t
    return d


def copy_desc(d, lists16):
    """the same layer at new addresses: its tensors, quantised-order scale / bias and lists cloned"""
    import ctypes
    from vptq_b200 import native
    t = {k: (v.clone() if v is not None else None) for k, v in d._t.items()}
    q = [x.clone() for x in d._keep]
    n = native.LinearDesc()
    ctypes.memmove(ctypes.addressof(n), ctypes.addressof(d), ctypes.sizeof(n))
    for k in ("indices", "centroids", "res_centroids", "perm", "weight_scale", "weight_bias"):
        setattr(n, k, t[k].data_ptr())
    n.weight_scale_q, n.weight_bias_q = q[0].data_ptr(), q[1].data_ptr()
    if lists16:
        n.lists_stream, n.lists_tab = q[2].data_ptr(), q[3].data_ptr()
    n._t, n._keep = t, tuple(q)
    return n


def gpu_info():
    from bench_decode_batch import gpu_info as g
    return g()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tokens", default="1,2,3,4")
    ap.add_argument("--layers", type=int, default=80)
    ap.add_argument("--copies405", type=int, default=6)
    a = ap.parse_args()

    import torch
    from vptq_b200 import native

    torch.cuda.set_device(0)
    dev, dt = torch.device("cuda:0"), torch.float16
    gen = torch.Generator(device=dev).manual_seed(0)
    toks = [int(t) for t in a.tokens.split(",")]
    result = dict(tool="bench_decode_v16", model="llama3-70b v16-k65536-256 synthetic", layers=a.layers,
                  steps=a.steps, warmup=a.warmup, **gpu_info(), routes={}, per_launch_us={})
    pdl = native.FLAG_PDL
    h, kv, f = 8192, 1024, 28672
    shapes = dict(q=(h, h), k=(h, kv), v=(h, kv), o=(h, h), gate=(h, f), up=(h, f), down=(f, h))
    # one generated layer with lists; the default route's descriptors point to the same tensors without them
    base = {n: descs_of(make_layer(I, O, dev, gen, dt), I, O, dt, True) for n, (I, O) in shapes.items()}
    stack = []
    for li in range(a.layers):
        L = {}
        for n, d in base.items():
            c = d if li == 0 else copy_desc(d, True)
            plain = native.make_desc(dtype=dt, in_features=d.in_features, out_features=d.out_features, vector_len=V,
                                     num_centroids=K, num_res_centroids=KR, num_codebooks=1, group_size=d.in_features,
                                     outlier_size=0, outlier_vector_len=-1, num_outlier_centroids=-1,
                                     outlier_indices=None, outlier_centroids=None, bias=None, lists16=False,
                                     **c._t)
            L[n] = dict(l16=c, plain=plain)
        stack.append(L)
    torch.cuda.synchronize()
    result["gpu_mem_gb"] = round(torch.cuda.memory_allocated() / 2 ** 30, 1)
    groups = [["q", "k", "v"], ["o"], ["gate", "up"], ["down"]]

    def plan(route, T):
        x0 = torch.randn(T, h, device=dev).to(dt)
        launches, x = [], x0
        for L in stack:
            qkv = torch.empty(T, h + 2 * kv, dtype=dt, device=dev)
            o = torch.empty(T, h, dtype=dt, device=dev)
            gu = torch.empty(T, 2 * f, dtype=dt, device=dev)
            down = torch.empty(T, h, dtype=dt, device=dev)
            io = [(x, [qkv[:, :h], qkv[:, h:h + kv], qkv[:, h + kv:]]), (qkv[:, :h], [o]),
                  (o, [gu[:, :f], gu[:, f:]]), (gu[:, :f], [down])]
            for names, (xin, ys) in zip(groups, io):
                if route == "lists16":
                    descs = [L[n]["l16"] for n in names]
                    if native.lists16_max_tokens(descs) >= T:
                        fn = native.FusedGemvLists16(descs, ys)
                        launches.append((lambda fn=fn, xin=xin: fn(xin, pdl), "+".join(names)))
                    else:
                        for d, y in zip(descs, ys):
                            fn = native.FusedGemvLists16([d], [y])
                            launches.append((lambda fn=fn, xin=xin: fn(xin, pdl), "+".join(names)))
                elif T <= 2:
                    fn = native.FusedGemv([L[n]["plain"] for n in names], ys)
                    launches.append((lambda fn=fn, xin=xin: fn(xin, pdl), "+".join(names)))
                else:
                    for n, y in zip(names, ys):
                        launches.append((lambda d=L[n]["plain"], y=y, xin=xin: native.quant_gemm(d, xin, y),
                                         "+".join(names)))
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

    for T in toks:
        for route in ("default", "lists16"):
            launches = plan(route, T)
            step = lambda: [fn() for fn, _ in launches]
            step()
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=s):
                    step()
            torch.cuda.synchronize()
            us = time_events(g.replay, a.steps, a.warmup)
            per = {}
            for key in dict.fromkeys(k for _, k in launches):
                same = [fn for fn, k in launches if k == key]          # every layer's launches of this group
                per[key] = round(time_events(lambda: [fn() for fn in same], 3, 1) / a.layers, 1)
            result["routes"][f"{route}_t{T}"] = dict(tokens=T, us_per_step=round(us, 1),
                                                     tokens_per_s=round(T * 1e6 / us, 1), us_per_launch=per)
            del g
    del stack, base
    torch.cuda.empty_cache()

    # Llama-3.1-405B: q / o (16384 x 16384), gate+up (2 x 53248 x 16384), down (16384 x 53248, default route only)
    for name, I, outs in (("405b_q_or_o", 16384, [16384]), ("405b_gate+up", 16384, [53248, 53248]),
                          ("405b_down", 53248, [16384])):
        first = [descs_of(make_layer(I, O, dev, gen, dt), I, O, dt, True) for O in outs]
        copies = [first] + [[copy_desc(d, bool(d.lists_stream)) for d in first] for _ in range(a.copies405 - 1)]
        r = {}
        for T in toks:
            x = torch.randn(T, I, device=dev).to(dt)
            for route in ("default", "lists16"):
                fns = []
                for ds in copies:
                    ys = [torch.empty(T, d.out_features, dtype=dt, device=dev) for d in ds]
                    if route == "lists16":
                        if native.lists16_max_tokens(ds) < T:
                            break
                        fns.append(lambda fn=native.FusedGemvLists16(ds, ys): fn(x, pdl))
                    elif T <= 2:
                        fns.append(lambda fn=native.FusedGemv(ds, ys): fn(x, pdl))
                    else:
                        fns += [lambda d=d, y=y: native.quant_gemm(d, x, y) for d, y in zip(ds, ys)]
                if fns:
                    r[f"{route}_t{T}"] = round(time_events(lambda: [fn() for fn in fns], 5, 2) / len(copies), 1)
        result["per_launch_us"][name] = r
        del copies, first
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
