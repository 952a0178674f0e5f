"""Decode-only vector-length-16 layers (set_list_decode + set_lists_prefill + prepare(drop_packed=True)) against full
layers that keep their packed index words, on synthetic v16-k65536-256 layers (perm and norm on, random indices).

    python tools/bench_lists16_prefill.py [--tokens 16 128 2048 8192] [--out FILE]

  (a) the dense weight: vptq_b200_lists_dequant from the v = 16 lists, W and Wt, against the packed dequant
      (vptq_b200_dequant, the generic v = 16 kernel); Llama-3-70B q/o, k/v, gate/up, down and Llama-3.1-405B q in
      fp16, 70B q/o in bf16 too;
  (b) the whole op on the 70B shapes, fp16: forward (y = x W^T + bias) and input gradient (dX = dY W) of the
      decode-only module against the full module, both with set_list_decode;
  (c) one 70B decoder layer's seven linears: resident bytes with packed words + lists against lists only, times 80
      layers; and the 1..4-token step (the seven calls back to back), both routes with set_list_decode.
CUDA events, mean of 10 calls after 3 warm-ups.  One JSON line per measurement, the GPU's name, power limit and
clocks first.  Needs a GPU: there is no CPU fall-back.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

K, KR, V = 65536, 256, 16
SHAPES = {"70b_q_o": (8192, 8192), "70b_k_v": (8192, 1024), "70b_gate_up": (8192, 28672), "70b_down": (28672, 8192),
          "405b_q": (16384, 16384)}                                    # (in_features, out_features)
LAYER_70B = ((8192, 8192), (8192, 1024), (8192, 1024), (8192, 8192), (8192, 28672), (8192, 28672), (28672, 8192))


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


def module(I, O, dt, seed, decode_only):
    """a v16-k65536-256 VQuantLinear with bias and set_list_decode; decode_only: also set_lists_prefill and
    prepare(drop_packed=True)"""
    from bench_decode_v16 import make_layer
    from vptq_b200 import VQuantLinear
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = make_layer(I, O, "cuda", g, dt)
    m = VQuantLinear(I, O, vector_lens=[-1, V], num_centroids=[-1, K], num_res_centroids=[-1, KR], group_num=1,
                     group_size=I, outlier_size=0, indices_as_float=False, enable_norm=True, enable_perm=True,
                     is_indice_packed=True, bias=True, device="cuda", dtype=dt, enable_proxy_error=False)
    with torch.no_grad():
        m.indices.data = t["indices"]
        m.centroids.weight.data = t["centroids"]
        m.res_centroids.weight.data = t["res_centroids"]
        m.perm.data, m.weight_scale.data, m.weight_bias.data = t["perm"], t["weight_scale"], t["weight_bias"]
        m.bias.data = (0.01 * torch.randn(O, device="cuda", generator=g)).to(dt)
    m.eval().set_list_decode()
    if decode_only:
        m.set_lists_prefill().prepare(drop_packed=True)
    else:
        m.prepare()
    return m


def resident(m):
    """bytes of the module's parameters, buffers and descriptor-owned tensors (quantised-order scale / bias, lists)"""
    seen, n = set(), 0
    for t in list(m.parameters()) + list(m.buffers()) + list(m._desc_cache[0]._keep):
        if t.data_ptr() not in seen:
            seen.add(t.data_ptr())
            n += t.numel() * t.element_size()
    return n


def main():
    from bench_decode_batch import gpu_info
    from vptq_b200 import native
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, nargs="+", default=[16, 128, 2048, 8192])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lists16_prefill needs a GPU")
    lines = [{"gpu": gpu_info()}]

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)
    print(json.dumps(lines[0]), flush=True)

    # (a) the dense weight
    for name, (I, O) in list(SHAPES.items()) + [("70b_q_o_bf16", SHAPES["70b_q_o"])]:
        dt = torch.bfloat16 if name.endswith("bf16") else torch.float16
        m = module(I, O, dt, seed=I + O, decode_only=False)
        d = m._desc_cache[0]
        w, w2 = torch.empty(O, I, dtype=dt, device="cuda"), torch.empty(O, I, dtype=dt, device="cuda")
        ldt = (O + 63) // 64 * 64
        wt = torch.empty(I, ldt, dtype=dt, device="cuda")
        t_packed = timed(lambda: native.dequant(d, w))
        t_w = timed(lambda: native.lists_dequant(d, w2, I))
        t_wt = timed(lambda: native.lists_dequant(d, wt, ldt, native.FLAG_TRANSPOSE))
        emit({"part": "a", "shape": name, "O": O, "I": I, "packed_dequant_ms": round(t_packed, 4),
              "lists_w_ms": round(t_w, 4), "lists_wt_ms": round(t_wt, 4), "w_ratio": round(t_w / t_packed, 3),
              "wt_ratio": round(t_wt / t_packed, 3),
              "bit_identical": bool(torch.equal(w.view(torch.int16), w2.view(torch.int16)))})
        del m, d, w, w2, wt
        native.release_workspaces()
        torch.cuda.empty_cache()

    # (b) the whole op, 70B shapes
    for name in ("70b_q_o", "70b_k_v", "70b_gate_up", "70b_down"):
        I, O = SHAPES[name]
        full = module(I, O, torch.float16, seed=I + O, decode_only=False)
        dec = module(I, O, torch.float16, seed=I + O, decode_only=True)
        dfull, ddec = full._desc_cache[0], dec._desc_cache[0]
        for T in a.tokens:
            x = (torch.randn(T, I, device="cuda") * 0.5).half()
            dy = (torch.randn(T, O, device="cuda") * 0.5).half()
            dx = torch.empty(T, I, dtype=torch.float16, device="cuda")
            with torch.no_grad():
                f_full, f_dec = timed(lambda: full(x)), timed(lambda: dec(x))
                same = bool(torch.equal(full(x).view(torch.int16), dec(x).view(torch.int16)))
            b_full = timed(lambda: native.quant_gemm_dgrad(dfull, dy, dx))
            b_dec = timed(lambda: native.lists_quant_gemm(ddec, dy, dx, native.FLAG_TRANSPOSE))
            emit({"part": "b", "shape": name, "tokens": T, "forward_full_ms": round(f_full, 4),
                  "forward_lists_ms": round(f_dec, 4), "forward_ratio": round(f_dec / f_full, 3),
                  "forward_bit_identical": same, "dgrad_full_ms": round(b_full, 4),
                  "dgrad_lists_ms": round(b_dec, 4), "dgrad_ratio": round(b_dec / b_full, 3)})
            del x, dy, dx
        del full, dec, dfull, ddec
        native.release_workspaces()
        torch.cuda.empty_cache()

    # (c) one 70B decoder layer: resident bytes (x 80) and the 1..4-token step of its seven linears
    full = [module(I, O, torch.float16, seed=i, decode_only=False) for i, (I, O) in enumerate(LAYER_70B)]
    dec = [module(I, O, torch.float16, seed=i, decode_only=True) for i, (I, O) in enumerate(LAYER_70B)]
    rf, rd = sum(resident(m) for m in full), sum(resident(m) for m in dec)
    emit({"part": "c", "what": "resident bytes, 80 layers x 7 linears", "full_plus_lists_GB": round(80 * rf / 1e9, 2),
          "decode_only_GB": round(80 * rd / 1e9, 2), "freed_GB": round(80 * (rf - rd) / 1e9, 2)})
    for T in (1, 2, 3, 4):
        xs = {I: (torch.randn(T, I, device="cuda") * 0.5).half() for I in (8192, 28672)}
        with torch.no_grad():
            step = lambda ms: [m(xs[m.in_features]) for m in ms]
            t_full, t_dec = timed(lambda: step(full), iters=20), timed(lambda: step(dec), iters=20)
        emit({"part": "c", "tokens": T, "layer_step_full_ms": round(t_full, 4), "layer_step_decode_only_ms":
              round(t_dec, 4), "ratio": round(t_dec / t_full, 3)})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()
